"""Per-kernel CPU restatement of the C-ABI op contracts (TEST INFRASTRUCTURE ONLY).

`EmuOps` implements the interface of `micro_diffusion_b200.ops.CudaOps` with plain torch on CPU
tensors: same argument meaning, same output buffers, same storage dtypes (so bf16 rounding happens at
the same points as in the kernels).  It exists so that (a) the host-side engine -- buffer plans, index
arithmetic, the hand-written backward -- can be checked against `oracle.port` without a GPU, and
(b) every CUDA kernel has an op-level reference on the GPU box (tests/test_kernels_gpu.py).
It is never imported by `micro_diffusion_b200`.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

NT, TN = 0, 1
EPI_BF16, EPI_F32, EPI_RESID, EPI_ATOMIC, EPI_ACT_DUAL, EPI_ACT_GRAD, EPI_SWIGLU, EPI_SWIGLU_GRAD = 0, 1, 2, 3, 4, 5, 6, 7


def _f(t):
    return t.float()


def _expand_mod(m, T, rows):
    """[samples, D] -> [rows, D]"""
    return m.float().repeat_interleave(T, dim=0)[:rows]


def interleave_perm(f: int) -> torch.Tensor:
    """perm[p] = row of the natural w1 | w2 stack ([2f, D]) that sits at row p of the 32-interleaved stack."""
    p = torch.arange(2 * f)
    blk, inn = p // 64, p % 64
    return torch.where(inn < 32, 32 * blk + inn, f + 32 * blk + (inn - 32))


class EmuOps:
    is_emulation = True

    def __init__(self, device="cpu", exact=False):
        """exact=True keeps every "bf16" buffer in fp32 (no rounding anywhere): used to check the engine's
        hand-derived backward against autograd on the oracle to ~1e-5."""
        self.device = torch.device(device)
        self.launches = 0
        self.exact = exact
        self.lowp_dtype = torch.float32 if exact else torch.bfloat16

    def _r(self, t):
        """bf16 rounding point inside a kernel (identity in exact mode)"""
        return t if self.exact else t.bfloat16().float()

    def empty(self, shape, dtype):
        # poison so that reads of never-written memory show up in tests
        if self.exact and dtype == torch.bfloat16:
            dtype = torch.float32
        t = torch.empty(shape, dtype=dtype, device=self.device)
        if dtype.is_floating_point:
            t.fill_(float("nan"))
        else:
            t.fill_(-7777)
        return t

    def zeros(self, shape, dtype):
        if self.exact and dtype == torch.bfloat16:
            dtype = torch.float32
        return torch.zeros(shape, dtype=dtype, device=self.device)

    # ------------------------------------------------------------------ GEMM
    def gemm(self, A, B, Cm, *, layout=NT, epi=EPI_BF16, C2=None, bias=None, res=None, gate=None, rows_per_gate=0,
             res_mod=0, splits=1, act=0, alpha=1.0, aux=None, row_interleave=0):
        self.launches += 1
        batched = A.dim() == 3
        A3, B3, C3 = (A, B, Cm) if batched else (A.unsqueeze(0), B.unsqueeze(0), Cm.unsqueeze(0))
        assert self.exact or (A3.dtype == torch.bfloat16 and B3.dtype == torch.bfloat16)
        if layout == NT:
            acc = torch.einsum("bmk,bnk->bmn", _f(A3), _f(B3))
        else:
            acc = torch.einsum("bkm,bkn->bmn", _f(A3), _f(B3))
        acc = acc * (alpha if alpha != 0 else 1.0)
        if bias is not None:
            acc = acc + (bias.float().reshape(acc.shape[0], 1, -1) if bias.dim() == 2 else bias.float()[None, None, :])
        M = acc.shape[1]
        if epi == EPI_BF16:
            assert self.exact or Cm.dtype == torch.bfloat16
            C3.copy_(acc)
        elif epi == EPI_F32:
            assert Cm.dtype == torch.float32
            C3.copy_(acc)
        elif epi == EPI_ATOMIC:
            assert Cm.dtype == torch.float32 and bias is None, "the accumulate epilogue takes no bias"
            if row_interleave:  # rows arrive in the 32-interleaved order of a w1 | w2 stack, the gradient is in parameter order
                C3.index_add_(1, interleave_perm(row_interleave), acc)
            else:
                C3.add_(acc)
        elif epi == EPI_SWIGLU:
            # columns in the interleaved order: [64j, 64j+32) = u1 block j, [64j+32, 64j+64) = u2 block j
            u = self._r(acc)
            C3.copy_(u)
            nb = u.shape[-1] // 64
            ub = u.float().reshape(u.shape[0], u.shape[1], nb, 2, 32)
            h = F.silu(ub[:, :, :, 0]) * ub[:, :, :, 1]
            (C2 if batched else C2.unsqueeze(0)).copy_(h.reshape(u.shape[0], u.shape[1], nb * 32))
        elif epi == EPI_SWIGLU_GRAD:
            x3 = aux if batched else aux.unsqueeze(0)
            nb = acc.shape[-1] // 32
            ub = _f(x3).reshape(acc.shape[0], acc.shape[1], nb, 2, 32)
            a, b = ub[:, :, :, 0], ub[:, :, :, 1]
            d = acc.reshape(acc.shape[0], acc.shape[1], nb, 32)
            sg = torch.sigmoid(a)
            du = torch.stack([d * b * (sg * (1 + a * (1 - sg))), d * a * sg], dim=3)
            C3.copy_(du.reshape(acc.shape[0], acc.shape[1], nb * 64))
        elif epi == EPI_ACT_DUAL:
            assert (self.exact or Cm.dtype == torch.bfloat16) and C2 is not None
            pre = self._r(acc)
            C3.copy_(pre)
            a = F.gelu(pre.float(), approximate="tanh" if act == 1 else "none")
            (C2 if batched else C2.unsqueeze(0)).copy_(a)
        elif epi == EPI_ACT_GRAD:
            assert (self.exact or Cm.dtype == torch.bfloat16) and aux is not None and bias is None
            x3 = aux if batched else aux.unsqueeze(0)
            C3.copy_(acc * self._gelu_grad(_f(x3), act))
        elif epi == EPI_RESID:
            assert Cm.dtype == torch.float32 and res is not None
            if C2 is not None:
                (C2 if batched else C2.unsqueeze(0)).copy_(acc)
            if gate is not None:
                acc = acc * _expand_mod(gate, rows_per_gate, M)[None]
            r3 = res if res.dim() == 3 else res.unsqueeze(0)
            if res_mod > 0:
                idx = torch.arange(M) % res_mod
                r3 = r3[:, idx]
            C3.copy_(r3.float() + acc)
        else:
            raise ValueError(epi)

    # ------------------------------------------------------------------ norms
    def ln_fwd(self, x, y, mean, rstd, *, gamma=None, shift=None, scale=None, T, src_rows=None, eps=1e-6,
               y_add=None, gate_add=None, x_new=None):
        self.launches += 1
        rows, D = y.shape
        xv = _f(x).reshape(-1, D)
        if src_rows is not None:
            xv = xv[src_rows.long()]
        if y_add is not None:
            ya = _f(y_add).reshape(-1, D)
            if src_rows is not None:
                ya = ya[src_rows.long()]
            if gate_add is not None:
                ya = ya * _expand_mod(gate_add, T, rows)
            xv = xv + ya
            if src_rows is not None:
                x_new[src_rows.long()] = xv
            else:
                x_new.copy_(xv)
        mu = xv.mean(1, keepdim=True)
        var = ((xv - mu) ** 2).mean(1, keepdim=True)
        rs = torch.rsqrt(var + eps)
        o = (xv - mu) * rs
        if gamma is not None:
            o = o * gamma.float()
        if scale is not None:
            o = o * (1 + _expand_mod(scale, T, rows))
        if shift is not None:
            o = o + _expand_mod(shift, T, rows)
        y.copy_(o)
        if mean is not None:
            mean.copy_(mu.flatten())
        if rstd is not None:
            rstd.copy_(rs.flatten())

    def ln_bwd(self, dy, x, mean, rstd, *, gamma=None, scale=None, T, src_rows=None, dx=None, dx_mode=0,
               dgamma=None, dshift=None, dscale=None, dy_next=None, y_next=None, gate_next=None, dgate_next=None):
        self._ln_bwd(dy, x, mean, rstd, gamma=gamma, scale=scale, T=T, src_rows=src_rows, dx=dx, dx_mode=dx_mode,
                     dgamma=dgamma, dshift=dshift, dscale=dscale)
        if dy_next is not None:  # fused tail == gate_bwd on the updated dx
            assert dx is not None and dx_mode == 0
            self.launches -= 1
            self.gate_bwd(dx, dy_next, y=y_next, gate=gate_next, dgate=dgate_next, T=T)

    def _ln_bwd(self, dy, x, mean, rstd, *, gamma=None, scale=None, T, src_rows=None, dx=None, dx_mode=0,
                dgamma=None, dshift=None, dscale=None):
        self.launches += 1
        rows, D = dy.shape
        xv = _f(x).reshape(-1, D)
        if src_rows is not None:
            xv = xv[src_rows.long()]
        d = _f(dy)
        xh = (xv - mean[:, None]) * rstd[:, None]
        w = torch.ones(rows, D)
        if gamma is not None:
            w = w * gamma.float()
        if scale is not None:
            w = w * (1 + _expand_mod(scale, T, rows))
        g = d * w
        m1 = g.mean(1, keepdim=True)
        m2 = (g * xh).mean(1, keepdim=True)
        dxv = rstd[:, None] * (g - m1 - xh * m2)
        if dx is not None:
            if dx_mode == 0:
                dx.add_(dxv)
            elif dx_mode == 1:
                dx.copy_(dxv)
            else:
                dx.index_add_(0, src_rows.long(), dxv)
        ns = rows // T
        A = d.reshape(ns, T, D).sum(1)
        Bc = (d * xh).reshape(ns, T, D).sum(1)
        if dshift is not None:
            dshift.add_(A)
        if dscale is not None:
            dscale.add_(Bc * (gamma.float() if gamma is not None else 1.0))
        if dgamma is not None:
            dgamma.add_((Bc * ((1 + scale.float()) if scale is not None else 1.0)).sum(0))

    def rownorm_fwd(self, x, rstd, eps=1e-6, nslice=1):
        self.launches += 1
        rows, W = x.shape[0], x.shape[1] // nslice
        rv = rstd.view(nslice, rows)
        for s in range(nslice):
            xs = x[:, s * W:(s + 1) * W]
            xv = _f(xs)
            mu = xv.mean(1, keepdim=True)
            rs = torch.rsqrt(((xv - mu) ** 2).mean(1, keepdim=True) + eps)
            xs.copy_((xv - mu) * rs)
            rv[s].copy_(rs.flatten())

    def rownorm_bwd(self, dy, xhat, rstd, nslice=1):
        self.launches += 1
        rows, W = dy.shape[0], dy.shape[1] // nslice
        rv = rstd.view(nslice, rows)
        for s in range(nslice):
            ds = dy[:, s * W:(s + 1) * W]
            d, xh = _f(ds), _f(xhat[:, s * W:(s + 1) * W])
            m1 = d.mean(1, keepdim=True)
            m2 = (d * xh).mean(1, keepdim=True)
            ds.copy_(rv[s][:, None] * (d - m1 - xh * m2))

    def gate_bwd(self, dres, dy, *, y=None, gate=None, dgate=None, T):
        self.launches += 1
        rows, D = dres.shape
        o = dres.float()
        if gate is not None:
            o = o * _expand_mod(gate, T, rows)
        dy.copy_(o)
        if dgate is not None and y is not None:
            dgate.add_((dres.float() * _f(y)).reshape(rows // T, T, D).sum(1))

    # ------------------------------------------------------------------ attention
    @staticmethod
    def _heads(x, B, T, H, hd):
        return _f(x)[:, : H * hd].reshape(B, T, H, hd).permute(0, 2, 1, 3)

    def attn_fwd(self, q, k, v, o, lse, B, H, Tq, Tk, hd):
        self.launches += 1
        qh, kh, vh = self._heads(q, B, Tq, H, hd), self._heads(k, B, Tk, H, hd), self._heads(v, B, Tk, H, hd)
        s = torch.einsum("bhqd,bhkd->bhqk", qh, kh) / math.sqrt(hd)
        lse_nat = torch.logsumexp(s, dim=-1)
        p = torch.exp(s - lse_nat[..., None])
        out = torch.einsum("bhqk,bhkd->bhqd", self._r(p), vh)  # P is rounded to bf16 for the PV MMA
        o[:, : H * hd].copy_(out.permute(0, 2, 1, 3).reshape(B * Tq, H * hd))
        lse.copy_(lse_nat * 1.4426950408889634)

    def attn_bwd(self, dout, q, k, v, o, lse, delta, dq, dk, dv, B, H, Tq, Tk, hd):
        self.launches += 1
        qh, kh, vh = self._heads(q, B, Tq, H, hd), self._heads(k, B, Tk, H, hd), self._heads(v, B, Tk, H, hd)
        doh, oh = self._heads(dout, B, Tq, H, hd), self._heads(o, B, Tq, H, hd)
        scale = 1.0 / math.sqrt(hd)
        s = torch.einsum("bhqd,bhkd->bhqk", qh, kh) * scale
        p = torch.exp2(s * 1.4426950408889634 - lse[..., None])
        dl = (doh * oh).sum(-1)
        delta.copy_(dl)
        dvv = torch.einsum("bhqk,bhqd->bhkd", self._r(p), doh)
        dp = torch.einsum("bhqd,bhkd->bhqk", doh, vh)
        ds = self._r(p * (dp - dl[..., None]))
        dqq = torch.einsum("bhqk,bhkd->bhqd", ds, kh) * scale
        dkk = torch.einsum("bhqk,bhqd->bhkd", ds, qh) * scale
        dq[:, : H * hd].copy_(dqq.permute(0, 2, 1, 3).reshape(B * Tq, H * hd))
        dk[:, : H * hd].copy_(dkk.permute(0, 2, 1, 3).reshape(B * Tk, H * hd))
        dv[:, : H * hd].copy_(dvv.permute(0, 2, 1, 3).reshape(B * Tk, H * hd))

    # ------------------------------------------------------------------ feed-forward tails
    def swiglu_fwd(self, u, h):
        self.launches += 1
        f = h.shape[1]
        a, b = _f(u[:, :f]), _f(u[:, f:])
        h.copy_(F.silu(a) * b)

    def swiglu_bwd(self, dh, u, du):
        self.launches += 1
        f = dh.shape[1]
        a, b, d = _f(u[:, :f]), _f(u[:, f:]), _f(dh)
        sg = torch.sigmoid(a)
        du[:, :f].copy_(d * b * (sg * (1 + a * (1 - sg))))
        du[:, f:].copy_(d * a * sg)

    @staticmethod
    def _gelu_grad(x, act):
        with torch.enable_grad():
            x = x.detach().clone().requires_grad_(True)
            y = F.gelu(x, approximate="tanh" if act == 1 else "none")
            (g,) = torch.autograd.grad(y.sum(), x)
        return g.detach()

    def act_fwd(self, pre, out, act):
        self.launches += 1
        out.copy_(F.gelu(_f(pre), approximate="tanh" if act == 1 else "none"))

    def act_bwd(self, dact, pre, dpre, act):
        self.launches += 1
        dpre.copy_(_f(dact) * self._gelu_grad(_f(pre), act))

    def gelu_tanh_f32_fwd(self, c, out):
        self.launches += 1
        out.copy_(F.gelu(c.float(), approximate="tanh"))

    def gelu_tanh_f32_bwd(self, dact, c, dc, accumulate):
        self.launches += 1
        v = dact * self._gelu_grad(c, 1)
        if accumulate:
            dc.add_(v)
        else:
            dc.copy_(v)

    # ------------------------------------------------------------------ MoE
    def moe_gate_fwd(self, x, wg, probs):
        self.launches += 1
        probs.copy_(F.softmax(_f(x) @ wg.float().t(), dim=-1))

    def moe_topk(self, probs, idx, gval, inv, B, T, E, k):
        self.launches += 1
        pr = probs.reshape(B, T, E).permute(0, 2, 1)  # (B,E,T)
        # descending by prob, ties by lower token id (stable sort on the negated key)
        order = torch.sort(-pr, dim=-1, stable=True).indices
        top = order[..., :k]
        idx.copy_(top.to(torch.int32))
        gval.copy_(torch.gather(pr, 2, top))
        inv.fill_(-1)
        b_ix = torch.arange(B)[:, None, None].expand(B, E, k)
        e_ix = torch.arange(E)[None, :, None].expand(B, E, k)
        j_ix = torch.arange(k, dtype=torch.int32)[None, None, :].expand(B, E, k)
        inv.reshape(B, T, E)[b_ix, top, e_ix] = j_ix

    def moe_gather(self, x, idx, xin, B, T, E, k):
        self.launches += 1
        D = x.shape[1]
        rows = (torch.arange(B)[:, None, None] * T + idx.long().reshape(B, E, k))  # (B,E,k)
        xin.reshape(E, B, k, D).copy_(x[rows.permute(1, 0, 2)])

    def moe_combine_fwd(self, h2, gval, inv, xres, gate, xout, ymoe, B, T, E, k):
        self.launches += 1
        D = h2.shape[-1]
        h = _f(h2).reshape(E, B, k, D)
        acc = torch.zeros(B, T, D)
        iv = inv.reshape(B, T, E).long()
        for e in range(E):
            sel = iv[:, :, e] >= 0
            slot = iv[:, :, e].clamp(min=0)
            g = torch.gather(gval.reshape(B, E, k)[:, e], 1, slot)  # (B,T)
            hv = torch.gather(h[e], 1, slot[..., None].expand(B, T, D))
            acc += torch.where(sel[..., None], g[..., None] * hv, torch.zeros(()))
        acc = acc.reshape(B * T, D)
        if ymoe is not None:
            ymoe.copy_(acc)
        if xout is not None:
            gt = _expand_mod(gate, T, B * T) if gate is not None else 1.0
            xout.copy_(xres.float() + gt * acc)

    def moe_combine_bwd(self, dy, h2, gval, idx, dh2, dgval, B, T, E, k):
        self.launches += 1
        D = h2.shape[-1]
        rows = (torch.arange(B)[:, None, None] * T + idx.long().reshape(B, E, k))  # (B,E,k)
        dyr = _f(dy)[rows]  # (B,E,k,D)
        h = _f(h2).reshape(E, B, k, D).permute(1, 0, 2, 3)
        dgval.reshape(B, E, k).copy_((h * dyr).sum(-1))
        dh2.reshape(E, B, k, D).copy_((gval.reshape(B, E, k)[..., None] * dyr).permute(1, 0, 2, 3))

    def moe_dx_bwd(self, dxin, inv, dgval, probs, wg, dscores, dx, B, T, E, k):
        self.launches += 1
        D = dx.shape[-1]
        iv = inv.reshape(B, T, E).long()
        sel = iv >= 0
        slot = iv.clamp(min=0)
        # dgval is (B,E,k): pick [b, e, slot[b,t,e]]
        dg = dgval.reshape(B, E, k)
        dp = torch.stack([torch.gather(dg[:, e], 1, slot[:, :, e]) for e in range(E)], dim=-1)
        dp = torch.where(sel, dp, torch.zeros(()))
        pr = probs.reshape(B, T, E)
        ds = pr * (dp - (pr * dp).sum(-1, keepdim=True))
        dscores.copy_(ds.reshape(B * T, E))
        acc = ds.reshape(B * T, E) @ wg.float()
        dxi = _f(dxin).reshape(E, B, k, D)
        for e in range(E):
            hv = torch.gather(dxi[e], 1, slot[:, :, e][..., None].expand(B, T, D))
            acc += torch.where(sel[:, :, e][..., None], hv, torch.zeros(())).reshape(B * T, D)
        dx.copy_(acc)

    def moe_gate_wgrad(self, dscores, x, dwg):
        self.launches += 1
        dwg.add_(dscores.float().t() @ _f(x))

    # ------------------------------------------------------------------ masking
    def mask_sort(self, noise, ids_shuffle, ids_restore, mask, keep_rows, keep):
        self.launches += 1
        B, T = noise.shape
        sh = torch.sort(noise, dim=1, stable=True).indices
        rs = torch.argsort(sh, dim=1)
        if ids_shuffle is not None:
            ids_shuffle.copy_(sh.to(torch.int32))
        if ids_restore is not None:
            ids_restore.copy_(rs.to(torch.int32))
        if mask is not None:
            mask.copy_((rs >= keep).float())
        if keep_rows is not None:
            keep_rows.copy_((torch.arange(B)[:, None] * T + sh[:, :keep]).reshape(-1).to(torch.int32))

    def gather_rows(self, x, src_rows, y):
        self.launches += 1
        y.copy_(x[src_rows.long()])

    def scatter_rows(self, dy, src_rows, dx):
        self.launches += 1
        dx.index_add_(0, src_rows.long(), dy)

    # ------------------------------------------------------------------ EDM
    def cond_prepare(self, cap, keep, out, cap_out=None):
        self.launches += 1
        B = cap.shape[0]
        c = cap.reshape(B, -1)
        if keep is not None:
            c = (c * keep.reshape(B, 1).to(torch.float16)).to(torch.float16)
        out.reshape(B, -1).copy_(c.float())
        if cap_out is not None:
            cap_out.reshape(B, -1).copy_(c)

    def patchify(self, x, scale, patches, p):
        self.launches += 1
        B, Cc, H, W = x.shape
        v = x.float() * (scale.view(B, 1, 1, 1) if scale is not None else 1.0)
        pm = v.reshape(B, Cc, H // p, p, W // p, p).permute(0, 2, 4, 1, 3, 5)
        patches.copy_(pm.reshape(B * (H // p) * (W // p), Cc * p * p))

    def edm_prepare(self, lat, eps, rnd, sigma_in, p_mean, p_std, sigma_data, xn, patches, coef, p):
        self.launches += 1
        B, Cc, H, W = lat.shape
        sigma = sigma_in.float() if sigma_in is not None else torch.exp(rnd.float().flatten() * p_std + p_mean)
        sd = sigma_data
        coef[0].copy_(sigma)
        coef[1].copy_(sd ** 2 / (sigma ** 2 + sd ** 2))
        coef[2].copy_(sigma * sd / (sigma ** 2 + sd ** 2).sqrt())
        coef[3].copy_(1 / (sd ** 2 + sigma ** 2).sqrt())
        coef[4].copy_(sigma.log() / 4)
        coef[5].copy_((sigma ** 2 + sd ** 2) / (sigma * sd) ** 2)
        v = lat.float() + sigma.view(B, 1, 1, 1) * eps
        xn.copy_(v)
        pm = (coef[3].view(B, 1, 1, 1) * v).reshape(B, Cc, H // p, p, W // p, p).permute(0, 2, 4, 1, 3, 5)
        patches.copy_(pm.reshape(B * (H // p) * (W // p), Cc * p * p))

    def timestep_embed(self, t, out):
        self.launches += 1
        dim = out.shape[1]
        half = dim // 2
        freqs = torch.exp(-math.log(10000.0) * torch.arange(half, dtype=torch.float32) / half)
        a = t.float()[:, None] * freqs[None]
        out.copy_(torch.cat([torch.cos(a), torch.sin(a)], dim=-1))

    @staticmethod
    def _residual(ftok, keep_tok, lat, xn, coef, p, Tk):
        """(B,Tk,C,p,p) tensor of D - x at the kept patches."""
        B, Cc, H, W = lat.shape
        gw = W // p
        T = (H // p) * gw
        tok = (keep_tok.long().reshape(B, Tk) % T) if keep_tok is not None else torch.arange(T)[None].expand(B, T)

        def patches(img):
            return img.float().reshape(B, Cc, H // p, p, gw, p).permute(0, 2, 4, 1, 3, 5).reshape(B, T, Cc, p, p)

        sel = tok[:, :, None, None, None].expand(B, Tk, Cc, p, p)
        xp = torch.gather(patches(lat), 1, sel)
        xnp = torch.gather(patches(xn), 1, sel)
        f = ftok.float().reshape(B, Tk, p, p, Cc).permute(0, 1, 4, 2, 3)
        return coef[1].view(B, 1, 1, 1, 1) * xnp + coef[2].view(B, 1, 1, 1, 1) * f - xp

    def edm_loss_fwd(self, ftok, keep_tok, lat, xn, coef, per_sample, loss, p, Tk):
        self.launches += 1
        B, Cc = lat.shape[:2]
        d = self._residual(ftok, keep_tok, lat, xn, coef, p, Tk)
        ps = (coef[5].view(B, 1, 1, 1, 1) * d * d).sum(dim=(1, 2, 3, 4)) / (Cc * p * p) / Tk
        per_sample.copy_(ps)
        loss.add_(ps.mean())

    def edm_loss_bwd(self, ftok, keep_tok, lat, xn, coef, gscale, dftok, p, Tk):
        self.launches += 1
        B, Cc = lat.shape[:2]
        d = self._residual(ftok, keep_tok, lat, xn, coef, p, Tk)
        g = (gscale.float()[0] / B / Tk / (Cc * p * p)) * (coef[5] * 2 * coef[2]).view(B, 1, 1, 1, 1) * d
        dftok.copy_(g.permute(0, 1, 3, 4, 2).reshape(B * Tk, p * p * Cc))

    def edm_output(self, ftok, ids_restore, mask_token, xn, coef, fx, dx, p, Tk):
        self.launches += 1
        ref = fx if fx is not None else dx
        B, Cc, H, W = ref.shape
        T = (H // p) * (W // p)
        Nf = p * p * Cc
        f = ftok.float().reshape(B, Tk, Nf)
        if ids_restore is not None:
            mt = mask_token.float().reshape(1, 1, Nf) if mask_token is not None else torch.zeros(1, 1, Nf)
            full = torch.cat([f, mt.expand(B, T - Tk, Nf)], 1)
            f = torch.gather(full, 1, ids_restore.long().reshape(B, T)[..., None].expand(B, T, Nf))
        g = H // p
        img = f.reshape(B, g, W // p, p, p, Cc).permute(0, 5, 1, 3, 2, 4).reshape(B, Cc, H, W)
        if fx is not None:
            fx.copy_(img)
        if dx is not None:
            dx.copy_(coef[1].view(B, 1, 1, 1) * xn + coef[2].view(B, 1, 1, 1) * img)

    # ------------------------------------------------------------------ utilities
    def mean_tokens_fwd(self, x, out, B, L):
        self.launches += 1
        out.copy_(x.float().reshape(B, L, -1).mean(1))

    def mean_tokens_bwd(self, d, dx, B, L):
        self.launches += 1
        dx.reshape(B, L, -1).add_(d.float()[:, None, :] / L)

    def cast_bf16(self, x, y):
        self.launches += 1
        y.copy_(x)

    def colsum(self, x, out):
        self.launches += 1
        out.add_(_f(x).sum(0))

    def cast_transpose(self, w, wb, wbt, interleave_half=0):
        self.launches += 1
        if interleave_half:  # output row p holds parameter row perm[p]
            w = w.index_select(-2, interleave_perm(interleave_half))
        if wb is not None:
            wb.copy_(w)
        if wbt is not None:
            wbt.copy_(w.transpose(-1, -2))

    def set_deterministic(self, on=True, workspace_bytes=0):
        pass  # the CPU contracts are deterministic by construction

    def cast_transpose_multi(self, flat, wb, wbt, desc, total_tiles):
        self.launches += 1
        for off, rows, cols, half, need_t, _, _, _ in desc.tolist():
            n = rows * cols
            w = flat[off:off + n].view(rows, cols)
            if half:
                w = w.index_select(0, interleave_perm(half))
            wb[off:off + n].view(rows, cols).copy_(w)
            if need_t:
                wbt[off:off + n].view(cols, rows).copy_(w.t())

    def sumsq(self, x, out):
        self.launches += 1
        out.add_((x.double() ** 2).sum().float())

    def adamw(self, p, g, m, v, sumsq, clip, lr, beta1, beta2, eps, wd, step, nonfinite=None):
        self.launches += 1
        gs = 1.0
        if sumsq is not None and not math.isfinite(float(sumsq[0])):
            if nonfinite is not None:
                nonfinite.fill_(1)
            return
        if sumsq is not None and clip > 0:
            gs = min(1.0, clip / (float(sumsq[0]) ** 0.5 + 1e-6))
        gg = g * gs
        p.mul_(1 - lr * wd)
        m.mul_(beta1).add_(gg, alpha=1 - beta1)
        v.mul_(beta2).addcmul_(gg, gg, value=1 - beta2)
        bc1, bc2 = 1 - beta1 ** step, 1 - beta2 ** step
        p.addcdiv_(m, v.sqrt() / math.sqrt(bc2) + eps, value=-lr / bc1)
