"""Forward / backward orchestration of the MicroDiT training hot path over the C-ABI kernels.

One Python object drives the whole path LatentDiffusion.forward -> edm_loss -> model_forward_wrapper ->
DiT.forward_without_cfg (reference model.py:104-210, dit.py:455-519) and its hand-derived backward as a
fixed sequence of kernel launches on the current CUDA stream.  PyTorch provides device memory and the
autograd hook (`models/model.py` wraps `forward_loss`/`backward` in one autograd.Function); every FLOP
is in libmicrodit_b200.so.

Numerics: bf16 GEMM / attention operands with fp32 accumulation (the reference's amp_bf16 regime,
train.py:113); the residual stream, LayerNorm statistics, softmax, routing probabilities, loss and all
parameter gradients are fp32.  Saved activations are bf16 except the residual stream.
"""
from __future__ import annotations

import os
from types import SimpleNamespace as NS
from typing import Optional

import torch

from .arch import BlockSpec, DiTConfig
from .params import ParamStore

NT, TN = 0, 1
EPI_BF16, EPI_F32, EPI_RESID, EPI_ATOMIC, EPI_ACT_DUAL, EPI_ACT_GRAD, EPI_SWIGLU, EPI_SWIGLU_GRAD = 0, 1, 2, 3, 4, 5, 6, 7
ACT_ERF, ACT_TANH = 0, 1
BF16, F32, I32 = torch.bfloat16, torch.float32, torch.int32


class Engine:
    def __init__(self, cfg: DiTConfig, store: ParamStore, ops, sm_count: int = 132):
        self.cfg, self.store, self.ops = cfg, store, ops
        self.sm_count = sm_count
        self.fuse_act = os.environ.get("MD_FUSE_ACT", "1") != "0"  # expert GELU / GELU' in the GEMM epilogues (A/B knob)
        # gated-residual backward of the next branch emitted by the preceding LayerNorm backward (A/B knob)
        self.fuse_ln = os.environ.get("MD_FUSE_LN", "1") != "0"
        self.L = None  # caption length, set per call
        self._sampler_graphs = {}

    # ================================================================== helpers
    # True while backward_output(param_grads=False) runs: every weight-gradient GEMM, bias column sum and LayerNorm
    # d gamma is skipped and the flat gradient buffer is not touched
    _skip_wgrad = False

    def _gv(self, name):
        """Gradient view of one parameter, or None while weight gradients are skipped."""
        return None if self._skip_wgrad else self.store.g[name]

    def _Gv(self, name):
        """Gradient view of a GEMM group (ParamStore.G), or None while weight gradients are skipped."""
        return None if self._skip_wgrad else self.store.G(name)

    def _colsum(self, x, out):
        """Bias gradient out += column sums of x (skipped when out is None)."""
        if out is not None:
            self.ops.colsum(x, out)

    def _bkw(self, key):
        """{"bias": fp32 bias} of a use_bias Linear / stacked group (ParamStore.bias), {} when it has none: a bias-free model
        issues its GEMMs with exactly the arguments it always did."""
        b = self.store.bias(key)
        return {} if b is None else {"bias": b}

    def _gb(self, key):
        """Gradient view of the bias of a Linear / stacked group, or None (no bias, or weight gradients skipped)."""
        return None if self._skip_wgrad else self.store.gbias(key)

    def _wgrad(self, dY, X, G):
        """G[P,Q] (+)= dY[r,P]^T X[r,Q]  (reduction over the rows r); the library picks the split of the
        reduction that fills the SMs (splits=0).  Skipped when G is None."""
        if G is not None:
            self.ops.gemm(dY, X, G, layout=TN, epi=EPI_ATOMIC, splits=0)

    def _wgrad_w12(self, name, dU, X):
        """Weight gradient of a w1 | w2 stack; with the fused SwiGLU layout the rows of d u arrive interleaved."""
        if not self._skip_wgrad:
            self.ops.gemm(dU, X, self.store.G(name), layout=TN, epi=EPI_ATOMIC, splits=0,
                          row_interleave=self.store.interleave.get(name, 0))

    def _transposed(self, name):
        """Transposed bf16 copy of a matrix the training step never needs one of (the patch embed and the first caption
        projection, whose inputs are data): made on demand for the input gradients of backward_output."""
        st = self.store
        g = st.layout.groups[name]
        wt = self.ops.empty((g.cols, g.rows), BF16)
        self.ops.cast_transpose(st.flat[g.offset: g.offset + g.numel].view(g.rows, g.cols), None, wt)
        return wt

    def _swiglu_fwd(self, name_w12, x, u, hact):
        """u = x W12^T (+ [b1 | b2]), hact = silu(u1) * u2 (dit.py:88-89): one GEMM when the stack is interleaved (the
        epilogue maps the natural-order bias onto the interleaved columns), GEMM + pass otherwise."""
        o, st = self.ops, self.store
        if st.interleave.get(name_w12, 0):
            o.gemm(x, st.W(name_w12), u, epi=EPI_SWIGLU, C2=hact, **self._bkw(name_w12))
        else:
            o.gemm(x, st.W(name_w12), u, **self._bkw(name_w12))
            o.swiglu_fwd(u, hact)

    def _swiglu_bwd(self, name_w12, name_w3, dy, u, du):
        """du = d(silu(u1) * u2) for d hact = dy W3: inside the w3 dgrad GEMM when the stack is interleaved.  With biases,
        also the bias gradient of w1 | w2: the column sums of du, in [b1 | b2] order."""
        o, st = self.ops, self.store
        f = u.shape[1] // 2
        half = st.interleave.get(name_w12, 0)
        if half:
            o.gemm(dy, st.WT(name_w3), du, epi=EPI_SWIGLU_GRAD, aux=u)
        else:
            dh = o.empty((dy.shape[0], f), BF16)
            o.gemm(dy, st.WT(name_w3), dh)
            o.swiglu_bwd(dh, u, du)
        g12 = self._gb(name_w12)
        if g12 is not None:
            if half:
                o.colsum_interleaved(du, g12, half)
            else:
                o.colsum(du, g12)

    def _mods(self, key, D, mod):
        o = self.store.layout.ada_offset[key]
        return [mod[:, o + i * D: o + (i + 1) * D] for i in range(6)]

    # ================================================================== stage-wide caption K/V projection
    def _kv_fwd(self, group, ykv, nblk, D2):
        """kv_linear of every block of a stage in one GEMM: [B*L, Dy] x [nblk*2D, Dy]^T (utils.py:118)."""
        o, st = self.ops, self.store
        kv_all = o.empty((ykv.shape[0], nblk * D2), BF16)
        o.gemm(ykv, st.W(group), kv_all, **self._bkw(group))
        return kv_all

    def _kv_bwd(self, group, dkv_all, ykv, dykv):
        """Weight (and bias) gradient of the stacked kv_linear and the gradient flowing into the caption tokens."""
        o, st = self.ops, self.store
        self._colsum(dkv_all, self._gb(group))
        self._wgrad(dkv_all, ykv, self._Gv(group))
        o.gemm(dkv_all, st.WT(group), dykv, epi=EPI_RESID, res=dykv)

    # ================================================================== block forward
    def _ln_add(self, x, pend, out, mean, rstd, *, gamma, shift=None, scale=None, T, src_rows=None, rows_all=None):
        """LayerNorm of (x + pending gated residual).  `pend` = (y bf16, gate view | None) left by the previous
        sub-block, applied here instead of in that sub-block's GEMM epilogue.  Returns the updated stream."""
        o = self.ops
        if pend is None:
            o.ln_fwd(x, out, mean, rstd, gamma=gamma, shift=shift, scale=scale, T=T, src_rows=src_rows, eps=self.cfg.norm_eps)
            return x
        xn = o.empty(tuple(x.shape), F32)
        o.ln_fwd(x, out, mean, rstd, gamma=gamma, shift=shift, scale=scale, T=T, src_rows=src_rows, eps=self.cfg.norm_eps,
                 y_add=pend[0], gate_add=pend[1], x_new=xn)
        return xn

    def _materialize(self, x, pend, T):
        """Apply a pending residual where a plain tensor is needed (only reached by non-zoo configurations)."""
        if pend is None:
            return x
        o = self.ops
        scratch = o.empty(tuple(x.shape), BF16)
        return self._ln_add(x, pend, scratch, None, None, gamma=None, T=T)

    def _block_fwd(self, bs: BlockSpec, x, pend, kv, B, T, L, mod, keep: bool, kv_normed: bool = False):
        """One DiTBlock (dit.py:232-239).  `x` + `pend` is the block input; returns (stream, pending, saved)."""
        o, st, cfg = self.ops, self.store, self.cfg
        P = st.p
        n, D, h, f, hd = bs.name, bs.dim, bs.attn_dim, bs.ffn_dim, cfg.head_dim
        M = B * T
        eps = cfg.norm_eps
        sh_a, sc_a, g_a, sh_m, sc_m, g_m = self._mods(n, D, mod)
        sv = NS()
        # ---- self attention (dit.py:236, utils.py:178-196)
        sv.xm = o.empty((M, D), BF16); sv.mean1 = o.empty((M,), F32); sv.rstd1 = o.empty((M,), F32)
        sv.x = self._ln_add(x, pend, sv.xm, sv.mean1, sv.rstd1, gamma=P[n + ".norm1.weight"], shift=sh_a, scale=sc_a, T=T)
        sv.qkv = o.empty((M, 3 * h), BF16)
        o.gemm(sv.xm, st.W(n + ".attn.qkv.weight"), sv.qkv, **self._bkw(n + ".attn.qkv.weight"))
        sv.rqk = o.empty((2, M), F32)  # ln_q and ln_k (utils.py:183-186) in one launch: adjacent slices of qkv
        o.rownorm_fwd(sv.qkv[:, :2 * h], sv.rqk, eps, nslice=2)
        sv.att = o.empty((M, h), BF16); sv.lse = o.empty((B, bs.heads, T), F32)
        o.attn_fwd(sv.qkv[:, :h], sv.qkv[:, h:2 * h], sv.qkv[:, 2 * h:], sv.att, sv.lse, B, bs.heads, T, T, hd)
        sv.ya = o.empty((M, D), BF16)
        o.gemm(sv.att, st.W(n + ".attn.proj.weight"), sv.ya, **self._bkw(n + ".attn.proj.weight"))
        # ---- cross attention to the caption tokens (dit.py:237, utils.py:116-136)
        sv.xn2 = o.empty((M, D), BF16); sv.mean2 = o.empty((M,), F32); sv.rstd2 = o.empty((M,), F32)
        sv.x1 = self._ln_add(sv.x, (sv.ya, g_a), sv.xn2, sv.mean2, sv.rstd2, gamma=P[n + ".norm2.weight"], T=T)
        sv.qx = o.empty((M, D), BF16)
        o.gemm(sv.xn2, st.W(n + ".cross_attn.q_linear.weight"), sv.qx, **self._bkw(n + ".cross_attn.q_linear.weight"))
        sv.kv = kv  # this block's [B*L, 2D] column slice of the stage-wide K/V projection
        sv.rq2 = o.empty((M,), F32); sv.rk2 = o.empty((B * L,), F32)
        o.rownorm_fwd(sv.qx, sv.rq2, eps)
        if not kv_normed:  # a PromptCache holds K already normalised
            o.rownorm_fwd(sv.kv[:, :D], sv.rk2, eps)
        sv.att2 = o.empty((M, D), BF16); sv.lse2 = o.empty((B, bs.xheads, T), F32)
        o.attn_fwd(sv.qx, sv.kv[:, :D], sv.kv[:, D:], sv.att2, sv.lse2, B, bs.xheads, T, L, hd)
        yx = o.empty((M, D), BF16)
        o.gemm(sv.att2, st.W(n + ".cross_attn.proj.weight"), yx, **self._bkw(n + ".cross_attn.proj.weight"))
        # ---- feed-forward (dit.py:238)
        sv.xm3 = o.empty((M, D), BF16); sv.mean3 = o.empty((M,), F32); sv.rstd3 = o.empty((M,), F32)
        sv.x2 = self._ln_add(sv.x1, (yx, None), sv.xm3, sv.mean3, sv.rstd3, gamma=P[n + ".norm3.weight"], shift=sh_m,
                             scale=sc_m, T=T)
        sv.ym = o.empty((M, D), BF16)
        if not bs.moe:  # SwiGLU (dit.py:88-89); its gated residual is left pending for the next LayerNorm
            sv.u = o.empty((M, 2 * f), BF16)
            sv.hact = o.empty((M, f), BF16)
            self._swiglu_fwd(n + ".mlp.w12", sv.xm3, sv.u, sv.hact)
            o.gemm(sv.hact, st.W(n + ".mlp.w3.weight"), sv.ym, **self._bkw(n + ".mlp.w3.weight"))
            out, pend_out = sv.x2, (sv.ym, g_m)
        else:  # expert-choice MoE (dit.py:126-143): the combine kernel applies the gated residual itself
            E = cfg.num_experts
            k = int(cfg.expert_capacity * T / E)
            sv.k = k
            sv.probs = o.empty((M, E), F32)
            o.moe_gate_fwd(sv.xm3, P[n + ".mlp.gate.weight"], sv.probs)
            sv.idx = o.empty((B, E, k), I32); sv.gval = o.empty((B, E, k), F32); sv.inv = o.empty((B, T, E), I32)
            o.moe_topk(sv.probs, sv.idx, sv.gval, sv.inv, B, T, E, k)
            sv.xin = o.empty((E, B * k, D), BF16)
            o.moe_gather(sv.xm3, sv.idx, sv.xin, B, T, E, k)
            sv.hpre = o.empty((E, B * k, f), BF16); sv.hact = o.empty((E, B * k, f), BF16)
            # GELU in the epilogue of the first expert GEMM (8 epilogue warps, both outputs through TMA stores): the
            # [E, B*k, f] hidden tensor is written once as pre-activation and once as activation, never re-read here
            if self.fuse_act:
                o.gemm(sv.xin, st.WT(n + ".mlp.w1"), sv.hpre, epi=EPI_ACT_DUAL, C2=sv.hact, act=ACT_ERF)
            else:
                o.gemm(sv.xin, st.WT(n + ".mlp.w1"), sv.hpre)
                o.act_fwd(sv.hpre, sv.hact, ACT_ERF)
            sv.h2 = o.empty((E, B * k, D), BF16)
            o.gemm(sv.hact, st.WT(n + ".mlp.w2"), sv.h2)
            out = o.empty((M, D), F32)
            o.moe_combine_fwd(sv.h2, sv.gval, sv.inv, sv.x2, g_m, out, sv.ym, B, T, E, k)
            pend_out = None
        return out, pend_out, (sv if keep else None)

    # ================================================================== block backward
    def _ffn_gate_args(self, bs: BlockSpec, sv, mod, dmod):
        """What the backward chain needs to enter a block's feed-forward branch: y, gate and d gate of x + g_m * y."""
        return dict(y_next=sv.ym, gate_next=self._mods(bs.name, bs.dim, mod)[5], dgate_next=self._mods(bs.name, bs.dim, dmod)[5])

    def _block_bwd(self, bs: BlockSpec, sv, dx, dkv, B, T, L, mod, dmod, dy_in=None, nxt=None):
        """dx (f32 [M,D]): in = grad wrt the block output, out = grad wrt the block input (in place).
        dkv (bf16 [B*L, 2D] column slice of the stage-wide buffer) receives d loss / d (K, V) of this block.
        dy_in: gate_m * dx already in bf16 (emitted by the LayerNorm backward that produced dx); nxt: the
        _ffn_gate_args of the block the chain enters next -- this block's last LayerNorm backward then emits that
        block's dy_in, which is returned."""
        o, st, cfg = self.ops, self.store, self.cfg
        P = st.p
        n, D, h, f, hd = bs.name, bs.dim, bs.attn_dim, bs.ffn_dim, cfg.head_dim
        M = B * T
        fuse = self.fuse_ln
        sh_a, sc_a, g_a, sh_m, sc_m, g_m = self._mods(n, D, mod)
        dsh_a, dsc_a, dg_a, dsh_m, dsc_m, dg_m = self._mods(n, D, dmod)
        # ---- feed-forward branch
        if dy_in is None:
            dy = o.empty((M, D), BF16)
            o.gate_bwd(dx, dy, y=sv.ym, gate=g_m, dgate=dg_m, T=T)
        else:
            dy = dy_in
        dxm = o.empty((M, D), BF16)
        if not bs.moe:
            self._colsum(dy, self._gb(n + ".mlp.w3.weight"))
            du = o.empty((M, 2 * f), BF16)
            self._swiglu_bwd(n + ".mlp.w12", n + ".mlp.w3.weight", dy, sv.u, du)
            self._wgrad(dy, sv.hact, self._Gv(n + ".mlp.w3.weight"))
            o.gemm(du, st.WT(n + ".mlp.w12"), dxm)
            self._wgrad_w12(n + ".mlp.w12", du, sv.xm3)
        else:
            E, k = cfg.num_experts, sv.k
            dh2 = o.empty((E, B * k, D), BF16); dgval = o.empty((B, E, k), F32)
            o.moe_combine_bwd(dy, sv.h2, sv.gval, sv.idx, dh2, dgval, B, T, E, k)
            dhpre = o.empty((E, B * k, f), BF16)
            if self.fuse_act:  # d hact -> d hpre inside the dgrad GEMM's epilogue (GELU' at the saved pre-activation)
                o.gemm(dh2, st.W(n + ".mlp.w2"), dhpre, epi=EPI_ACT_GRAD, aux=sv.hpre, act=ACT_ERF)
            else:
                dhact = o.empty((E, B * k, f), BF16)
                o.gemm(dh2, st.W(n + ".mlp.w2"), dhact)
                o.act_bwd(dhact, sv.hpre, dhpre, ACT_ERF)
            self._wgrad(sv.hact, dh2, self._Gv(n + ".mlp.w2"))
            dxin = o.empty((E, B * k, D), BF16)
            o.gemm(dhpre, st.W(n + ".mlp.w1"), dxin)
            self._wgrad(sv.xin, dhpre, self._Gv(n + ".mlp.w1"))
            dscores = o.empty((M, E), F32)
            o.moe_dx_bwd(dxin, sv.inv, dgval, sv.probs, P[n + ".mlp.gate.weight"], dscores, dxm, B, T, E, k)
            if not self._skip_wgrad:
                o.moe_gate_wgrad(dscores, sv.xm3, self._gv(n + ".mlp.gate.weight"))
        dy = o.empty((M, D), BF16)
        o.ln_bwd(dxm, sv.x2, sv.mean3, sv.rstd3, gamma=P[n + ".norm3.weight"], scale=sc_m, T=T, dx=dx, dx_mode=0,
                 dgamma=self._gv(n + ".norm3.weight"), dshift=dsh_m, dscale=dsc_m, dy_next=dy if fuse else None)
        # ---- cross attention branch (no gate, no modulation): dy = bf16(dx)
        if not fuse:
            o.gate_bwd(dx, dy, T=T)
        self._colsum(dy, self._gb(n + ".cross_attn.proj.weight"))
        datt2 = o.empty((M, D), BF16)
        o.gemm(dy, st.WT(n + ".cross_attn.proj.weight"), datt2)
        self._wgrad(dy, sv.att2, self._Gv(n + ".cross_attn.proj.weight"))
        dqx = o.empty((M, D), BF16)
        delta = o.empty((B, bs.xheads, T), F32)
        o.attn_bwd(datt2, sv.qx, sv.kv[:, :D], sv.kv[:, D:], sv.att2, sv.lse2, delta, dqx, dkv[:, :D], dkv[:, D:], B,
                   bs.xheads, T, L, hd)
        o.rownorm_bwd(dqx, sv.qx, sv.rq2)
        o.rownorm_bwd(dkv[:, :D], sv.kv[:, :D], sv.rk2)
        self._colsum(dqx, self._gb(n + ".cross_attn.q_linear.weight"))
        dxn2 = o.empty((M, D), BF16)
        o.gemm(dqx, st.WT(n + ".cross_attn.q_linear.weight"), dxn2)
        self._wgrad(dqx, sv.xn2, self._Gv(n + ".cross_attn.q_linear.weight"))
        dy = o.empty((M, D), BF16)
        if fuse:
            o.ln_bwd(dxn2, sv.x1, sv.mean2, sv.rstd2, gamma=P[n + ".norm2.weight"], T=T, dx=dx, dx_mode=0,
                     dgamma=self._gv(n + ".norm2.weight"), dy_next=dy, y_next=sv.ya, gate_next=g_a, dgate_next=dg_a)
        else:
            o.ln_bwd(dxn2, sv.x1, sv.mean2, sv.rstd2, gamma=P[n + ".norm2.weight"], T=T, dx=dx, dx_mode=0,
                     dgamma=self._gv(n + ".norm2.weight"))
            o.gate_bwd(dx, dy, y=sv.ya, gate=g_a, dgate=dg_a, T=T)
        # ---- self attention branch
        self._colsum(dy, self._gb(n + ".attn.proj.weight"))
        datt = o.empty((M, h), BF16)
        o.gemm(dy, st.WT(n + ".attn.proj.weight"), datt)
        self._wgrad(dy, sv.att, self._Gv(n + ".attn.proj.weight"))
        dqkv = o.empty((M, 3 * h), BF16)
        delta = o.empty((B, bs.heads, T), F32)
        o.attn_bwd(datt, sv.qkv[:, :h], sv.qkv[:, h:2 * h], sv.qkv[:, 2 * h:], sv.att, sv.lse, delta, dqkv[:, :h],
                   dqkv[:, h:2 * h], dqkv[:, 2 * h:], B, bs.heads, T, T, hd)
        o.rownorm_bwd(dqkv[:, :2 * h], sv.qkv[:, :2 * h], sv.rqk, nslice=2)
        self._colsum(dqkv, self._gb(n + ".attn.qkv.weight"))
        dxm1 = o.empty((M, D), BF16)
        o.gemm(dqkv, st.WT(n + ".attn.qkv.weight"), dxm1)
        self._wgrad(dqkv, sv.xm, self._Gv(n + ".attn.qkv.weight"))
        dy_out = o.empty((M, D), BF16) if (fuse and nxt is not None) else None
        o.ln_bwd(dxm1, sv.x, sv.mean1, sv.rstd1, gamma=P[n + ".norm1.weight"], scale=sc_a, T=T, dx=dx, dx_mode=0,
                 dgamma=self._gv(n + ".norm1.weight"), dshift=dsh_a, dscale=dsc_a, dy_next=dy_out,
                 **(nxt if dy_out is not None else {}))
        return dy_out

    # ================================================================== conditioning stem
    def _stem_fwd(self, cap, drop, cnoise, B, keep: bool, cap_out=None):
        """dit.py:480-485 + the stacked adaLN linear: caption half, then the time-dependent half."""
        return self._time_fwd(self._caption_fwd(cap, drop, B, cap_out), cnoise, B)

    def _caption_fwd(self, cap, drop, B, cap_out=None):
        """Everything of the conditioning stem that depends on the caption only (dit.py:481-484)."""
        o, st, cfg = self.ops, self.store, self.cfg
        P = st.p
        D, hd, eps = cfg.dim, cfg.head_dim, cfg.norm_eps
        L = cap.shape[-2]
        R = B * L
        s = NS(L=L)
        s.ycap = o.empty((R, cap.shape[-1]), BF16)
        if cap.dtype == torch.float16:
            o.cond_prepare(cap.reshape(B, -1), drop, s.ycap, cap_out)
        else:
            raise TypeError("caption_latents must be float16 (the batch contract of latents_loader.py:52-55)")
        # CaptionProjection = Mlp(fc1 -> GELU-tanh -> LN -> fc2) (utils.py:63-68, 317-318)
        s.a1pre = o.empty((R, D), BF16); s.a1 = o.empty((R, D), BF16)
        o.gemm(s.ycap, st.W("y_embedder.y_proj.fc1.weight"), s.a1pre, epi=EPI_ACT_DUAL, C2=s.a1,
               bias=P["y_embedder.y_proj.fc1.bias"], act=ACT_TANH)
        s.a1n = o.empty((R, D), BF16); s.m_a = o.empty((R,), F32); s.r_a = o.empty((R,), F32)
        o.ln_fwd(s.a1, s.a1n, s.m_a, s.r_a, gamma=P["y_embedder.y_proj.norm.weight"], T=L, eps=eps)
        s.y0 = o.empty((R, D), F32)
        o.gemm(s.a1n, st.W("y_embedder.y_proj.fc2.weight"), s.y0, epi=EPI_F32, bias=P["y_embedder.y_proj.fc2.bias"])
        # AttentionBlockPromptEmbedding (dit.py:53-56)
        H = D // hd
        s.yn1 = o.empty((R, D), BF16); s.m1 = o.empty((R,), F32); s.r1 = o.empty((R,), F32)
        o.ln_fwd(s.y0, s.yn1, s.m1, s.r1, gamma=P["y_emb_preprocess.norm1.weight"], T=L, eps=eps)
        s.qkv = o.empty((R, 3 * D), BF16)
        o.gemm(s.yn1, st.W("y_emb_preprocess.attn.qkv.weight"), s.qkv, **self._bkw("y_emb_preprocess.attn.qkv.weight"))
        s.rqk = o.empty((2, R), F32)
        o.rownorm_fwd(s.qkv[:, :2 * D], s.rqk, eps, nslice=2)
        s.att = o.empty((R, D), BF16); s.lse = o.empty((B, H, L), F32)
        o.attn_fwd(s.qkv[:, :D], s.qkv[:, D:2 * D], s.qkv[:, 2 * D:], s.att, s.lse, B, H, L, L, hd)
        s.y1 = o.empty((R, D), F32)
        o.gemm(s.att, st.W("y_emb_preprocess.attn.proj.weight"), s.y1, epi=EPI_RESID, res=s.y0,
               **self._bkw("y_emb_preprocess.attn.proj.weight"))
        fp = cfg.prompt_ffn_dim
        s.yn2 = o.empty((R, D), BF16); s.m2 = o.empty((R,), F32); s.r2 = o.empty((R,), F32)
        o.ln_fwd(s.y1, s.yn2, s.m2, s.r2, gamma=P["y_emb_preprocess.norm2.weight"], T=L, eps=eps)
        s.u = o.empty((R, 2 * fp), BF16)
        s.hact = o.empty((R, fp), BF16)
        self._swiglu_fwd("y_emb_preprocess.mlp.w12", s.yn2, s.u, s.hact)
        s.y2 = o.empty((R, D), F32)
        o.gemm(s.hact, st.W("y_emb_preprocess.mlp.w3.weight"), s.y2, epi=EPI_RESID, res=s.y1,
               **self._bkw("y_emb_preprocess.mlp.w3.weight"))
        s.ybf = o.empty((R, D), BF16)
        o.cast_bf16(s.y2, s.ybf)
        # pooled caption -> Mlp (dit.py:484)
        s.pool = o.empty((B, D), BF16)
        o.mean_tokens_fwd(s.y2, s.pool, B, L)
        s.p1pre = o.empty((B, D), BF16); s.p1 = o.empty((B, D), BF16)
        o.gemm(s.pool, st.W("pooled_y_emb_process.fc1.weight"), s.p1pre, epi=EPI_ACT_DUAL, C2=s.p1,
               bias=P["pooled_y_emb_process.fc1.bias"], act=ACT_TANH)
        s.p1n = o.empty((B, D), BF16); s.m_p = o.empty((B,), F32); s.r_p = o.empty((B,), F32)
        o.ln_fwd(s.p1, s.p1n, s.m_p, s.r_p, gamma=P["pooled_y_emb_process.norm.weight"], T=1, eps=eps)
        return s

    def _time_fwd(self, s, cnoise, B):
        """TimestepEmbedder on c_noise (utils.py:283-285; dit.py:480), c = t + pooled caption, all adaLN vectors."""
        o, st, cfg = self.ops, self.store, self.cfg
        P = st.p
        D = cfg.dim
        s.tfreq = o.empty((B, cfg.freq_dim), BF16)
        o.timestep_embed(cnoise, s.tfreq)
        s.t1pre = o.empty((B, D), BF16); s.t1 = o.empty((B, D), BF16)
        o.gemm(s.tfreq, st.W("t_embedder.mlp.0.weight"), s.t1pre, epi=EPI_ACT_DUAL, C2=s.t1,
               bias=P["t_embedder.mlp.0.bias"], act=ACT_TANH)
        s.temb = o.empty((B, D), F32)
        o.gemm(s.t1, st.W("t_embedder.mlp.2.weight"), s.temb, epi=EPI_F32, bias=P["t_embedder.mlp.2.bias"])
        # c = t + pooled (dit.py:485)
        s.c = o.empty((B, D), F32)
        o.gemm(s.p1n, st.W("pooled_y_emb_process.fc2.weight"), s.c, epi=EPI_RESID, res=s.temb,
               bias=P["pooled_y_emb_process.fc2.bias"])
        # every adaLN_modulation (GELU-tanh -> Linear; dit.py:227-235, utils.py:231-237) as ONE GEMM
        s.cact = o.empty((B, D), BF16)
        o.gelu_tanh_f32_fwd(s.c, s.cact)
        s.mod = o.empty((B, st.layout.ada_rows), F32)
        o.gemm(s.cact, st.W("ada"), s.mod, epi=EPI_F32, bias=st.ada_bias)
        return s

    def _stem_bwd(self, s, dmod, dy2, B, want_dt=True, want_dy=True):
        """dmod f32 [B, ada_rows] (filled by the blocks), dy2 f32 [B*L, D] grad wrt the caption tokens.  Returns the bf16
        gradients at the pre-activations of t_embedder.mlp.0 and y_embedder.y_proj.fc1 (the input-gradient exits of
        backward_output).  While weight gradients are skipped, the timestep branch runs only for want_dt and the caption
        branch only for want_dy."""
        o, st, cfg = self.ops, self.store, self.cfg
        P = st.p
        D, hd, L = cfg.dim, cfg.head_dim, s.L
        R = B * L
        H = D // hd
        # ---- adaLN stack
        dmod_bf = o.empty(tuple(dmod.shape), BF16)
        o.cast_bf16(dmod, dmod_bf)
        self._wgrad(dmod_bf, s.cact, self._Gv("ada"))
        self._colsum(dmod, None if self._skip_wgrad else st.g_ada_bias)
        dcact = o.zeros((B, D), F32)  # K = sum(6D) ~ 2e5 with only a handful of output tiles: split the reduction
        o.gemm(dmod_bf, st.WT("ada"), dcact, epi=EPI_ATOMIC, splits=0)
        dc = o.empty((B, D), F32)
        o.gelu_tanh_f32_bwd(dcact, s.c, dc, False)
        dc_bf = o.empty((B, D), BF16)
        o.cast_bf16(dc, dc_bf)
        # ---- timestep embedder (c = temb + pooled: dc flows to both)
        self._colsum(dc, self._gv("t_embedder.mlp.2.bias"))
        self._wgrad(dc_bf, s.t1, self._Gv("t_embedder.mlp.2.weight"))
        dt1pre = None
        if want_dt or not self._skip_wgrad:
            dt1 = o.empty((B, D), BF16)
            o.gemm(dc_bf, st.WT("t_embedder.mlp.2.weight"), dt1)
            dt1pre = o.empty((B, D), BF16)
            o.act_bwd(dt1, s.t1pre, dt1pre, ACT_TANH)
            self._colsum(dt1pre, self._gv("t_embedder.mlp.0.bias"))
            self._wgrad(dt1pre, s.tfreq, self._Gv("t_embedder.mlp.0.weight"))
        if not (want_dy or not self._skip_wgrad):
            return dt1pre, None
        # ---- pooled caption Mlp
        self._colsum(dc, self._gv("pooled_y_emb_process.fc2.bias"))
        self._wgrad(dc_bf, s.p1n, self._Gv("pooled_y_emb_process.fc2.weight"))
        dp1n = o.empty((B, D), BF16)
        o.gemm(dc_bf, st.WT("pooled_y_emb_process.fc2.weight"), dp1n)
        dp1 = o.empty((B, D), BF16)
        o.ln_bwd(dp1n, s.p1, s.m_p, s.r_p, gamma=P["pooled_y_emb_process.norm.weight"], T=1, dx=dp1, dx_mode=1,
                 dgamma=self._gv("pooled_y_emb_process.norm.weight"))
        dp1pre = o.empty((B, D), BF16)
        o.act_bwd(dp1, s.p1pre, dp1pre, ACT_TANH)
        self._colsum(dp1pre, self._gv("pooled_y_emb_process.fc1.bias"))
        self._wgrad(dp1pre, s.pool, self._Gv("pooled_y_emb_process.fc1.weight"))
        dpool = o.empty((B, D), F32)
        o.gemm(dp1pre, st.WT("pooled_y_emb_process.fc1.weight"), dpool, epi=EPI_F32)
        o.mean_tokens_bwd(dpool, dy2, B, L)
        # ---- prompt block: SwiGLU
        fp = cfg.prompt_ffn_dim
        dyb = o.empty((R, D), BF16)
        o.gate_bwd(dy2, dyb, T=L)
        self._colsum(dy2, self._gb("y_emb_preprocess.mlp.w3.weight"))
        du = o.empty((R, 2 * fp), BF16)
        self._swiglu_bwd("y_emb_preprocess.mlp.w12", "y_emb_preprocess.mlp.w3.weight", dyb, s.u, du)
        self._wgrad(dyb, s.hact, self._Gv("y_emb_preprocess.mlp.w3.weight"))
        dyn = o.empty((R, D), BF16)
        o.gemm(du, st.WT("y_emb_preprocess.mlp.w12"), dyn)
        self._wgrad_w12("y_emb_preprocess.mlp.w12", du, s.yn2)
        o.ln_bwd(dyn, s.y1, s.m2, s.r2, gamma=P["y_emb_preprocess.norm2.weight"], T=L, dx=dy2, dx_mode=0,
                 dgamma=self._gv("y_emb_preprocess.norm2.weight"))
        # ---- prompt block: self attention
        o.gate_bwd(dy2, dyb, T=L)
        self._colsum(dy2, self._gb("y_emb_preprocess.attn.proj.weight"))
        datt = o.empty((R, D), BF16)
        o.gemm(dyb, st.WT("y_emb_preprocess.attn.proj.weight"), datt)
        self._wgrad(dyb, s.att, self._Gv("y_emb_preprocess.attn.proj.weight"))
        dqkv = o.empty((R, 3 * D), BF16); delta = o.empty((B, H, L), F32)
        o.attn_bwd(datt, s.qkv[:, :D], s.qkv[:, D:2 * D], s.qkv[:, 2 * D:], s.att, s.lse, delta, dqkv[:, :D],
                   dqkv[:, D:2 * D], dqkv[:, 2 * D:], B, H, L, L, hd)
        o.rownorm_bwd(dqkv[:, :2 * D], s.qkv[:, :2 * D], s.rqk, nslice=2)
        self._colsum(dqkv, self._gb("y_emb_preprocess.attn.qkv.weight"))
        o.gemm(dqkv, st.WT("y_emb_preprocess.attn.qkv.weight"), dyn)
        self._wgrad(dqkv, s.yn1, self._Gv("y_emb_preprocess.attn.qkv.weight"))
        o.ln_bwd(dyn, s.y0, s.m1, s.r1, gamma=P["y_emb_preprocess.norm1.weight"], T=L, dx=dy2, dx_mode=0,
                 dgamma=self._gv("y_emb_preprocess.norm1.weight"))
        # ---- caption projection
        o.gate_bwd(dy2, dyb, T=L)
        self._colsum(dy2, self._gv("y_embedder.y_proj.fc2.bias"))
        self._wgrad(dyb, s.a1n, self._Gv("y_embedder.y_proj.fc2.weight"))
        da1n = o.empty((R, D), BF16)
        o.gemm(dyb, st.WT("y_embedder.y_proj.fc2.weight"), da1n)
        da1 = o.empty((R, D), BF16)
        o.ln_bwd(da1n, s.a1, s.m_a, s.r_a, gamma=P["y_embedder.y_proj.norm.weight"], T=L, dx=da1, dx_mode=1,
                 dgamma=self._gv("y_embedder.y_proj.norm.weight"))
        da1pre = o.empty((R, D), BF16)
        o.act_bwd(da1, s.a1pre, da1pre, ACT_TANH)
        self._colsum(da1pre, self._gv("y_embedder.y_proj.fc1.bias"))
        self._wgrad(da1pre, s.ycap, self._Gv("y_embedder.y_proj.fc1.weight"))
        return dt1pre, da1pre

    # ================================================================== denoiser forward
    def prompt_cache(self, cap):
        """Sampler fast path (SURVEY.md §8 f-4): everything the denoiser derives from the caption alone -- the caption
        stem (dit.py:481-484), the mixer's caption map (dit.py:491) and the K/V projections of all 34 cross-attention
        layers with K already QK-normalised (utils.py:122-129) -- computed once per prompt batch instead of once per
        denoiser call (59 calls for a 30-step Heun run).  Inference only; tied to the current weights."""
        o, st, cfg = self.ops, self.store, self.cfg
        P = st.p
        token = self.weights_token() if self.weights_token is not None else None
        st.refresh_copies(o, token)
        B, D, Dm, eps = cap.shape[0], cfg.dim, cfg.mixer_dim, cfg.norm_eps
        pc = NS(B=B, token=token)
        s = self._caption_fwd(cap, None, B)
        L = s.L
        pc.s = s
        if cfg.use_patch_mixer:
            if cfg.has_mixer_maps:
                y_n = o.empty((B * L, D), BF16); m = o.empty((B * L,), F32); r = o.empty((B * L,), F32)
                o.ln_fwd(s.y2, y_n, m, r, gamma=P["patch_mixer_map_y.0.weight"], T=L, eps=eps)
                pc.ymix = o.empty((B * L, Dm), BF16)
                o.gemm(y_n, st.W("patch_mixer_map_y.1.weight"), pc.ymix, **self._bkw("patch_mixer_map_y.1.weight"))
            else:
                pc.ymix = s.ybf
            pc.kv_m = self._kv_fwd("kv.patch_mixer", pc.ymix, len(cfg.mixer_blocks), 2 * Dm)
            rk = o.empty((B * L,), F32)
            for i in range(len(cfg.mixer_blocks)):
                o.rownorm_fwd(pc.kv_m[:, i * 2 * Dm:i * 2 * Dm + Dm], rk, eps)
        pc.kv_b = self._kv_fwd("kv.blocks", s.ybf, len(cfg.blocks), 2 * D)
        rk = o.empty((B * L,), F32)
        for i in range(len(cfg.blocks)):
            o.rownorm_fwd(pc.kv_b[:, i * 2 * D:i * 2 * D + D], rk, eps)
        return pc

    def _denoiser_fwd(self, lat, eps_noise, rnd, sigma_in, cap, drop, mask_ratio, mask_noise, edm, keep: bool,
                      raw_t=None, cap_out=None, prompt=None):
        o, st, cfg = self.ops, self.store, self.cfg
        P = st.p
        wtoken = self.weights_token() if self.weights_token is not None else None
        st.refresh_copies(o, wtoken, part="front")
        B, C, Hh, Ww = lat.shape
        p, D, Dm = cfg.patch_size, cfg.dim, cfg.mixer_dim
        T = (Hh // p) * (Ww // p)
        assert T == cfg.num_patches and C == cfg.in_channels, "input does not match the model's latent shape"
        c = NS(B=B, T=T, mask_ratio=mask_ratio, lat=lat, raw_t=raw_t)
        # ---- noise + preconditioning + im2col (model.py:182-188, 153-166)
        c.patches = o.empty((B * T, cfg.patch_dim), BF16)
        if raw_t is None:
            c.xn = o.empty((B, C, Hh, Ww), F32)
            c.coef = o.empty((6, B), F32)
            o.edm_prepare(lat, eps_noise, rnd, sigma_in, edm["P_mean"], edm["P_std"], edm["sigma_data"], c.xn,
                          c.patches, c.coef, p)
            cnoise = c.coef[4]
        else:  # plain DiT.forward(x, t, y): x is already preconditioned, t is the network's time input
            c.xn = c.coef = None
            o.patchify(lat, None, c.patches, p)
            cnoise = raw_t
        # ---- patch embed + positional table (dit.py:479)
        x0 = o.empty((B * T, D), F32)
        o.gemm(c.patches, st.W("x_embedder.proj.weight"), x0, epi=EPI_RESID, res=self.pos_embed.reshape(T, D),
               res_mod=T, bias=P["x_embedder.proj.bias"])
        # ---- conditioning
        if prompt is not None:
            assert not keep and prompt.B == B, "a PromptCache serves inference calls of the batch it was built for"
            if self.weights_token is not None and prompt.token != self.weights_token():
                raise RuntimeError("PromptCache is stale: the weights changed since it was built")
            s = self._time_fwd(NS(**vars(prompt.s)), cnoise, B)
        else:
            s = self._stem_fwd(cap, drop, cnoise, B, keep, cap_out)
        kvn = prompt is not None
        c.stem = s
        L = s.L
        mod = s.mod
        # ---- patch mixer on all T tokens (dit.py:489-493)
        c.mixer_sv = []
        if cfg.use_patch_mixer:
            if cfg.has_mixer_maps:
                c.xin_n = o.empty((B * T, D), BF16); c.m_xin = o.empty((B * T,), F32); c.r_xin = o.empty((B * T,), F32)
                o.ln_fwd(x0, c.xin_n, c.m_xin, c.r_xin, gamma=P["patch_mixer_map_xin.0.weight"], T=T, eps=cfg.norm_eps)
                xm = o.empty((B * T, Dm), F32)
                o.gemm(c.xin_n, st.W("patch_mixer_map_xin.1.weight"), xm, epi=EPI_F32, **self._bkw("patch_mixer_map_xin.1.weight"))
                if prompt is None:
                    c.y_n = o.empty((B * L, D), BF16); c.m_y = o.empty((B * L,), F32); c.r_y = o.empty((B * L,), F32)
                    o.ln_fwd(s.y2, c.y_n, c.m_y, c.r_y, gamma=P["patch_mixer_map_y.0.weight"], T=L, eps=cfg.norm_eps)
                    c.ymix = o.empty((B * L, Dm), BF16)
                    o.gemm(c.y_n, st.W("patch_mixer_map_y.1.weight"), c.ymix, **self._bkw("patch_mixer_map_y.1.weight"))
            else:
                xm, c.ymix = x0, s.ybf
            c.x0 = x0
            pend = None
            D2m = 2 * Dm
            kv_m = prompt.kv_m if kvn else self._kv_fwd("kv.patch_mixer", c.ymix, len(cfg.mixer_blocks), D2m)
            for i, bs in enumerate(cfg.mixer_blocks):
                xm, pend, sv = self._block_fwd(bs, xm, pend, kv_m[:, i * D2m:(i + 1) * D2m], B, T, L, mod, keep, kvn)
                c.mixer_sv.append(sv)
        else:
            xm, pend = x0, None
        # ---- random patch masking (dit.py:495-504, utils.py:382-414)
        if mask_ratio > 0:
            Tk = int(T * (1 - mask_ratio))
            c.ids_restore = o.empty((B, T), I32); c.mask = o.empty((B, T), F32); c.keep_rows = o.empty((B * Tk,), I32)
            o.mask_sort(mask_noise, None, c.ids_restore, c.mask, c.keep_rows, Tk)
        else:
            Tk = T
            c.ids_restore = c.mask = c.keep_rows = None
        c.Tk = Tk
        if cfg.has_mixer_maps:  # LN + Linear back to the backbone width, applied after masking (dit.py:506-508)
            c.xk_n = o.empty((B * Tk, Dm), BF16); c.m_xo = o.empty((B * Tk,), F32); c.r_xo = o.empty((B * Tk,), F32)
            c.xm_out = self._ln_add(xm, pend, c.xk_n, c.m_xo, c.r_xo, gamma=P["patch_mixer_map_xout.0.weight"], T=Tk,
                                    src_rows=c.keep_rows)
            xb = o.empty((B * Tk, D), F32)
            o.gemm(c.xk_n, st.W("patch_mixer_map_xout.1.weight"), xb, epi=EPI_F32,
                   **self._bkw("patch_mixer_map_xout.1.weight"))
            pend = None
        elif mask_ratio > 0:
            xm = self._materialize(xm, pend, T)
            xb = o.empty((B * Tk, xm.shape[1]), F32)
            o.gather_rows(xm, c.keep_rows, xb)
            pend = None
        else:
            xb = xm
        # ---- backbone (dit.py:510-511)
        st.refresh_copies(o, wtoken, part="back")
        c.block_sv = []
        kv_b = prompt.kv_b if kvn else self._kv_fwd("kv.blocks", s.ybf, len(cfg.blocks), 2 * D)
        for i, bs in enumerate(cfg.blocks):
            xb, pend, sv = self._block_fwd(bs, xb, pend, kv_b[:, i * 2 * D:(i + 1) * 2 * D], B, Tk, L, mod, keep, kvn)
            c.block_sv.append(sv)
        # ---- final layer (utils.py:236-240)
        fo = st.layout.ada_offset["final_layer"]
        sh_f, sc_f = mod[:, fo:fo + D], mod[:, fo + D:fo + 2 * D]
        c.xf = o.empty((B * Tk, D), BF16); c.m_f = o.empty((B * Tk,), F32); c.r_f = o.empty((B * Tk,), F32)
        c.xlast = self._ln_add(xb, pend, c.xf, c.m_f, c.r_f, gamma=P["final_layer.norm_final.weight"], shift=sh_f,
                               scale=sc_f, T=Tk)
        c.ftok = o.empty((B * Tk, cfg.patch_dim), F32)
        o.gemm(c.xf, st.W("final_layer.linear.weight"), c.ftok, epi=EPI_F32, bias=P["final_layer.linear.bias"])
        return c

    # ================================================================== public entry points
    def forward_loss(self, lat, cap, drop, rnd, eps_noise, mask_ratio, mask_noise, edm, keep=True, cap_out=None):
        """edm_loss (model.py:181-210).  Returns a context holding `loss` (f32 [1]) and `per_sample`."""
        o = self.ops
        c = self._denoiser_fwd(lat, eps_noise, rnd, None, cap, drop, mask_ratio, mask_noise, edm, keep, cap_out=cap_out)
        B = c.B
        c.per_sample = o.empty((B,), F32)
        c.loss = o.zeros((1,), F32)
        o.edm_loss_fwd(c.ftok, c.keep_rows, lat, c.xn, c.coef, c.per_sample, c.loss, self.cfg.patch_size, c.Tk)
        return c

    def denoise(self, x_noisy, sigma, cap, mask_ratio=0.0, mask_noise=None, edm=None, want_raw=False, prompt=None):
        """model_forward_wrapper (model.py:144-179) without gradients: D_x (and optionally F_x, mask).
        `prompt` = prompt_cache(cap) skips the caption-only work."""
        o = self.ops
        zero = o.zeros(tuple(x_noisy.shape), F32)
        c = self._denoiser_fwd(x_noisy, zero, None, sigma, cap, None, mask_ratio, mask_noise, edm, keep=False,
                               prompt=prompt)
        B, C, Hh, Ww = x_noisy.shape
        dx = o.empty((B, C, Hh, Ww), F32)
        fx = o.empty((B, C, Hh, Ww), F32) if want_raw else None
        o.edm_output(c.ftok, c.ids_restore, self.mask_token.reshape(-1), c.xn, c.coef, fx, dx, self.cfg.patch_size, c.Tk)
        return dx, fx, c.mask

    def denoise_cfg(self, x2, sigma2, cfg, edm, prompt):
        """model_forward_wrapper's guided branch (model.py:188-202) without gradients: the denoiser on the doubled batch
        x2 = [x; x] with the prompt cache of [caption; zeros], then guidance and preconditioning in one kernel.  cfg: f32 [1]
        on the device.  Returns D f32 [B,C,H,W]."""
        o = self.ops
        c = self._denoiser_fwd(x2, o.zeros(tuple(x2.shape), F32), None, sigma2, None, None, 0.0, None, edm, keep=False,
                               prompt=prompt)
        B = x2.shape[0] // 2
        dx = o.empty((B, *x2.shape[1:]), F32)
        o.edm_output_cfg(c.ftok, x2[:B], sigma2, cfg, dx, edm["sigma_data"], self.cfg.patch_size)
        return dx

    def sampler(self, B, guided, shape, cap_shape):
        """The SamplerGraph of one (batch, CFG or not, latent shape, caption shape) in the current precision and
        deterministic mode, captured on first use and kept until release_sampler_graphs() or a rebind of the weights."""
        key = (B, bool(guided), tuple(shape), tuple(cap_shape), self.ops.prec, self.ops._det_ws is not None)
        g = self._sampler_graphs.get(key)
        if g is None:
            g = self._sampler_graphs[key] = SamplerGraph(self, B, guided, shape, cap_shape)
        return g

    def release_sampler_graphs(self):
        """Drop every captured sampler graph and the memory pool they hold."""
        self._sampler_graphs.clear()

    def forward_raw(self, x, t, cap, mask_ratio=0.0, mask_noise=None, keep=False):
        """DiT.forward_without_cfg (dit.py:455-519): (F_x, mask).  keep=True saves the activations and returns
        (F_x, mask, ctx) for backward_output(ctx, ...)."""
        o = self.ops
        c = self._denoiser_fwd(x, None, None, None, cap, None, mask_ratio, mask_noise, None, keep=keep, raw_t=t)
        B, C, Hh, Ww = x.shape
        fx = o.empty((B, C, Hh, Ww), F32)
        o.edm_output(c.ftok, c.ids_restore, self.mask_token.reshape(-1), None, None, fx, None, self.cfg.patch_size, c.Tk)
        return (fx, c.mask, c) if keep else (fx, c.mask)

    def backward(self, c, gscale):
        """Accumulate d(loss * gscale) / d(parameters) into the flat gradient buffer."""
        o, cfg = self.ops, self.cfg
        dmod, dy2 = self._bwd_accumulators(c)
        # ---- loss -> final layer
        dftok = o.empty((c.B * c.Tk, cfg.patch_dim), BF16)
        o.edm_loss_bwd(c.ftok, c.keep_rows, c.lat, c.xn, c.coef, gscale, dftok, cfg.patch_size, c.Tk)
        self._backward_from_tokens(c, dftok, dmod, dy2)

    def backward_output(self, c, dF, *, param_grads: bool, want_dx: bool, want_dt: bool, want_dy: bool):
        """Vector-Jacobian product of forward_raw(..., keep=True) for the cotangent dF (f32 [B,C,H,W]) of F_x.

        param_grads=True accumulates d<F_x, dF>/d(parameters) into the flat gradient buffer like backward();
        param_grads=False (every DiT parameter frozen) skips all weight gradients and writes nothing there.
        Returns (dx f32 [B,C,H,W], dt f32 [B], dy f32 [B*L, caption_channels]), None where not wanted: the
        gradients wrt forward_raw's x, t and (the bf16 storage of) the caption."""
        o, st, cfg = self.ops, self.store, self.cfg
        B, T, Tk, p = c.B, c.T, c.Tk, cfg.patch_size
        dmod, dy2 = self._bwd_accumulators(c)
        dftok = o.empty((B * Tk, cfg.patch_dim), BF16)
        o.unpatchify_bwd(dF, c.keep_rows, dftok, p, Tk)
        self._skip_wgrad = not param_grads
        try:
            dx0b, dt1pre, da1pre = self._backward_from_tokens(c, dftok, dmod, dy2, grads_ready_hook=False,
                                                              want_dx0=want_dx, want_dt=want_dt, want_dy=want_dy)
        finally:
            self._skip_wgrad = False
        dx = dt = dy = None
        if want_dx:  # patch-embed dgrad (N = C*p*p) + col2im
            dpatches = o.empty((B * T, cfg.patch_dim), F32)
            o.gemm(dx0b, self._transposed("x_embedder.proj.weight"), dpatches, epi=EPI_F32)
            dx = o.empty(tuple(c.lat.shape), F32)
            o.patchify_bwd(dpatches, None, dx, p)
        if want_dt:  # t_embedder.mlp.0 dgrad + the sinusoid's adjoint
            dfreq = o.empty((B, cfg.freq_dim), F32)
            o.gemm(dt1pre, st.WT("t_embedder.mlp.0.weight"), dfreq, epi=EPI_F32)
            dt = o.empty((B,), F32)
            o.timestep_embed_bwd(dfreq, c.raw_t, dt)
        if want_dy:  # y_embedder.y_proj.fc1 dgrad
            wt = self._transposed("y_embedder.y_proj.fc1.weight")
            dy = o.empty((da1pre.shape[0], wt.shape[0]), F32)
            o.gemm(da1pre, wt, dy, epi=EPI_F32)
        return dx, dt, dy

    def _bwd_accumulators(self, c):
        """dmod (grad wrt every adaLN vector) and dy2 (grad wrt the caption tokens: all cross-attentions + pooled path)."""
        o = self.ops
        return o.zeros(tuple(c.stem.mod.shape), F32), o.zeros((c.B * c.stem.L, self.cfg.dim), F32)

    def _backward_from_tokens(self, c, dftok, dmod, dy2, grads_ready_hook=True, want_dx0=False, want_dt=False,
                              want_dy=False):
        """The backward shared by backward() and backward_output(), from d ftok (bf16 [B*Tk, p*p*C], the final-layer token
        gradient) down to every parameter and the conditioning stem.  Returns (dx0b, dt1pre, da1pre): the bf16 gradients
        at the patch-embed output, the timestep MLP's and the caption projection's pre-activations (None when not
        computed; want_* only matter while weight gradients are skipped)."""
        o, st, cfg = self.ops, self.store, self.cfg
        P = st.p
        B, T, Tk = c.B, c.T, c.Tk
        D, Dm = cfg.dim, cfg.mixer_dim
        s = c.stem
        L = s.L
        mod = s.mod
        self._colsum(dftok, self._gv("final_layer.linear.bias"))
        self._wgrad(dftok, c.xf, self._Gv("final_layer.linear.weight"))
        dxf = o.empty((B * Tk, D), BF16)
        o.gemm(dftok, st.WT("final_layer.linear.weight"), dxf)
        fo = st.layout.ada_offset["final_layer"]
        sc_f = mod[:, fo + D:fo + 2 * D]
        dx = o.zeros((B * Tk, D), F32)
        nb = len(cfg.blocks)
        fuse = self.fuse_ln and nb > 0 and cfg.blocks[-1].dim == D
        dy = o.empty((B * Tk, D), BF16) if fuse else None
        o.ln_bwd(dxf, c.xlast, c.m_f, c.r_f, gamma=P["final_layer.norm_final.weight"], scale=sc_f, T=Tk, dx=dx,
                 dx_mode=0, dgamma=self._gv("final_layer.norm_final.weight"), dshift=dmod[:, fo:fo + D],
                 dscale=dmod[:, fo + D:fo + 2 * D], dy_next=dy,
                 **(self._ffn_gate_args(cfg.blocks[-1], c.block_sv[-1], mod, dmod) if fuse else {}))
        # ---- backbone
        dkv_b = o.empty((B * L, nb * 2 * D), BF16)
        for i in range(nb - 1, -1, -1):
            nxt = self._ffn_gate_args(cfg.blocks[i - 1], c.block_sv[i - 1], mod, dmod) if i > 0 else None
            dy = self._block_bwd(cfg.blocks[i], c.block_sv[i], dx, dkv_b[:, i * 2 * D:(i + 1) * 2 * D], B, Tk, L, mod, dmod,
                                 dy_in=dy, nxt=nxt)
            c.block_sv[i] = None  # release this block's saved activations
        self._kv_bwd("kv.blocks", dkv_b, s.ybf, dy2)
        del dkv_b
        if grads_ready_hook and self.on_backbone_grads_ready is not None:
            # every gradient of blocks.* / final_layer.* / the stacked kv.blocks is final from here on: the
            # data-parallel reducer can start moving ~3/4 of the bytes while the mixer and stem backward still run
            self.on_backbone_grads_ready()
        # ---- un-mask / mixer-out map
        if cfg.has_mixer_maps:
            dxb = o.empty((B * Tk, D), BF16)
            o.gate_bwd(dx, dxb, T=Tk)
            self._colsum(dx, self._gb("patch_mixer_map_xout.1.weight"))
            self._wgrad(dxb, c.xk_n, self._Gv("patch_mixer_map_xout.1.weight"))
            dxk = o.empty((B * Tk, Dm), BF16)
            o.gemm(dxb, st.WT("patch_mixer_map_xout.1.weight"), dxk)
            dxm = o.zeros((B * T, Dm), F32)
            o.ln_bwd(dxk, c.xm_out, c.m_xo, c.r_xo, gamma=P["patch_mixer_map_xout.0.weight"], T=Tk,
                     src_rows=c.keep_rows, dx=dxm, dx_mode=2 if c.keep_rows is not None else 0,
                     dgamma=self._gv("patch_mixer_map_xout.0.weight"))
        elif c.keep_rows is not None:
            dxm = o.zeros((B * T, dx.shape[1]), F32)
            o.scatter_rows(dx, c.keep_rows, dxm)
        else:
            dxm = dx
        # ---- patch mixer
        if cfg.use_patch_mixer:
            dymix = o.zeros((B * L, Dm), F32) if cfg.has_mixer_maps else dy2
            nm = len(cfg.mixer_blocks)
            dkv_m = o.empty((B * L, nm * 2 * Dm), BF16)
            dy = None
            for i in range(nm - 1, -1, -1):
                nxt = self._ffn_gate_args(cfg.mixer_blocks[i - 1], c.mixer_sv[i - 1], mod, dmod) if i > 0 else None
                dy = self._block_bwd(cfg.mixer_blocks[i], c.mixer_sv[i], dxm, dkv_m[:, i * 2 * Dm:(i + 1) * 2 * Dm], B, T, L,
                                     mod, dmod, dy_in=dy, nxt=nxt)
                c.mixer_sv[i] = None
            self._kv_bwd("kv.patch_mixer", dkv_m, c.ymix, dymix)
            del dkv_m
            if cfg.has_mixer_maps:
                # caption map: y_mixer = Linear(LN(y))
                dymb = o.empty((B * L, Dm), BF16)
                o.gate_bwd(dymix, dymb, T=L)
                self._colsum(dymix, self._gb("patch_mixer_map_y.1.weight"))
                self._wgrad(dymb, c.y_n, self._Gv("patch_mixer_map_y.1.weight"))
                dyn = o.empty((B * L, D), BF16)
                o.gemm(dymb, st.WT("patch_mixer_map_y.1.weight"), dyn)
                o.ln_bwd(dyn, s.y2, c.m_y, c.r_y, gamma=P["patch_mixer_map_y.0.weight"], T=L, dx=dy2, dx_mode=0,
                         dgamma=self._gv("patch_mixer_map_y.0.weight"))
                # token map: x_mixer = Linear(LN(x0))
                dxmb = o.empty((B * T, Dm), BF16)
                o.gate_bwd(dxm, dxmb, T=T)
                self._colsum(dxm, self._gb("patch_mixer_map_xin.1.weight"))
                self._wgrad(dxmb, c.xin_n, self._Gv("patch_mixer_map_xin.1.weight"))
                dxn = o.empty((B * T, D), BF16)
                o.gemm(dxmb, st.WT("patch_mixer_map_xin.1.weight"), dxn)
                dx0 = o.zeros((B * T, D), F32)
                o.ln_bwd(dxn, c.x0, c.m_xin, c.r_xin, gamma=P["patch_mixer_map_xin.0.weight"], T=T, dx=dx0, dx_mode=0,
                         dgamma=self._gv("patch_mixer_map_xin.0.weight"))
            else:
                dx0 = dxm
        else:
            dx0 = dxm
        # ---- patch embed
        dx0b = None
        if want_dx0 or not self._skip_wgrad:
            dx0b = o.empty(tuple(dx0.shape), BF16)
            o.gate_bwd(dx0, dx0b, T=T)
        self._colsum(dx0, self._gv("x_embedder.proj.bias"))
        self._wgrad(dx0b, c.patches, self._Gv("x_embedder.proj.weight"))
        # ---- conditioning stem
        if want_dt or want_dy or not self._skip_wgrad:
            return (dx0b, *self._stem_bwd(s, dmod, dy2, B, want_dt, want_dy))
        return dx0b, None, None

    # buffers owned by the nn.Module (pos_embed / mask_token), attached by models.dit.DiT
    pos_embed: Optional[torch.Tensor] = None
    weights_token = None  # callable -> hashable; set by models.dit.DiT
    on_backbone_grads_ready = None  # optional callable, see backward()
    mask_token: Optional[torch.Tensor] = None


class SamplerGraph:
    """The Heun sampler of LatentDiffusion._heun as replays of captured CUDA graphs.

    Three graphs share one memory pool: the prompt cache of the caption (Engine.prompt_cache), one full Heun step
    (stage in -> denoiser -> euler -> denoiser -> correct -> step + 1) and the last step (stage in -> denoiser -> euler ->
    step + 1).  Every per-step value lives in device memory -- the schedule table, the step index, the pre-drawn noise,
    the guidance scale -- so a run is a fixed sequence of replays with no host decision and no host sync in between.
    Static buffers: the fp64 state x / x_hat / d_cur, the fp32 denoiser input and sigma (doubled for CFG), the caption
    (with the zero half for CFG), the table, the step index and the noise of `max_steps` steps (grown, with a recapture,
    when a run asks for more)."""

    def __init__(self, eng, B, guided, shape, cap_shape):
        dev = eng.ops.device
        f64 = torch.float64
        self.eng, self.B, self.guided = eng, B, bool(guided)
        B2 = 2 * B if guided else B
        self.x = torch.zeros((B, *shape), dtype=f64, device=dev)
        self.x_hat = torch.zeros_like(self.x)
        self.d_cur = torch.zeros_like(self.x)
        self.xin = torch.zeros((B2, *shape), dtype=F32, device=dev)
        self.sigma = torch.ones((B2,), dtype=F32, device=dev)
        self.cap = torch.zeros((B2, *cap_shape), dtype=torch.float16, device=dev)
        self.cfg = torch.ones((1,), dtype=F32, device=dev)
        self.step = torch.zeros((1,), dtype=torch.int32, device=dev)
        self.max_steps = 0
        self.table = self.noise = None  # device table and noise, sized for max_steps
        self.graphs = None
        self.den = {}       # graph name -> the denoiser outputs D of its calls (static addresses in the pool)
        self.captures = 0   # number of captures so far (a replay of an unchanged setting does not recapture)
        self.runs = 0       # sampler runs served
        self.pool = None

    def _stage(self, stage, den=None):
        o = self.eng.ops
        o.edm_heun(stage, self.x, self.x_hat, self.d_cur, den, self.noise if stage == o.HEUN_IN else None,
                   None if stage == o.HEUN_CORRECT else self.xin, self.sigma, self.table, self.step, self.s_noise)

    def _denoise(self):
        eng, edm = self.eng, self.edm
        if self.guided:
            return eng.denoise_cfg(self.xin, self.sigma, self.cfg, edm, self.pc)
        return eng.denoise(self.xin, self.sigma, None, 0.0, None, edm, prompt=self.pc)[0]

    def _body(self, name):
        """What one graph holds; the same launches run eagerly for the warm-up."""
        o = self.eng.ops
        if name == "prompt":
            self.pc = self.eng.prompt_cache(self.cap)
            return
        self._stage(o.HEUN_IN)
        dens = [self._denoise()]
        self._stage(o.HEUN_EULER, dens[0])
        if name == "step":
            dens.append(self._denoise())
            self._stage(o.HEUN_CORRECT, dens[1])
        o.edm_heun(o.HEUN_NEXT, None, None, None, None, None, None, None, None, self.step, 1.0)
        self.den[name] = dens

    def _capture(self):
        # warm-up: every launch once outside capture (tensor-map cache, cudaFuncSetAttribute, lazy module loads), on the
        # run's own inputs; the caller re-writes the state before replaying
        for name in ("prompt", "step", "last"):
            self.step.zero_()
            self._body(name)
        self.pool = torch.cuda.graph_pool_handle()
        self.graphs = {}
        for name in ("prompt", "step", "last"):
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, pool=self.pool):
                self._body(name)
            self.graphs[name] = g
        self.captures += 1

    def run(self, x0, t_steps, t_hat, noise, cap, cfg, s_noise, edm, debug=None):
        """x0 f64 [B,C,H,W] = x * t_steps[0]; t_steps / t_hat: host f64 (n+1 / n values); noise: the n draws of the eager
        loop; cap: fp16 caption [B, ...].  Returns the final state in fp32, like _heun.  `debug(k, call, D)` (optional) sees
        the denoiser output of every call after the replay that made it."""
        eng, o = self.eng, self.eng.ops
        n = len(t_hat)
        token = eng.weights_token() if eng.weights_token is not None else None
        eng.store.refresh_copies(o, token)  # weights updated since the capture: new bf16 copies, outside the graphs
        if n > self.max_steps or s_noise != getattr(self, "s_noise", s_noise) or edm != getattr(self, "edm", edm):
            self.graphs, self.den, self.pc = None, {}, None
            if n > self.max_steps:
                self.max_steps = n
                self.table = torch.zeros(2 * n + 1, dtype=torch.float64, device=o.device)
                self.noise = torch.zeros((n, *self.x.shape), dtype=torch.float64, device=o.device)
        self.s_noise, self.edm = s_noise, dict(edm)
        self.table.copy_(SamplerGraph.schedule_table(t_steps, t_hat, self.max_steps))
        for k, nk in enumerate(noise):
            self.noise[k].copy_(nk)
        B = self.B
        self.cap[:B].copy_(cap)
        if self.guided:
            self.cap[B:].zero_()
            self.cfg.fill_(cfg)
        if self.graphs is None:
            self.x.copy_(x0)
            self._capture()
        self.x.copy_(x0)
        self.step.zero_()
        self._replay(n, debug)
        self.runs += 1
        return self.x.to(torch.float32)

    def _replay(self, n, debug):
        """The run itself: graph replays only, nothing that waits for the device."""
        g = self.graphs
        g["prompt"].replay()
        for k in range(n):
            name = "last" if k == n - 1 else "step"
            g[name].replay()
            if debug is not None:
                for j, d in enumerate(self.den[name]):
                    debug(k, j, d)

    @staticmethod
    def schedule_table(t_steps, t_hat, max_steps):
        """The schedule table md_edm_heun reads (host f64 [2*max_steps+1]): t_steps (n+1 values, the last one 0) at
        [0, n], t_hat (n values) at [max_steps+1, max_steps+1+n), zeros elsewhere."""
        n = len(t_hat)
        tab = torch.zeros(2 * max_steps + 1, dtype=torch.float64)
        tab[:n + 1] = t_steps
        tab[max_steps + 1:max_steps + 1 + n] = t_hat
        return tab
