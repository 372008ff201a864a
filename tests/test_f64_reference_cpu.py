"""The float64 references (tests/f64_reference.py) against the CPU contracts without a GPU: every reference on the same
seeded inputs as oracle.emu_ops.EmuOps(exact=True) -- and, for the ops EmuOps does not implement, the test-side
emulations of tests/dit_vjp_common.py and tests/bias_common.py -- at fp32-reassociation tolerance.  Two statements of
one contract written independently: if they disagree, one of them is wrong.  The three adjoint maps are also checked as
adjoints of the forward references (<J v, w> == <v, J^T w> in float64), and the closed-form derivatives against
autograd."""
import math

import pytest
import torch

from oracle.emu_ops import EmuOps
from tests import f64_reference as R
from tests.bias_common import BiasEmuOps
from tests.test_kernels_gpu import F32, I32, close, g, rnd

EMU = EmuOps("cpu", exact=True)
D64 = torch.float64


def agree(emu, ref, what, rtol=2e-6):
    """fp32 restatement vs float64 restatement: relative L2 <= rtol and per element 4 fp32 ulps of max(|ref|, rms)
    scaled for reassociation (close() of tests/test_kernels_gpu.py with its fp32 floor of 2^-16)."""
    close(emu.float(), ref.float(), what, rtol)


def _routing(B, T, E, k, seed):
    """probs of a random router and the top-k slot tables of EmuOps.moe_topk: (probs, idx, gval, inv)."""
    probs = torch.softmax(rnd((B * T, E), seed), -1)
    idx = torch.zeros(B, E, k, dtype=I32); gval = torch.zeros(B, E, k); inv = torch.zeros(B, T, E, dtype=I32)
    EMU.moe_topk(probs, idx, gval, inv, B, T, E, k)
    return probs, idx, gval, inv


# ------------------------------------------------------------------------------------------------ GEMM
@pytest.mark.parametrize("layout,batch", [(0, 1), (1, 1), (0, 3), (1, 3)])
def test_gemm_epilogues(layout, batch):
    M, N, K = 70, 48, 40
    A = rnd((batch, M, K) if layout == 0 else (batch, K, M), 1)
    B = rnd((batch, N, K) if layout == 0 else (batch, K, N), 2)
    if batch == 1:
        A, B = A[0], B[0]
    shp = (batch, M, N) if batch > 1 else (M, N)
    bias = rnd((N,), 3)
    C = torch.zeros(shp); EMU.gemm(A, B, C, layout=layout, epi=1, bias=bias, alpha=0.5)
    agree(C, R.gemm(A, B, layout, alpha=0.5, bias=bias), "gemm f32 + bias")
    acc = rnd(shp, 4); C = acc.clone(); EMU.gemm(A, B, C, layout=layout, epi=3, splits=4)
    agree(C, R.gemm(A, B, layout, accumulate=acc), "gemm accumulate")
    T = 10
    res = rnd((T, N), 5); gate = rnd((M // T, 2 * N), 6)
    C = torch.zeros(shp); EMU.gemm(A, B, C, layout=layout, epi=2, bias=bias, res=res, res_mod=T, gate=gate[:, N:],
                                   rows_per_gate=T)
    agree(C, R.gemm(A, B, layout, bias=bias, res=res, res_mod=T, gate=gate[:, N:], rows_per_gate=T), "gemm resid")
    if layout == 0:
        for act in (0, 1):
            pre, out = torch.zeros(shp), torch.zeros(shp)
            EMU.gemm(A, B, pre, epi=4, C2=out, bias=bias, act=act, alpha=0.05)
            rp, ro = R.gemm(A, B, alpha=0.05, bias=bias, act=act)
            agree(pre, rp, "act dual pre"); agree(out, ro, "act dual out")
            aux = rnd(shp, 7, scale=1.5); dp = torch.zeros(shp)
            EMU.gemm(A, B, dp, epi=5, aux=aux, act=act, alpha=0.05)
            agree(dp, R.gemm(A, B, alpha=0.05, aux=aux, act=act), "act grad")


def test_gemm_row_interleave():
    f, K, N = 96, 50, 40
    du = rnd((K, 2 * f), 1); x = rnd((K, N), 2); base = rnd((2 * f, N), 3)
    C = base.clone(); EMU.gemm(du, x, C, layout=1, epi=3, splits=0, row_interleave=f)
    ref = base.double().clone()
    ref.index_add_(0, R.interleaved_to_natural(f), R.matmul(du, x, 1))
    agree(C, ref, "interleaved wgrad")


@pytest.mark.parametrize("act", [0, 1])
def test_gelu_closed_form_derivative_is_autograd(act):
    x = rnd((4096,), 1, scale=3.0).double()
    dg = R._grads(lambda v: R.gelu(v, act), [x], torch.ones_like(x))[0]
    assert torch.allclose(R.gelu_grad(x, act), dg, rtol=1e-12, atol=1e-12)
    # and the forward is torch's own GELU
    ref = torch.nn.functional.gelu(x, approximate="tanh" if act else "none")
    assert torch.allclose(R.gelu(x, act), ref, rtol=1e-12, atol=1e-14)


# ------------------------------------------------------------------------------------------------ norms
@pytest.mark.parametrize("rows,D,T", [(128, 256, 64), (154, 192, 77)])
def test_layernorm(rows, D, T):
    ns = rows // T
    x = rnd((rows, D), 1, scale=2.0) + 0.5
    gamma = 1 + 0.1 * rnd((D,), 2); mod = rnd((ns, 6 * D), 3, scale=0.5)
    y = torch.zeros(rows, D); mean = torch.zeros(rows); rstd = torch.zeros(rows)
    EMU.ln_fwd(x, y, mean, rstd, gamma=gamma, shift=mod[:, D:2 * D], scale=mod[:, 3 * D:4 * D], T=T)
    ry, rmu, rrs, _ = R.ln_fwd(x, gamma=gamma, shift=mod[:, D:2 * D], scale=mod[:, 3 * D:4 * D], T=T)
    agree(y, ry, "ln y"); agree(mean, rmu, "mean"); agree(rstd, rrs, "rstd")
    # pending residual: x_new = x + gate * y_add normalised in the same pass
    ya = rnd((rows, D), 4); xn = torch.zeros(rows, D)
    EMU.ln_fwd(x, y, mean, rstd, gamma=gamma, shift=mod[:, D:2 * D], scale=mod[:, 3 * D:4 * D], T=T, y_add=ya,
               gate_add=mod[:, 2 * D:3 * D], x_new=xn)
    ry, rmu, rrs, rxn = R.ln_fwd(x, gamma=gamma, shift=mod[:, D:2 * D], scale=mod[:, 3 * D:4 * D], T=T, y_add=ya,
                                 gate_add=mod[:, 2 * D:3 * D])
    agree(xn, rxn, "x_new"); agree(xn, R.pending_residual(x, ya, mod[:, 2 * D:3 * D], T), "x_new (pending_residual)")
    agree(y, ry, "ln y after residual")
    # backward at the exact statistics of x, with the fused next-branch tail
    _, mu, rs, _ = R.ln_fwd(x, T=T)
    dy = rnd((rows, D), 5); dx0 = rnd((rows, D), 6); dmod = torch.zeros(ns, 6 * D); dg = torch.zeros(D)
    yn = rnd((rows, D), 7); dyn = torch.zeros(rows, D)
    dx = dx0.clone()
    EMU.ln_bwd(dy, x, mu.float(), rs.float(), gamma=gamma, scale=mod[:, 3 * D:4 * D], T=T, dx=dx, dgamma=dg,
               dshift=dmod[:, :D], dscale=dmod[:, 2 * D:3 * D], dy_next=dyn, y_next=yn, gate_next=mod[:, 5 * D:],
               dgate_next=dmod[:, 4 * D:5 * D])
    rdx, rdg, rdsh, rdsc = R.ln_bwd(dy, x, gamma=gamma, scale=mod[:, 3 * D:4 * D], T=T)
    agree(dx, dx0.double() + rdx, "ln dx"); agree(dg, rdg, "dgamma")
    agree(dmod[:, :D], rdsh, "dshift"); agree(dmod[:, 2 * D:3 * D], rdsc, "dscale")
    rdyn, rdgn = R.gate_bwd(dx0.double() + rdx, y=yn, gate=mod[:, 5 * D:], T=T)
    agree(dyn, rdyn, "dy_next"); agree(dmod[:, 4 * D:5 * D], rdgn, "dgate_next")


def test_layernorm_gather_scatter():
    rows_all, D, B, T, Tk = 64, 256, 2, 32, 8
    x = rnd((rows_all, D), 1)
    src = torch.stack([torch.randperm(T, generator=g(7))[:Tk] + b * T for b in range(B)]).reshape(-1).to(I32)
    gamma = 1 + 0.1 * rnd((D,), 2)
    rows = B * Tk
    y = torch.zeros(rows, D); mean = torch.zeros(rows); rstd = torch.zeros(rows)
    EMU.ln_fwd(x, y, mean, rstd, gamma=gamma, T=Tk, src_rows=src)
    ry, rmu, rrs, _ = R.ln_fwd(x, gamma=gamma, T=Tk, src_rows=src)
    agree(y, ry, "gathered y")
    dy = rnd((rows, D), 4); dx = torch.zeros(rows_all, D); dg = torch.zeros(D)
    EMU.ln_bwd(dy, x, rmu.float(), rrs.float(), gamma=gamma, T=Tk, src_rows=src, dx=dx, dx_mode=2, dgamma=dg)
    rdx, rdg, _, _ = R.ln_bwd(dy, x, gamma=gamma, shift=False, T=Tk, src_rows=src)
    agree(dx, R.scatter_rows(rdx, src, rows_all), "scattered dx"); agree(dg, rdg, "dgamma")
    # the pending residual scattered back to the gathered rows
    ya = rnd((rows_all, D), 5); xn = torch.zeros(rows_all, D)
    EMU.ln_fwd(x, y, mean, rstd, gamma=gamma, T=Tk, src_rows=src, y_add=ya, x_new=xn)
    ry, _, _, rxn = R.ln_fwd(x, gamma=gamma, T=Tk, src_rows=src, y_add=ya)
    agree(xn[src.long()], rxn, "gathered x_new"); agree(y, ry, "gathered y after residual")


def test_rownorm_and_its_vjp():
    rows, W = 77, 512
    x = rnd((rows, W), 1, scale=3.0)
    xe = x.clone(); rstd = torch.zeros(rows)
    EMU.rownorm_fwd(xe, rstd)
    rx, rr = R.rownorm_fwd(x)
    agree(xe, rx, "rownorm x"); agree(rstd, rr, "rstd")
    dy = rnd((rows, W), 2); de = dy.clone()
    EMU.rownorm_bwd(de, rx.float(), rr.float())
    ref = R.rownorm_bwd(dy, rx, rr)
    agree(de, ref, "rownorm dy")
    # the closed form is the VJP of the forward
    auto = R._grads(lambda v: R.rownorm_fwd(v)[0], [x], dy)[0]
    assert torch.allclose(ref, auto, rtol=1e-10, atol=1e-12)


def test_gate_bwd():
    rows, D, T = 128, 256, 64
    dres = rnd((rows, D), 1); y = rnd((rows, D), 2); mod = rnd((2, 4 * D), 3)
    dy = torch.zeros(rows, D); dmod = torch.zeros(2, 4 * D)
    EMU.gate_bwd(dres, dy, y=y, gate=mod[:, D:2 * D], dgate=dmod[:, 2 * D:3 * D], T=T)
    rdy, rdg = R.gate_bwd(dres, y=y, gate=mod[:, D:2 * D], T=T)
    agree(dy, rdy, "dy"); agree(dmod[:, 2 * D:3 * D], rdg, "dgate")


# ------------------------------------------------------------------------------------------------ FFN tails
def test_swiglu_and_gelu():
    rows, f = 64, 256
    u = rnd((rows, 2 * f), 1, scale=2.0); h = torch.zeros(rows, f)
    EMU.swiglu_fwd(u, h); agree(h, R.swiglu_fwd(u), "swiglu")
    dh = rnd((rows, f), 2); du = torch.zeros(rows, 2 * f)
    EMU.swiglu_bwd(dh, u, du); agree(du, R.swiglu_bwd(dh, u), "swiglu bwd")
    for act in (0, 1):
        x = rnd((rows, f), 3, scale=2.0); o = torch.zeros(rows, f)
        EMU.act_fwd(x, o, act); agree(o, R.act_fwd(x, act), f"act fwd {act}")
        EMU.act_bwd(dh, x, o, act); agree(o, R.act_bwd(dh, x, act), f"act bwd {act}")
    c = rnd((7, 512), 4, scale=2.0); o = torch.zeros(7, 512)
    EMU.gelu_tanh_f32_fwd(c, o); agree(o, R.gelu(c, 1), "gelu tanh f32")


# ------------------------------------------------------------------------------------------------ attention
@pytest.mark.parametrize("B,H,Tq,Tk,hd", [(2, 2, 64, 77, 64), (1, 3, 50, 40, 32)])
def test_attention(B, H, Tq, Tk, hd):
    hsz = H * hd
    q = rnd((B * Tq, hsz), 1); kv = rnd((B * Tk, 2 * hsz), 2); do = rnd((B * Tq, hsz), 3)
    o = torch.zeros(B * Tq, hsz); lse = torch.zeros(B, H, Tq)
    EMU.attn_fwd(q, kv[:, :hsz], kv[:, hsz:], o, lse, B, H, Tq, Tk, hd)
    ro, rl = R.attn_fwd(q, kv[:, :hsz], kv[:, hsz:], B, H, Tq, Tk, hd)
    agree(o, ro, "o"); agree(lse, rl, "lse (log2)")
    dq = torch.zeros(B * Tq, hsz); dkv = torch.zeros(B * Tk, 2 * hsz)
    EMU.attn_bwd(do, q, kv[:, :hsz], kv[:, hsz:], ro.float(), rl.float(), torch.zeros(B, H, Tq), dq, dkv[:, :hsz],
                 dkv[:, hsz:], B, H, Tq, Tk, hd)
    rdq, rdk, rdv = R.attn_bwd(do, q, kv[:, :hsz], kv[:, hsz:], B, H, Tq, Tk, hd)
    agree(dq, rdq, "dq"); agree(dkv[:, :hsz], rdk, "dk"); agree(dkv[:, hsz:], rdv, "dv")


# ------------------------------------------------------------------------------------------------ MoE
@pytest.mark.parametrize("B,T,E,k,D", [(2, 64, 8, 16, 128), (3, 33, 4, 8, 64)])
def test_moe_router(B, T, E, k, D):
    rows = B * T
    x = rnd((rows, D), 1); wg = rnd((E, D), 2, scale=D ** -0.5)
    probs = torch.zeros(rows, E)
    EMU.moe_gate_fwd(x, wg, probs); agree(probs, R.moe_gate_fwd(x, wg), "probs")
    _, idx, gval, inv = _routing(B, T, E, k, 3)
    probs = R.moe_gate_fwd(x, wg).float()
    EMU.moe_topk(probs, idx, gval, inv, B, T, E, k)
    h2 = rnd((E, B * k, D), 4); xres = rnd((rows, D), 5); mod = rnd((B, 2 * D), 6)
    xout = torch.zeros(rows, D); ym = torch.zeros(rows, D)
    EMU.moe_combine_fwd(h2, gval, inv, xres, mod[:, D:], xout, ym, B, T, E, k)
    ry, rx = R.moe_combine_fwd(h2, gval, idx, B, T, E, k, xres, mod[:, D:])
    agree(ym, ry, "ymoe"); agree(xout, rx, "xout")
    dy = rnd((rows, D), 7); dh2 = torch.zeros(E, B * k, D); dgv = torch.zeros(B, E, k)
    EMU.moe_combine_bwd(dy, h2, gval, idx, dh2, dgv, B, T, E, k)
    rdh2, rdg = R.moe_combine_bwd(dy, h2, gval, idx, B, T, E, k)
    agree(dh2, rdh2, "dh2"); agree(dgv, rdg, "dgval")
    dxin = rnd((E, B * k, D), 8); ds = torch.zeros(rows, E); dx = torch.zeros(rows, D)
    EMU.moe_dx_bwd(dxin, inv, dgv, probs, wg, ds, dx, B, T, E, k)
    rds, rdx = R.moe_dx_bwd(dxin, idx, dgv, probs, wg, B, T, E, k)
    agree(ds, rds, "dscores"); agree(dx, rdx, "dx")
    base = rnd((E, D), 9); dwg = base.clone()
    EMU.moe_gate_wgrad(ds, x, dwg); agree(dwg, R.moe_gate_wgrad(ds, x, base), "dwg")


# ------------------------------------------------------------------------------------------------ EDM
@pytest.mark.parametrize("masked,use_sigma", [(True, False), (False, True)])
def test_edm(masked, use_sigma):
    B, C, H, p = 3, 4, 16, 2
    T = (H // p) ** 2
    Tk = T // 4 if masked else T
    lat = rnd((B, C, H, H), 1, scale=0.8); eps = rnd((B, C, H, H), 2); r = rnd((B,), 3)
    sig = torch.exp(rnd((B,), 4)) if use_sigma else None
    xn = torch.zeros(B, C, H, H); pt = torch.zeros(B * T, C * p * p); coef = torch.zeros(6, B)
    EMU.edm_prepare(lat, eps, None if use_sigma else r, sig, -0.6, 1.2, 0.9, xn, pt, coef, p)
    rxn, rpt, rco = R.edm_prepare(lat, eps, p, rnd=None if use_sigma else r, sigma_in=sig, p_mean=-0.6, p_std=1.2,
                                  sigma_data=0.9)
    agree(xn, rxn, "xn"); agree(pt, rpt, "patches"); agree(coef, rco, "coef")
    kr = None
    if masked:
        kr = torch.stack([torch.randperm(T, generator=g(5))[:Tk] + b * T for b in range(B)]).reshape(-1).to(I32)
    ftok = rnd((B * Tk, C * p * p), 6)
    ps = torch.zeros(B); loss = torch.zeros(1)
    EMU.edm_loss_fwd(ftok, kr, lat, xn, coef, ps, loss, p, Tk)
    rps, rloss = R.edm_loss_fwd(ftok, lat, rxn, rco, p, Tk, kr)
    agree(ps, rps, "per-sample loss"); agree(loss, rloss.reshape(1), "loss")
    gs = torch.tensor([0.37]); dft = torch.zeros(B * Tk, C * p * p)
    EMU.edm_loss_bwd(ftok, kr, lat, xn, coef, gs, dft, p, Tk)
    agree(dft, R.edm_loss_bwd(ftok, lat, rxn, rco, gs, p, Tk, kr), "dftok")
    rs = torch.stack([torch.randperm(T, generator=g(6 + b)) for b in range(B)]).to(I32) if masked else None
    mt = rnd((C * p * p,), 7)
    fx = torch.zeros(B, C, H, H); dx = torch.zeros(B, C, H, H)
    EMU.edm_output(ftok, rs, mt, xn, coef, fx, dx, p, Tk)
    rfx, rdx = R.edm_output(ftok, p, (B, C, H, H), rco, rxn, rs, mt)
    agree(fx, rfx, "F"); agree(dx, rdx, "D_x")


@pytest.mark.parametrize("scaled", [False, True])
def test_patchify_and_adjoints(scaled):
    B, C, H, p = 2, 4, 16, 2
    T = (H // p) ** 2
    emu = BiasEmuOps("cpu", exact=True)
    x = rnd((B, C, H, H), 1); sc = rnd((B,), 2) if scaled else None
    pt = torch.zeros(B * T, C * p * p)
    emu.patchify(x, sc, pt, p); agree(pt, R.patchify(x, p, sc), "patchify")
    dp = rnd((B * T, C * p * p), 3); dx = torch.zeros(B, C, H, H)
    emu.patchify_bwd(dp, sc, dx, p)
    rdx = R.patchify_bwd(dp, p, (B, C, H, H), sc)
    agree(dx, rdx, "patchify_bwd")
    # adjoint identity <patchify(x), dp> == <x, patchify^T(dp)>
    assert math.isclose(float((R.patchify(x, p, sc) * dp.double()).sum()), float((x.double() * rdx).sum()), rel_tol=1e-12)


@pytest.mark.parametrize("masked", [False, True])
def test_unpatchify_adjoint(masked):
    B, C, H, p = 2, 4, 16, 2
    T = (H // p) ** 2
    Tk = T // 4 if masked else T
    emu = BiasEmuOps("cpu", exact=True)
    kr = torch.stack([torch.randperm(T, generator=g(5))[:Tk] + b * T for b in range(B)]).reshape(-1).to(I32) if masked else None
    dF = rnd((B, C, H, H), 1); dft = torch.zeros(B * Tk, p * p * C)
    emu.unpatchify_bwd(dF, kr, dft, p, Tk)
    ref = R.unpatchify_bwd(dF, p, Tk, kr)
    agree(dft, ref, "unpatchify_bwd")
    f = rnd((B * Tk, p * p * C), 2)
    lhs = float((R.unpatchify(f, p, (B, C, H, H), keep_rows=kr) * dF.double()).sum())
    assert math.isclose(lhs, float((f.double() * ref).sum()), rel_tol=1e-12)
    if not masked:  # unpatchify == edm_output's F without masking
        fx = torch.zeros(B, C, H, H)
        EMU.edm_output(f, None, None, None, None, fx, None, p, Tk)
        agree(fx, R.unpatchify(f, p, (B, C, H, H)), "unpatchify")


@pytest.mark.parametrize("dim", [256, 257])
def test_timestep_embed_and_adjoint(dim):
    emu = BiasEmuOps("cpu", exact=True)
    t = rnd((5,), 1, scale=3.0); out = torch.zeros(5, dim)
    if dim % 2 == 0:  # the odd width (a zero last column) is the kernel's alone
        emu.timestep_embed(t, out)
        agree(out, R.timestep_embed(t, dim), "timestep embed")
    assert torch.equal(R.timestep_embed(t, dim)[:, -1] == 0, torch.full((5,), dim % 2 == 1))
    d = rnd((5, dim), 2); dt = torch.zeros(5)
    ref = R.timestep_embed_bwd(d, t)
    if dim % 2 == 0:
        emu.timestep_embed_bwd(d, t, dt)
        agree(dt, ref, "timestep embed bwd", 1e-5)
    # adjoint identity against the forward, direction v: <J v, d> == <v, J^T d>
    v = rnd((5,), 3).double()
    h = 1e-6
    jv = (R.timestep_embed(t.double() + h * v, dim) - R.timestep_embed(t.double() - h * v, dim)) / (2 * h)
    assert math.isclose(float((jv * d.double()).sum()), float((v * ref).sum()), rel_tol=1e-7)


def test_reductions():
    B, L, D = 3, 77, 256
    x = rnd((B * L, D), 1); out = torch.zeros(B, D)
    EMU.mean_tokens_fwd(x, out, B, L); agree(out, R.mean_tokens(x, B, L), "mean tokens")
    n = 100003
    v = rnd((n,), 2); ss = torch.zeros(1)
    EMU.sumsq(v, ss); agree(ss, R.sumsq(v).reshape(1), "sumsq")
    xs = rnd((700, 200), 3); base = rnd((200,), 4); cs = base.clone()
    EMU.colsum(xs, cs); agree(cs, base.double() + R.colsum(xs), "colsum")
    f = 96
    xi = rnd((300, 2 * f), 5); out = torch.zeros(2 * f)
    BiasEmuOps("cpu", exact=True).colsum_interleaved(xi, out, f)
    agree(out, R.colsum_interleaved(xi, f), "colsum interleaved")
    # the interleave map is a permutation: every natural column is hit once
    assert torch.equal(torch.sort(R.interleaved_to_natural(f)).values, torch.arange(2 * f))
