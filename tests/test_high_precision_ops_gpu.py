"""High-precision mode (CudaOps(precision="high"), every _TAKES_PREC entry point at prec=1, GEMMs as 3-way bf16 splits)
op by op against the float64 references of tests/f64_reference.py.

Every bound comes from an error model of the op, written out below, and is checked element by element; each case prints
its worst error as a fraction of its bound.  u = 2^-24 is the fp32 unit roundoff.

* Reductions of n terms t_i inside one row (LayerNorm / rownorm statistics, the per-sample and per-column sums of the
  backward passes, token means): recursive-summation worst case n u sum|t_i|, with the condition taken from the terms,
  not from the result -- dx = rstd (g - mean g - xhat mean(g xhat)) is bounded by rstd (|g| + |mean g| + |xhat| |mean(g
  xhat)|) plus the reduction terms, which is what cancellation amplifies.  Elementwise steps add c u |each term|.
* Dot products of random operands (GEMM, attention scores and the attention sums): the per-product errors are
  independent and zero-mean, so they add in quadrature.  GEMM: hi = bf16(x), lo = bf16(x - hi) leave |x - hi - lo| <=
  2^-17 |x| per operand and drop a_lo b_lo (<= 2^-18 |a b|), about 2^-16 |a_k b_k| per product; fp32 accumulation of the
  3K products adds about sqrt(3K) 2^-24 |a_k b_k| in RMS.  Element bound: 8 (2^-16 + sqrt(3K) 2^-24) sqrt(sum_k a_k^2
  b_k^2); the factor 8 covers the Gaussian tail over ~10^6 elements.  A plain bf16 GEMM (2^-9 per operand) misses that
  bound by more than 8x: asserted on every GEMM case.
* Every output that would be stored in bf16 outside high-precision mode also asserts that rounding the exact result to
  bf16 breaks its bound by at least 2x, so a prec=1 kernel that rounds through bf16 cannot pass.

MD_TEST_DRYRUN=1 runs the same cases on oracle.emu_ops.EmuOps("cpu", exact=True) (fp32 torch on the CPU, plus the
test-side emulations of the adjoints in tests/dit_vjp_common.py / tests/bias_common.py): the references, the error
models and the bounds are exercised without a GPU.  Only the pure-copy cases are skipped there.
"""
import math
import os

import pytest
import torch

from tests import f64_reference as R
from tests.test_kernels_gpu import DEV, F32, I32, g, rnd

pytestmark = pytest.mark.gpu
DRY = bool(os.environ.get("MD_TEST_DRYRUN"))
DEVICE = "cpu" if DRY else DEV
U = 2.0 ** -24
D64 = torch.float64


def _ops():
    if DRY:
        from tests.bias_common import BiasEmuOps
        return BiasEmuOps("cpu", exact=True)
    from micro_diffusion_b200.ops import CudaOps
    return CudaOps(DEV, precision="high")


def dv(t):
    return None if t is None else t.to(DEVICE).clone()


def host(t):
    if not DRY:
        torch.cuda.synchronize()
    return t.detach().cpu().double()


def within(got, ref, bound, what, teeth=True):
    """max |got - ref| / bound <= 1 (printed); teeth: rounding ref to bf16 would exceed the bound at least 2x."""
    got = host(got)
    ref, bound = ref.double(), bound.double().clamp_min(1e-300)
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    assert torch.isfinite(got).all(), f"{what}: non-finite output"
    ratio = float(((got - ref).abs() / bound).max()) if ref.numel() else 0.0
    print(f"\n[{what}] error / bound = {ratio:.3f}", end="")
    assert ratio <= 1.0, f"{what}: error {ratio:.2f}x its bound"
    if teeth:
        bf = float(((ref.float().bfloat16().double() - ref).abs() / bound).max())
        assert bf >= 2.0, f"{what}: a bf16 rounding of the result would pass the bound ({bf:.2f}x)"


def exact(got, src, what):
    got = host(got)
    assert torch.equal(got, src.double()), f"{what}: not an exact copy"


def red(terms, dim, n=None):
    """Worst-case recursive-summation error of sum(terms, dim) in units of u: n sum |t|."""
    a = terms.abs()
    return (n or terms.shape[dim]) * a.sum(dim)


# ------------------------------------------------------------------------------------------------ GEMM
def _sq_dot(A, B, layout):
    """sqrt(sum_k a_k^2 b_k^2): the RMS scale of a dot product's rounding errors."""
    return R.matmul(A.double() ** 2, B.double() ** 2, layout).sqrt()


def _gemm_scale(A, B, layout, K):
    return 8.0 * (2.0 ** -16 + math.sqrt(3 * K) * U) * _sq_dot(A, B, layout)


def _teeth_bf16_gemm(A, B, layout, bound, what):
    """A plain bf16 GEMM of the same operands misses the bound by a wide margin."""
    lowp = R.matmul(A.bfloat16(), B.bfloat16(), layout)
    ratio = float(((lowp - R.matmul(A, B, layout)).abs() / bound).max())
    print(f"\n[{what}] a bf16 GEMM would be at {ratio:.1f}x the bound", end="")
    assert ratio >= 8.0, f"{what}: bound too loose to tell a bf16 GEMM ({ratio:.1f}x)"


# ragged M and N (not tile multiples); TN operands are MN-major, so there M and N are their row pitches and must stay
# multiples of 8 (16-byte TMA rows); K a multiple of 8 but not of 64 (72, 200, 520)
GEMM_SHAPES = [(0, 300, 640, 1024, 1), (0, 1000, 200, 320, 1), (0, 96, 128, 192, 1), (1, 768, 1024, 4000, 1),
               (0, 640, 384, 128, 3), (1, 256, 200, 1000, 3), (0, 130, 100, 72, 1), (1, 200, 136, 200, 1)]


@pytest.mark.parametrize("layout,M,N,K,batch", GEMM_SHAPES)
def test_gemm_store_epilogues(layout, M, N, K, batch):
    """EPI_BF16 (stored fp32 in this mode) and EPI_F32 + bias.  Bound: the split / accumulation model above plus
    4 u |result| for the bias add and the alpha scale."""
    ops = _ops()
    A = rnd((batch, M, K) if layout == 0 else (batch, K, M), 1); B = rnd((batch, N, K) if layout == 0 else (batch, K, N), 2)
    if batch == 1:
        A, B = A[0], B[0]
    shp = A.shape[:-2] + (M, N)
    base = _gemm_scale(A, B, layout, K)
    _teeth_bf16_gemm(A, B, layout, base, f"gemm {M}x{N}x{K}")
    C = torch.full(shp, 3.0, device=DEVICE)
    ops.gemm(dv(A), dv(B), C, layout=layout, epi=0)
    ref = R.gemm(A, B, layout)
    within(C, ref, base + 4 * U * ref.abs(), f"gemm bf16-epilogue {M}x{N}x{K} b{batch} L{layout}")
    bias = rnd((N,), 3)
    C = torch.full(shp, 3.0, device=DEVICE)
    ops.gemm(dv(A), dv(B), C, layout=layout, epi=1, bias=dv(bias), alpha=0.5)
    ref = R.gemm(A, B, layout, alpha=0.5, bias=bias)
    within(C, ref, 0.5 * base + 4 * U * (ref.abs() + bias.double().abs()), f"gemm f32+bias {M}x{N}x{K} b{batch} L{layout}")


@pytest.mark.parametrize("layout,M,N,K", [(0, 512, 768, 256), (0, 300, 640, 1024), (0, 77, 96, 200), (1, 152, 200, 320)])
def test_gemm_residual_epilogue(layout, M, N, K):
    """EPI_RESID: res[m % res_mod] + gate[m // T] * (acc + bias).  Bound: |gate| times the GEMM bound, plus
    4 u (|res| + |gate (acc + bias)|) for the epilogue's multiply and add."""
    ops = _ops()
    T = 64 if M % 64 == 0 else M
    A = rnd((M, K) if layout == 0 else (K, M), 1); B = rnd((N, K) if layout == 0 else (K, N), 2)
    bias = rnd((N,), 3); res = rnd((T, N), 4); gate = rnd((M // T, 2 * N), 5)
    C = torch.zeros(M, N, device=DEVICE)
    ops.gemm(dv(A), dv(B), C, layout=layout, epi=2, bias=dv(bias), res=dv(res), res_mod=T, gate=dv(gate)[:, N:],
             rows_per_gate=T)
    ref = R.gemm(A, B, layout, bias=bias, res=res, res_mod=T, gate=gate[:, N:], rows_per_gate=T)
    gr = R._per_row(gate[:, N:], T, M).abs()
    gated = (ref - res.double()[torch.arange(M) % T]).abs()
    within(C, ref, gr * _gemm_scale(A, B, layout, K) + 4 * U * (ref.abs() + gated + res.double()[torch.arange(M) % T].abs()),
           f"gemm resid {M}x{N}x{K} L{layout}")


@pytest.mark.parametrize("layout,M,N,K,batch,splits", [(1, 768, 1024, 4000, 1, 4), (1, 768, 1024, 4000, 1, 0),
                                                       (0, 300, 640, 1024, 1, 4), (1, 256, 200, 1000, 3, 0),
                                                       (0, 64, 1024, 16, 1, 4), (1, 136, 104, 520, 1, 4)])
def test_gemm_accumulate_epilogue(layout, M, N, K, batch, splits):
    """EPI_ATOMIC with a split reduction (4 or auto): C + acc.  The partial sums of the splits are reassociated fp32
    adds, inside the accumulation term of the model; plus 4 u |C + acc| for the final add."""
    ops = _ops()
    A = rnd((batch, M, K) if layout == 0 else (batch, K, M), 1); B = rnd((batch, N, K) if layout == 0 else (batch, K, N), 2)
    if batch == 1:
        A, B = A[0], B[0]
    acc0 = rnd(A.shape[:-2] + (M, N), 6)
    C = dv(acc0)
    ops.gemm(dv(A), dv(B), C, layout=layout, epi=3, splits=splits)
    ref = R.gemm(A, B, layout, accumulate=acc0)
    within(C, ref, _gemm_scale(A, B, layout, K) + 4 * U * (ref.abs() + acc0.double().abs()),
           f"gemm atomic {M}x{N}x{K} b{batch} s{splits}", teeth=False)


@pytest.mark.parametrize("M,N,K,batch", [(512, 768, 256, 1), (1000, 200, 320, 1), (640, 384, 128, 3), (96, 128, 192, 1)])
@pytest.mark.parametrize("act", [0, 1])
def test_gemm_activation_epilogues(M, N, K, batch, act):
    """EPI_ACT_DUAL (pre = alpha acc + bias, out = gelu(pre)) and EPI_ACT_GRAD (alpha acc * gelu'(aux)), which this mode
    runs as an fp32 GEMM and a second pass.  Bounds: gelu' or |gelu''|-free cover: the GEMM bound carried through
    |gelu'(pre)| <= 1.2, plus 16 u (|out| + |pre| (1 + pre^2)) for erf / tanh evaluation (a few ulps each, through at
    most four dependent operations); the gradient: |gelu'(aux)| times the GEMM bound plus 16 u |acc| (1 + |aux|)^3."""
    ops = _ops()
    A = rnd((batch, M, K), 1); B = rnd((batch, N, K), 2); bias = rnd((N,), 3)
    aux = rnd((batch, M, N), 4, scale=1.5)
    if batch == 1:
        A, B, aux = A[0], B[0], aux[0]
    shp = aux.shape
    pre, out = torch.zeros(shp, device=DEVICE), torch.zeros(shp, device=DEVICE)
    ops.gemm(dv(A), dv(B), pre, epi=4, C2=out, bias=dv(bias), act=act, alpha=0.05)
    rp, ro = R.gemm(A, B, alpha=0.05, bias=bias, act=act)
    gb = 0.05 * _gemm_scale(A, B, 0, K) + 4 * U * (rp.abs() + bias.double().abs())
    within(pre, rp, gb, f"act dual pre {act} {M}x{N}x{K}")
    within(out, ro, 1.2 * gb + 16 * U * (ro.abs() + rp.abs() * (1 + rp ** 2)), f"act dual out {act} {M}x{N}x{K}")
    dp = torch.zeros(shp, device=DEVICE)
    ops.gemm(dv(A), dv(B), dp, epi=5, aux=dv(aux), act=act, alpha=0.05)
    ref = R.gemm(A, B, alpha=0.05, aux=aux, act=act)
    accr = 0.05 * R.matmul(A, B)
    within(dp, ref, R.gelu_grad(aux, act).abs() * 0.05 * _gemm_scale(A, B, 0, K)
           + 16 * U * accr.abs() * (1 + aux.double().abs()) ** 3, f"act grad {act} {M}x{N}x{K}")


# ------------------------------------------------------------------------------------------------ attention
def _attn_bounds(q, k, v, do, B, H, Tq, Tk, hd):
    """Quadrature error model of md_attn_*_f32 in units of u (see the module docstring): per-score error
    e_s = ||q o k||_2 / sqrt(hd) * sqrt(hd) + |s| + |lse|, the sums over keys / queries add sqrt(n) |term|."""
    qh, kh, vh, doh = (R._heads(t, B, T, H, hd) for t, T in ((q, Tq), (k, Tk), (v, Tk), (do, Tq)))
    sc = 1.0 / math.sqrt(hd)
    s = qh @ kh.transpose(-1, -2) * sc
    lse = torch.logsumexp(s, -1, keepdim=True)
    P = torch.exp(s - lse)
    o = P @ vh
    es2 = hd * ((qh ** 2) @ (kh ** 2).transpose(-1, -2)) * sc ** 2 + s ** 2 + lse ** 2 + Tk
    c = 8.0
    bo = c * U * (((P ** 2 * es2) @ vh ** 2).sqrt() + o.abs() * (lse.abs() + math.sqrt(Tk)))
    blse = c * U * (((P ** 2 * es2).sum(-1)).sqrt() + lse[..., 0].abs() + math.sqrt(Tk)) * R.LOG2E
    dp = doh @ vh.transpose(-1, -2)
    delta = (doh * o).sum(-1, keepdim=True)
    ep2 = hd * ((doh ** 2) @ (vh ** 2).transpose(-1, -2)) + hd * ((doh ** 2) * o ** 2).sum(-1, keepdim=True) \
        + (doh.abs() * bo / U).sum(-1, keepdim=True) ** 2
    eds2 = P ** 2 * ((dp - delta) ** 2 * es2 + ep2)          # (error of dS / u)^2
    ds = P * (dp - delta)
    bdv = c * U * ((P ** 2 * (es2 + Tq)).transpose(-1, -2) @ doh ** 2).sqrt()
    bdq = c * U * sc * ((eds2 + Tk * ds ** 2) @ kh ** 2).sqrt()
    bdk = c * U * sc * ((eds2 + Tq * ds ** 2).transpose(-1, -2) @ qh ** 2).sqrt()
    return (R._unheads(bo), blse[..., 0] if blse.dim() == 4 else blse, R._unheads(bdq), R._unheads(bdk), R._unheads(bdv))


@pytest.mark.parametrize("hd", [32, 64])
@pytest.mark.parametrize("B,H,Tq,Tk", [(2, 3, 64, 64), (2, 2, 64, 77), (1, 3, 256, 77), (2, 2, 100, 200), (2, 2, 130, 33),
                                       (1, 2, 1024, 1024)])
def test_attention_f32(B, H, Tq, Tk, hd):
    """md_attn_fwd_f32 / md_attn_bwd_f32 against softmax attention and its autograd in float64.  Bound: the quadrature
    model of _attn_bounds (score errors through exp, key / query sums, dS = P (dP - delta))."""
    ops = _ops()
    hsz = H * hd
    qkv = rnd((B * Tq, 3 * hsz + 64), 1); kv = rnd((B * Tk, 2 * hsz), 2); do = rnd((B * Tq, hsz), 3)
    q, k, v = qkv[:, :hsz], kv[:, :hsz], kv[:, hsz:]
    ro, rl = R.attn_fwd(q, k, v, B, H, Tq, Tk, hd)
    bo, bl, bdq, bdk, bdv = _attn_bounds(q, k, v, do, B, H, Tq, Tk, hd)
    qd, kd = dv(qkv), dv(kv)
    o = torch.zeros(B * Tq, hsz, device=DEVICE); lse = torch.zeros(B, H, Tq, device=DEVICE)
    ops.attn_fwd(qd[:, :hsz], kd[:, :hsz], kd[:, hsz:], o, lse, B, H, Tq, Tk, hd)
    tag = f"B{B} H{H} {Tq}/{Tk} hd{hd}"
    within(o, ro, bo, f"attn o {tag}"); within(lse, rl, bl, f"attn lse {tag}", teeth=False)
    rdq, rdk, rdv = R.attn_bwd(do, q, k, v, B, H, Tq, Tk, hd)
    dq = torch.zeros(B * Tq, hsz, device=DEVICE); dkv = torch.zeros(B * Tk, 2 * hsz, device=DEVICE)
    ops.attn_bwd(dv(do), qd[:, :hsz], kd[:, :hsz], kd[:, hsz:], dv(ro.float()), dv(rl.float()),
                 torch.zeros(B, H, Tq, device=DEVICE), dq, dkv[:, :hsz], dkv[:, hsz:], B, H, Tq, Tk, hd)
    within(dq, rdq, bdq, f"attn dq {tag}"); within(dkv[:, :hsz], rdk, bdk, f"attn dk {tag}")
    within(dkv[:, hsz:], rdv, bdv, f"attn dv {tag}")


# ------------------------------------------------------------------------------------------------ LayerNorm
def _ln_fwd_bounds(xa, xh_a, rstd, w, D, y):
    """LayerNorm forward in units-of-u-scaled form: xa = |x| (the residual sum's |terms| when a residual is folded
    in), xh_a = |xhat|.  mean: D * mean|x|; variance: D * mean(xhat^2) relative; y = xhat w + shift."""
    S = rstd[:, None] * xa.mean(1, keepdim=True) + xh_a * 1.0
    return 4 * U * (D * S * w.abs() + (xa * rstd[:, None] + xh_a) * w.abs() + y.abs())


@pytest.mark.parametrize("D", [512, 768, 1024, 192, 256, 2048])
@pytest.mark.parametrize("T", [64, 77, 256])
def test_layernorm(D, T):
    """md_ln_fwd / md_ln_bwd (team kernels at 512 / 768 / 1024, the generic kernel at 192 / 256, the 16-vector instance
    at 2048) with the pending residual and the fused next-branch tail.  Bounds (units of u, times 4): forward
    D (rstd mean|x| + |xhat|) |w| + |x| rstd |w| + |y|; backward dx: rstd (|g| + |mean g| + |xa| |mean(g xhat)|) +
    D rstd (mean|g| + |xa| mean|g xa|) + |dx|, with xa = (|x| + |mean|) rstd; the per-sample / per-column sums
    (d shift, d scale, d gamma, d gate) the recursive-summation worst case; dy_next |gate| bound(dx) + |dy_next|."""
    ops = _ops()
    ns = 2
    rows = ns * T
    x = rnd((rows, D), 1, scale=2.0) + 0.5
    gamma = 1 + 0.1 * rnd((D,), 2); mod = rnd((ns, 6 * D), 3, scale=0.5)
    ya = rnd((rows, D), 4)
    sh, sc, ga = mod[:, D:2 * D], mod[:, 3 * D:4 * D], mod[:, 2 * D:3 * D]
    y = torch.zeros(rows, D, device=DEVICE); mean = torch.zeros(rows, device=DEVICE); rstd = torch.zeros(rows, device=DEVICE)
    xn = torch.zeros(rows, D, device=DEVICE); md = dv(mod)
    ops.ln_fwd(dv(x), y, mean, rstd, gamma=dv(gamma), shift=md[:, D:2 * D], scale=md[:, 3 * D:4 * D], T=T, y_add=dv(ya),
               gate_add=md[:, 2 * D:3 * D], x_new=xn)
    ry, rmu, rrs, rxn = R.ln_fwd(x, gamma=gamma, shift=sh, scale=sc, T=T, y_add=ya, gate_add=ga)
    w = gamma.double() * (1 + R._per_row(sc, T, rows))
    xa = x.double().abs() + (ya.double() * R._per_row(ga, T, rows)).abs()
    xh = ((rxn - rmu[:, None]) * rrs[:, None])
    tag = f"D{D} T{T}"
    within(xn, rxn, 4 * U * xa, f"ln x_new {tag}", teeth=False)
    within(y, ry, _ln_fwd_bounds(xa, xh.abs(), rrs, w, D, ry) + 4 * U * sh.double().abs().repeat_interleave(T, 0),
           f"ln y {tag}")
    within(mean, rmu, 4 * U * D * xa.mean(1), f"ln mean {tag}", teeth=False)
    within(rstd, rrs, 4 * U * D * rrs * (1 + rrs * xa.mean(1)), f"ln rstd {tag}", teeth=False)
    # backward at the saved (exact, fp32-rounded) statistics of x_new, with the fused tail into the next branch
    dy = rnd((rows, D), 5); dx0 = rnd((rows, D), 6); yn = rnd((rows, D), 7)
    dx = dv(dx0); dg = torch.zeros(D, device=DEVICE); dmod = torch.zeros(ns, 6 * D, device=DEVICE)
    dyn = torch.zeros(rows, D, device=DEVICE)
    ops.ln_bwd(dv(dy), dv(rxn.float()), dv(rmu.float()), dv(rrs.float()), gamma=dv(gamma), scale=md[:, 3 * D:4 * D], T=T,
               dx=dx, dx_mode=0, dgamma=dg, dshift=dmod[:, :D], dscale=dmod[:, 2 * D:3 * D], dy_next=dyn, y_next=dv(yn),
               gate_next=md[:, 5 * D:], dgate_next=dmod[:, 4 * D:5 * D])
    rdx, rdg, rdsh, rdsc = R.ln_bwd(dy, rxn.float(), gamma=gamma, scale=sc, T=T)
    gg = dy.double() * w
    r = rrs[:, None]
    xa_h = (rxn.double().abs() + rmu.abs()[:, None]) * r
    m1, m2 = gg.mean(1, keepdim=True), (gg * xh).mean(1, keepdim=True)
    bdx = 4 * U * (r * (gg.abs() + m1.abs() + xa_h * m2.abs()) + D * r * ((gg.abs()).mean(1, keepdim=True)
                   + xa_h * (gg.abs() * xa_h).mean(1, keepdim=True)) + (dx0.double() + rdx).abs() + dx0.double().abs())
    within(dx, dx0.double() + rdx, bdx, f"ln dx {tag}", teeth=False)
    t_sh = dy.double().reshape(ns, T, D)
    t_sc = (dy.double() * xh).reshape(ns, T, D)
    bxh = 4 * U * (xa_h + D * xa_h)        # |error of xhat| / u scale per element (mean / rstd inputs rounded)
    within(dmod[:, :D], rdsh, 2 * U * red(t_sh, 1), f"ln dshift {tag}", teeth=False)
    within(dmod[:, 2 * D:3 * D], rdsc, 2 * U * red(t_sc, 1) * gamma.double().abs()
           + (dy.double().abs() * bxh).reshape(ns, T, D).sum(1) * gamma.double().abs(), f"ln dscale {tag}", teeth=False)
    t_g = (dy.double() * xh * (1 + R._per_row(sc, T, rows)))
    within(dg, rdg, 2 * U * red(t_g, 0) + (dy.double().abs() * bxh * (1 + R._per_row(sc, T, rows)).abs()).sum(0),
           f"ln dgamma {tag}", teeth=False)
    gn = R._per_row(mod[:, 5 * D:], T, rows)
    rdyn, rdgn = R.gate_bwd(dx0.double() + rdx, y=yn, gate=mod[:, 5 * D:], T=T)
    within(dyn, rdyn, gn.abs() * bdx + 2 * U * rdyn.abs(), f"ln dy_next {tag}")
    within(dmod[:, 4 * D:5 * D], rdgn, 2 * U * red(((dx0.double() + rdx) * yn.double()).reshape(ns, T, D), 1)
           + (bdx * yn.double().abs()).reshape(ns, T, D).sum(1), f"ln dgate_next {tag}", teeth=False)


def test_layernorm_gather_scatter_and_copy_out():
    """Gathered rows (src_rows) forward, the scattered dx (dx_mode 2) and the overwritten dx (dx_mode 1, the bf16 path's
    output, fp32 here), with the bounds of test_layernorm."""
    ops = _ops()
    rows_all, D, B, T, Tk = 128, 768, 2, 64, 16
    x = rnd((rows_all, D), 1)
    src = torch.stack([torch.randperm(T, generator=g(7))[:Tk] + b * T for b in range(B)]).reshape(-1).to(I32)
    gamma = 1 + 0.1 * rnd((D,), 2)
    rows = B * Tk
    y = torch.zeros(rows, D, device=DEVICE); mean = torch.zeros(rows, device=DEVICE); rstd = torch.zeros(rows, device=DEVICE)
    ops.ln_fwd(dv(x), y, mean, rstd, gamma=dv(gamma), T=Tk, src_rows=dv(src))
    ry, rmu, rrs, rxv = R.ln_fwd(x, gamma=gamma, T=Tk, src_rows=src)
    xh = (rxv - rmu[:, None]) * rrs[:, None]
    within(y, ry, _ln_fwd_bounds(rxv.abs(), xh.abs(), rrs, gamma.double().expand(rows, D), D, ry), "ln gathered y")
    dy = rnd((rows, D), 4)
    rdx, rdg, _, _ = R.ln_bwd(dy, x, gamma=gamma, shift=False, T=Tk, src_rows=src)
    gg = dy.double() * gamma.double()
    r = rrs[:, None]
    xa_h = (rxv.abs() + rmu.abs()[:, None]) * r
    bdx = 4 * U * (r * (gg.abs() + gg.mean(1, keepdim=True).abs() + xa_h * (gg * xh).mean(1, keepdim=True).abs())
                   + D * r * (gg.abs().mean(1, keepdim=True) + xa_h * (gg.abs() * xa_h).mean(1, keepdim=True)) + rdx.abs())
    dx = torch.zeros(rows_all, D, device=DEVICE); dg = torch.zeros(D, device=DEVICE)
    ops.ln_bwd(dv(dy), dv(x), dv(rmu.float()), dv(rrs.float()), gamma=dv(gamma), T=Tk, src_rows=dv(src), dx=dx, dx_mode=2,
               dgamma=dg)
    within(dx, R.scatter_rows(rdx, src, rows_all), R.scatter_rows(bdx, src, rows_all), "ln scattered dx", teeth=False)
    dxc = torch.full((rows, D), 7.0, device=DEVICE)
    ops.ln_bwd(dv(dy), dv(x), dv(rmu.float()), dv(rrs.float()), gamma=dv(gamma), T=Tk, src_rows=dv(src), dx=dxc, dx_mode=1)
    within(dxc, rdx, bdx, "ln dx (mode 1)")


# ------------------------------------------------------------------------------------------------ rownorm / gate
@pytest.mark.parametrize("rows,W,ld,off,ns", [(200, 512, 1536, 512, 1), (77, 1024, 2048, 0, 1), (33, 64, 192, 64, 1),
                                              (201, 512, 1536, 0, 2), (77, 768, 2304, 0, 2), (5, 64, 256, 64, 3),
                                              (40, 2048, 2048, 0, 1)])
def test_rownorm(rows, W, ld, off, ns):
    """md_rownorm_fwd / _bwd on column slices, every W-wide slice on its own.  Bounds as LayerNorm without affine
    parameters; backward rstd (|d| + |mean d| + |xhat| |mean(d xhat)|) + W rstd (mean|d| + |xhat| mean|d xhat|)."""
    ops = _ops()
    buf = rnd((rows, ld), 1, scale=3.0)
    rstd = torch.zeros(ns, rows, device=DEVICE)
    bd = dv(buf)
    ops.rownorm_fwd(bd[:, off:off + ns * W], rstd, 1e-6, nslice=ns)
    dyb = rnd((rows, ld), 2)
    dyd = dv(dyb)
    xh_all, rs_all = [], []
    for s in range(ns):
        xs = buf[:, off + s * W:off + (s + 1) * W]
        rx, rr = R.rownorm_fwd(xs)
        xh_all.append(rx); rs_all.append(rr)
        xa = xs.double().abs()
        within(bd[:, off + s * W:off + (s + 1) * W], rx, _ln_fwd_bounds(xa, rx.abs(), rr, torch.ones(1, dtype=D64), W, rx),
               f"rownorm x {rows}x{W} slice {s}")
        within(rstd[s], rr, 4 * U * W * rr * (1 + rr * xa.mean(1)), f"rownorm rstd slice {s}", teeth=False)
    xh_in = dv(torch.cat([t.float() for t in xh_all], 1))
    xbuf = torch.zeros(rows, ld, device=DEVICE); xbuf[:, off:off + ns * W] = xh_in
    rsd = dv(torch.stack([t.float() for t in rs_all]))
    ops.rownorm_bwd(dyd[:, off:off + ns * W], xbuf[:, off:off + ns * W], rsd, nslice=ns)
    for s in range(ns):
        d = dyb[:, off + s * W:off + (s + 1) * W].double()
        xh = xh_all[s].float().double(); r = rs_all[s].float().double()[:, None]
        ref = R.rownorm_bwd(d, xh, r[:, 0])
        m1, m2 = d.mean(1, keepdim=True), (d * xh).mean(1, keepdim=True)
        b = 4 * U * (r * (d.abs() + m1.abs() + xh.abs() * m2.abs()) + W * r * (d.abs().mean(1, keepdim=True)
                     + xh.abs() * (d * xh).abs().mean(1, keepdim=True)) + ref.abs())
        within(dyd[:, off + s * W:off + (s + 1) * W], ref, b, f"rownorm dy {rows}x{W} slice {s}")
    # the columns outside the slices are untouched
    keep = torch.ones(ld, dtype=torch.bool); keep[off:off + ns * W] = False
    assert torch.equal(host(bd)[:, keep], buf.double()[:, keep]) and torch.equal(host(dyd)[:, keep], dyb.double()[:, keep])


@pytest.mark.parametrize("rows,D,T", [(192, 768, 64), (154, 256, 77), (128, 2048, 64)])
def test_gate_bwd(rows, D, T):
    """md_gate_bwd: dy = gate dres (one product: 2 u |dy|), dgate = sum_t dres y (recursive summation over T)."""
    ops = _ops()
    dres = rnd((rows, D), 1); y = rnd((rows, D), 2); mod = rnd((rows // T, 4 * D), 3)
    dy = torch.zeros(rows, D, device=DEVICE); dmod = torch.zeros(rows // T, 4 * D, device=DEVICE); md = dv(mod)
    ops.gate_bwd(dv(dres), dy, y=dv(y), gate=md[:, D:2 * D], dgate=dmod[:, 2 * D:3 * D], T=T)
    rdy, rdg = R.gate_bwd(dres, y=y, gate=mod[:, D:2 * D], T=T)
    within(dy, rdy, 2 * U * rdy.abs(), f"gate dy {rows}x{D}")
    within(dmod[:, 2 * D:3 * D], rdg, 2 * U * red((dres.double() * y.double()).reshape(-1, T, D), 1), f"dgate {rows}x{D}",
           teeth=False)
    dy2 = torch.zeros(rows, D, device=DEVICE)
    ops.gate_bwd(dv(dres), dy2, T=T)
    within(dy2, dres.double(), 2 * U * dres.double().abs(), "gate_bwd copy")


# ------------------------------------------------------------------------------------------------ FFN tails
def test_swiglu_and_activations():
    """SwiGLU and GELU forward / backward.  Bounds: 16 u times the sum of |terms| of each formula (exp / erf / tanh are a
    few ulps each, composed through at most four operations): swiglu |h| + |u1 u2|; its gradient |du| + |d|
    (|u2| (1 + |u1|) + |u1|); gelu |y| + |x| (1 + x^2); its gradient |d| (1 + |x|)^3."""
    ops = _ops()
    rows, f = 300, 1024
    u = rnd((rows, 2 * f), 1, scale=2.0); h = torch.zeros(rows, f, device=DEVICE)
    ops.swiglu_fwd(dv(u), h)
    ref = R.swiglu_fwd(u); a, b = u[:, :f].double(), u[:, f:].double()
    within(h, ref, 16 * U * (ref.abs() + (a * b).abs()), "swiglu")
    dh = rnd((rows, f), 2); du = torch.zeros(rows, 2 * f, device=DEVICE)
    ops.swiglu_bwd(dv(dh), dv(u), du)
    ref = R.swiglu_bwd(dh, u); d = dh.double().abs()
    t = torch.cat([d * b.abs() * (1 + a.abs()), d * a.abs()], 1)
    within(du, ref, 16 * U * (ref.abs() + t), "swiglu bwd")
    for act in (0, 1):
        x = rnd((rows, f), 3, scale=2.0); out = torch.zeros(rows, f, device=DEVICE)
        ops.act_fwd(dv(x), out, act)
        ref = R.act_fwd(x, act); xa = x.double().abs()
        within(out, ref, 16 * U * (ref.abs() + xa * (1 + xa ** 2)), f"gelu fwd {act}")
        dp = torch.zeros(rows, f, device=DEVICE)
        ops.act_bwd(dv(dh), dv(x), dp, act)
        ref = R.act_bwd(dh, x, act)
        within(dp, ref, 16 * U * (ref.abs() + d * (1 + xa) ** 3), f"gelu bwd {act}")
    c = rnd((7, 512), 4, scale=2.0); out = torch.zeros(7, 512, device=DEVICE)
    ops.gelu_tanh_f32_fwd(dv(c), out)
    ref = R.gelu(c, 1); ca = c.double().abs()
    within(out, ref, 16 * U * (ref.abs() + ca * (1 + ca ** 2)), "gelu tanh f32 fwd")


# ------------------------------------------------------------------------------------------------ MoE
@pytest.mark.parametrize("B,T,E,cap,D", [(3, 64, 8, 2.0, 256), (2, 256, 8, 2.0, 768), (2, 100, 4, 1.0, 128),
                                          (3, 67, 8, 2.0, 1024), (1, 33, 16, 2.0, 512)])
def test_moe_router(B, T, E, cap, D):
    """Router softmax, expert gather (an exact copy), combine, combine_bwd, dx_bwd and the gate weight gradient.
    Bounds: scores x wg^T carry D u (|x| |wg|) (worst case), softmax turns a score error into a relative error of the
    probabilities: p (e_s + sum_j p_j e_s,j + E); combine sums <= E gated products: 4 u E sum|g h|; dscores / dx /
    the weight gradient: recursive summation of their terms."""
    ops = _ops()
    k = int(cap * T / E)
    rows = B * T
    x = rnd((rows, D), 1); wg = rnd((E, D), 2, scale=D ** -0.5)
    probs = torch.zeros(rows, E, device=DEVICE)
    ops.moe_gate_fwd(dv(x), dv(wg), probs)
    rp = R.moe_gate_fwd(x, wg)
    es = D * (x.double().abs() @ wg.double().abs().t())
    within(probs, rp, 4 * U * rp * (es + (rp * es).sum(-1, keepdim=True) + E), f"probs B{B} T{T} E{E} D{D}", teeth=False)
    from oracle.emu_ops import EmuOps
    pr = rp.float()
    idx = torch.zeros(B, E, k, dtype=I32); gval = torch.zeros(B, E, k); inv = torch.zeros(B, T, E, dtype=I32)
    EmuOps("cpu").moe_topk(pr, idx, gval, inv, B, T, E, k)
    if not DRY:
        xin = torch.zeros(E, B * k, D, device=DEVICE)
        ops.moe_gather(dv(x), dv(idx), xin, B, T, E, k)
        tok = (torch.arange(B)[:, None, None] * T + idx.long()).permute(1, 0, 2).reshape(E, B * k)
        exact(xin, x[tok], "moe gather")
    h2 = rnd((E, B * k, D), 3); xres = rnd((rows, D), 4); mod = rnd((B, 2 * D), 5)
    xout = torch.zeros(rows, D, device=DEVICE); ym = torch.zeros(rows, D, device=DEVICE)
    ops.moe_combine_fwd(dv(h2), dv(gval), dv(inv), dv(xres), dv(mod)[:, D:], xout, ym, B, T, E, k)
    ry, rx = R.moe_combine_fwd(h2, gval, idx, B, T, E, k, xres, mod[:, D:])
    ya, _ = R.moe_combine_fwd(h2.abs(), gval.abs(), idx, B, T, E, k)
    gt = R._per_row(mod[:, D:], T, rows).abs()
    within(ym, ry, 4 * U * E * ya, f"ymoe B{B} T{T} E{E} D{D}")
    within(xout, rx, 4 * U * (E * ya * gt + xres.double().abs() + rx.abs()), f"xout B{B} T{T} E{E} D{D}", teeth=False)
    dy = rnd((rows, D), 6); dh2 = torch.zeros(E, B * k, D, device=DEVICE); dg = torch.zeros(B, E, k, device=DEVICE)
    ops.moe_combine_bwd(dv(dy), dv(h2), dv(gval), dv(idx), dh2, dg, B, T, E, k)
    rdh2, rdg = R.moe_combine_bwd(dy, h2, gval, idx, B, T, E, k)
    within(dh2, rdh2, 2 * U * rdh2.abs(), f"dh2 B{B} T{T} E{E} D{D}")
    _, adg = R.moe_combine_bwd(dy.abs(), h2.abs(), gval, idx, B, T, E, k)
    within(dg, rdg, 2 * U * D * adg, f"dgval B{B} T{T} E{E} D{D}", teeth=False)
    dxin = rnd((E, B * k, D), 7); ds = torch.zeros(rows, E, device=DEVICE); dx = torch.zeros(rows, D, device=DEVICE)
    ops.moe_dx_bwd(dv(dxin), dv(inv), dv(rdg.float()), dv(pr), dv(wg), ds, dx, B, T, E, k)
    rds, rdx = R.moe_dx_bwd(dxin, idx, rdg.float(), pr, wg, B, T, E, k)
    dpa = torch.zeros(rows, E, dtype=D64)
    tok, e_, _ = R._routes(idx, B, E, k, T)
    dpa[tok, e_] = rdg.float().double().abs().reshape(-1)
    pd = pr.double()
    bds = 4 * U * E * pd * (dpa + (pd * dpa).sum(-1, keepdim=True))
    within(ds, rds, bds, f"dscores B{B} T{T} E{E} D{D}", teeth=False)
    dxa = rds.abs() @ wg.double().abs()
    dxa.index_add_(0, tok, dxin.double().abs()[e_, R._routes(idx, B, E, k, T)[2]])
    within(dx, rdx, 4 * U * 2 * E * dxa + bds @ wg.double().abs(), f"moe dx B{B} T{T} E{E} D{D}")
    base = rnd((E, D), 8); dwg = dv(base)
    ops.moe_gate_wgrad(dv(rds.float()), dv(x), dwg)
    ref = R.moe_gate_wgrad(rds.float(), x, base)
    within(dwg, ref, 2 * U * (rows * (rds.float().double().abs().t() @ x.double().abs()) + ref.abs()),
           f"dwg B{B} T{T} E{E} D{D}", teeth=False)


# ------------------------------------------------------------------------------------------------ EDM and DiT I/O maps
@pytest.mark.parametrize("B,C,H,p,masked,f16,use_sigma", [(4, 4, 32, 2, True, True, False), (2, 16, 16, 2, False, True, True),
                                                          (3, 4, 64, 2, True, False, False), (2, 4, 32, 4, False, False, True)])
def test_edm_prepare_and_loss_backward(B, C, H, p, masked, f16, use_sigma):
    """md_edm_prepare (rnd or sigma_in) and md_edm_loss_bwd.  Bounds: coefficients 16 u |c| (exp, sqrt, division);
    xn = lat + sigma eps: 4 u (|lat| + |sigma eps|) plus sigma's error times |eps|; patches c_in xn: 4 u |patch| plus
    |c_in| times xn's bound; dftok = gscale / (B Tk C p^2) 2 w c_out (c_skip xn + c_out F - x): 16 u times the sum of
    the |terms| of the residual."""
    ops = _ops()
    T = (H // p) ** 2
    Tk = T // 4 if masked else T
    lat = rnd((B, C, H, H), 1, torch.float16 if f16 else F32, 0.8); eps = rnd((B, C, H, H), 2); r = rnd((B,), 3)
    sig = torch.exp(rnd((B,), 9)) if use_sigma else None
    xn = torch.zeros(B, C, H, H, device=DEVICE); pt = torch.zeros(B * T, C * p * p, device=DEVICE)
    coef = torch.zeros(6, B, device=DEVICE)
    ops.edm_prepare(dv(lat), dv(eps), None if use_sigma else dv(r), dv(sig), -0.6, 1.2, 0.9, xn, pt, coef, p)
    rxn, rpt, rco = R.edm_prepare(lat, eps, p, rnd=None if use_sigma else r, sigma_in=sig, p_mean=-0.6, p_std=1.2,
                                  sigma_data=0.9)
    tag = f"B{B} C{C} H{H} p{p}"
    within(coef, rco, 16 * U * rco.abs(), f"coef {tag}", teeth=False)
    bsig = (16 * U * rco[0].abs()).reshape(B, 1, 1, 1)
    bxn = 4 * U * (lat.double().abs() + (rco[0].reshape(B, 1, 1, 1) * eps.double()).abs()) + bsig * eps.double().abs()
    within(xn, rxn, bxn, f"xn {tag}", teeth=False)
    within(pt, rpt, 16 * U * rpt.abs() + R.patchify(bxn, p, rco[3]), f"patches {tag}")
    kr = None
    if masked:
        kr = torch.stack([torch.randperm(T, generator=g(5))[:Tk] + b * T for b in range(B)]).reshape(-1).to(I32)
    ftok = rnd((B * Tk, C * p * p), 4)
    gs = torch.tensor([0.37]); dft = torch.zeros(B * Tk, C * p * p, device=DEVICE)
    xnf = rxn.float(); cof = rco.float()
    ops.edm_loss_bwd(dv(ftok), dv(kr), dv(lat), dv(xnf), dv(cof), dv(gs), dft, p, Tk)
    ref = R.edm_loss_bwd(ftok, lat, xnf, cof, gs, p, Tk, kr)
    # the gradient at |ftok|, |xn|, |coef| and -|lat| is scale * (sum of the |terms| of the residual)
    a = R.edm_loss_bwd(ftok.abs(), -lat.double().abs(), xnf.abs(), cof.abs(), gs, p, Tk, kr)
    within(dft, ref, 16 * U * (a.abs() + ref.abs()), f"dftok {tag}")


@pytest.mark.parametrize("B,C,H,p,scaled", [(2, 4, 32, 2, False), (3, 16, 16, 2, True), (2, 4, 32, 4, True)])
def test_patchify_and_adjoints(B, C, H, p, scaled):
    """md_patchify (a copy, times scale[b]: 2 u |x s|), md_patchify_bwd (its adjoint, a copy / product) and
    md_unpatchify_bwd (a gather: exact up to 2 u), with and without kept-token rows."""
    ops = _ops()
    T = (H // p) ** 2
    x = rnd((B, C, H, H), 1); sc = rnd((B,), 2) if scaled else None
    pt = torch.zeros(B * T, C * p * p, device=DEVICE)
    ops.patchify(dv(x), dv(sc), pt, p)
    ref = R.patchify(x, p, sc)
    within(pt, ref, 2 * U * ref.abs() + 1e-300, f"patchify B{B} C{C} p{p}")
    dp = rnd((B * T, C * p * p), 3); dx = torch.zeros(B, C, H, H, device=DEVICE)
    ops.patchify_bwd(dv(dp), dv(sc), dx, p)
    ref = R.patchify_bwd(dp, p, (B, C, H, H), sc)
    within(dx, ref, 2 * U * ref.abs() + 1e-300, f"patchify_bwd B{B} C{C} p{p}", teeth=False)
    for Tk in (T, T // 4):
        kr = None
        if Tk < T:
            kr = torch.stack([torch.randperm(T, generator=g(5))[:Tk] + b * T for b in range(B)]).reshape(-1).to(I32)
        dF = rnd((B, C, H, H), 4); dft = torch.zeros(B * Tk, p * p * C, device=DEVICE)
        ops.unpatchify_bwd(dv(dF), dv(kr), dft, p, Tk)
        ref = R.unpatchify_bwd(dF, p, Tk, kr)
        within(dft, ref, 2 * U * ref.abs() + 1e-300, f"unpatchify_bwd B{B} C{C} p{p} Tk{Tk}")


@pytest.mark.parametrize("n,dim", [(5, 512), (64, 256), (3, 1152)])
def test_timestep_embed_and_adjoint(n, dim):
    """md_timestep_embed / md_timestep_embed_bwd.  Bounds: the frequency exp(-ln(1e4) i / half) carries 16 u relative,
    so the angle a = t f carries 16 u |a| (1 + ln 1e4), and cos / sin of it 16 u (1 + |a| (1 + ln 1e4)); the adjoint sums
    half such terms times |dfreq| f."""
    ops = _ops()
    t = rnd((n,), 5, scale=3.0); out = torch.zeros(n, dim, device=DEVICE)
    ops.timestep_embed(dv(t), out)
    half = dim // 2
    fr = torch.exp(-math.log(10000.0) * torch.arange(half, dtype=D64) / half)
    a = (t.double()[:, None] * fr).abs() * (1 + math.log(10000.0))
    ref = R.timestep_embed(t, dim)
    within(out, ref, 16 * U * (1 + torch.cat([a, a], 1)), f"timestep embed n{n} dim{dim}")
    d = rnd((n, dim), 6); dt = torch.zeros(n, device=DEVICE)
    ops.timestep_embed_bwd(dv(d), dv(t), dt)
    ref = R.timestep_embed_bwd(d, t)
    terms = (d.double()[:, :half].abs() + d.double()[:, half:].abs()) * fr * (1 + a)
    within(dt, ref, 16 * U * half * terms.sum(1), f"timestep embed bwd n{n} dim{dim}", teeth=False)


def test_mean_tokens_and_caption_prepare():
    """md_mean_tokens_fwd (recursive summation over L tokens: L u sum|x| / L) and md_cond_prepare (fp16 captions times a
    0 / 1 keep flag: exact)."""
    ops = _ops()
    B, L, D = 3, 77, 256
    x = rnd((B * L, D), 1); out = torch.zeros(B, D, device=DEVICE)
    ops.mean_tokens_fwd(dv(x), out, B, L)
    ref = R.mean_tokens(x, B, L)
    within(out, ref, 2 * U * (L * x.double().abs().reshape(B, L, D).mean(1) + ref.abs()), "mean tokens")
    cap = rnd((B, 1, L, 1024), 4, torch.float16); keep = torch.tensor([1.0, 0.0, 1.0], dtype=torch.float64)
    ob = torch.full((B * L, 1024), 5.0, device=DEVICE); co = torch.zeros(B, 1, L, 1024, dtype=torch.float16, device=DEVICE)
    ops.cond_prepare(dv(cap).reshape(B, -1), dv(keep), ob, co)
    ref = cap.double().reshape(B, -1) * keep[:, None]
    exact(ob.reshape(B, -1), ref, "cond_prepare out")
    exact(co.reshape(B, -1), ref, "cond_prepare fp16 copy")


# ------------------------------------------------------------------------------------------------ pure copies
@pytest.mark.skipif(DRY, reason="pure copies: nothing on the CPU stands in for the kernel's store")
def test_casts_are_exact_copies():
    """cast_bf16, cast_transpose and cast_transpose_multi keep fp32 operands fp32 in this mode: bit-exact copies."""
    ops = _ops()
    v = rnd((100003,), 1); y = torch.zeros(100003, device=DEV)
    ops.cast_bf16(dv(v), y)
    exact(y, v, "cast_bf16")
    for shp in ((3, 100, 72), (1, 768, 2048), (1, 130, 8)):
        w = rnd(shp, 2); wb = torch.zeros(shp, device=DEV); wbt = torch.zeros(shp[0], shp[2], shp[1], device=DEV)
        ops.cast_transpose(dv(w), wb, wbt)
        exact(wb, w, f"cast_transpose {shp}"); exact(wbt, w.transpose(1, 2), f"cast_transpose^T {shp}")
    f = 96
    w = rnd((2 * f, 64), 3); wb = torch.zeros(2 * f, 64, device=DEV); wbt = torch.zeros(64, 2 * f, device=DEV)
    ops.cast_transpose(dv(w), wb, wbt, interleave_half=f)
    perm = R.interleaved_to_natural(f)
    exact(wb, w[perm], "interleaved cast"); exact(wbt, w[perm].t(), "interleaved cast^T")
    shapes = [(130, 70, 0, 1), (64, 64, 0, 1), (256, 48, 128, 1), (33, 200, 0, 0)]
    rows_, off, t = [], 0, 0
    for (r, c, half, need_t) in shapes:
        rows_.append([off, r, c, half, need_t, t, (c + 63) // 64, 0])
        t += ((c + 63) // 64) * ((r + 63) // 64)
        off += (r * c + 7) // 8 * 8
    flat = rnd((off,), 4); wb = torch.zeros(off, device=DEV); wbt = torch.zeros(off, device=DEV)
    ops.cast_transpose_multi(dv(flat), wb, wbt, dv(torch.tensor(rows_, dtype=torch.int64)), t)
    wbh, wbth = host(wb), host(wbt)
    for (o_, r, c, half, need_t, _, _, _) in rows_:
        w = flat[o_:o_ + r * c].view(r, c)
        if half:
            w = w[R.interleaved_to_natural(half)]
        assert torch.equal(wbh[o_:o_ + r * c].view(r, c), w.double())
        if need_t:
            assert torch.equal(wbth[o_:o_ + r * c].view(c, r), w.t().double())
