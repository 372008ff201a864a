"""Deterministic mode (md_set_deterministic) op by op, bf16 mode: every reduction that replaces a cross-block atomic by
workspace partials and a fixed-order second pass -- split-K GEMM (with row_interleave), ln_bwd / gate_bwd (one block per
sample, d gamma through the workspace), colsum, moe_gate_wgrad, sumsq, edm_loss_fwd.

For every case the mode is re-armed immediately before each call (which refills the workspace with the 0xFF NaN pattern,
so a reduction that reads a partial nobody wrote gives a non-finite result), the op runs twice and the outputs must be
bit-identical, agree with the CPU contract (oracle.emu_ops.EmuOps) at the bounds of tests/test_kernels_gpu.py, and the
reduced quantities must agree with the float64 references (tests/f64_reference.py) to fp32 reassociation: the
recursive-summation bound n u sum|t| over the n terms t of each sum (u = 2^-24), or for GEMM dot products of random
operands the quadrature form 8 sqrt(K) u sqrt(sum a_k^2 b_k^2).  A reduction that drops a partial of a split, slab or
sample is off by that partial -- orders of magnitude above these bounds even when the result stays bit-reproducible.

The library's minimum workspace is 1 MiB.  When partials do not fit, split-K falls back to an un-split reduction (still
deterministic); ln_bwd, colsum, moe_gate_wgrad and edm_loss_fwd refuse with "deterministic workspace too small".
md_sumsq needs grid * 4 bytes with its grid capped at 132 * 16 blocks (8448 bytes), so it always fits: its atomic
fallback cannot be reached at any size the library accepts.  md_edm_loss_fwd needs B * 4 bytes, which exceeds 1 MiB
from B = 262145 samples on; it used to take the atomics there and now returns the error like the others.
"""
import math

import pytest
import torch

from oracle.emu_ops import EmuOps
from tests import f64_reference as R
from tests.test_kernels_gpu import BF16, DEV, F32, I32, close, g, rnd

pytestmark = pytest.mark.gpu
U = 2.0 ** -24
MIN_WS = 1 << 20
WS = 256 << 20


def _ops():
    from micro_diffusion_b200.ops import CudaOps
    return CudaOps(DEV)


@pytest.fixture(autouse=True)
def _deterministic_mode_is_switched_off_again():
    """The switch is process-wide: whatever a test does, later tests of the same process run in the default mode."""
    from micro_diffusion_b200 import ops as O
    try:
        yield
    finally:
        _ops().set_deterministic(False)
        assert not O._DET_WORKSPACE, "deterministic workspace still registered"


def _arm(ops, nbytes):
    from micro_diffusion_b200 import ops as O
    ws = O._DET_WORKSPACE.get("ws")
    if ws is not None and ws.numel() != nbytes:   # set_deterministic keeps a larger buffer: release it first
        ops.set_deterministic(False)
    ops.set_deterministic(True, workspace_bytes=nbytes)


def twice(fn, tensors, ws=WS):
    """Run fn(ops, *device copies) twice in deterministic mode, re-armed before each run; assert every tensor argument
    comes out bit-identical; return the first run's tensors on the host."""
    ops = _ops()
    runs = []
    for _ in range(2):
        cu = [t.to(DEV).clone() if t is not None else None for t in tensors]
        _arm(ops, ws)
        fn(ops, *cu)
        torch.cuda.synchronize()
        runs.append([t.cpu() if t is not None else None for t in cu])
    for i, (a, b) in enumerate(zip(*runs)):
        if a is not None:
            assert torch.equal(a.view(torch.uint8) if a.is_floating_point() else a,
                               b.view(torch.uint8) if b.is_floating_point() else b), f"argument {i} differs between runs"
    return runs[0]


def emu(fn, tensors):
    cpu = [t.clone() if t is not None else None for t in tensors]
    fn(EmuOps("cpu"), *cpu)
    return cpu


def reassoc(got, ref, bound, what):
    got = got.double()
    assert torch.isfinite(got).all(), f"{what}: non-finite (a partial nobody wrote?)"
    ratio = float(((got - ref).abs() / bound.clamp_min(1e-300)).max())
    print(f"\n[{what}] error / reassociation bound = {ratio:.3f}", end="")
    assert ratio <= 1.0, f"{what}: {ratio:.2f}x the fp32 reassociation bound"


def _dot_bound(A, B, layout, K, C):
    return 8 * math.sqrt(K) * U * R.matmul(A.double() ** 2, B.double() ** 2, layout).sqrt() + 4 * U * C.abs()


# ------------------------------------------------------------------------------------------------ split-K GEMM
@pytest.mark.parametrize("layout,M,N,K,batch,splits", [
    (1, 768, 1024, 4000, 1, 4), (1, 768, 1024, 4000, 1, 0), (0, 300, 640, 1024, 1, 4), (0, 300, 640, 1024, 1, 0),
    (1, 256, 16, 4096, 1, 4), (1, 256, 200, 1000, 3, 0), (0, 640, 384, 1024, 3, 4),
    (0, 64, 1024, 16, 1, 4),      # one k-block: three of the four splits are empty and must write zero partials
])
def test_split_k_gemm(layout, M, N, K, batch, splits):
    A = rnd((batch, M, K) if layout == 0 else (batch, K, M), 1, BF16); B = rnd((batch, N, K) if layout == 0 else (batch, K, N), 2, BF16)
    C0 = rnd((batch, M, N), 6)
    if batch == 1:
        A, B, C0 = A[0], B[0], C0[0]

    def f(o, A, B, C):
        o.gemm(A, B, C, layout=layout, epi=3, splits=splits)
    cu = twice(f, [A, B, C0])
    cpu = emu(f, [A, B, C0])
    close(cu[2], cpu[2], "split-K gemm", 1e-4)
    ref = R.gemm(A, B, layout, accumulate=C0)
    reassoc(cu[2], ref, _dot_bound(A, B, layout, K, ref), f"split-K weight gradient {M}x{N}x{K} b{batch} s{splits}")


@pytest.mark.parametrize("M,f,K", [(512, 256, 128), (1000, 96, 192), (300, 2816, 64), (4096, 128, 256)])
def test_split_k_row_interleave(M, f, K):
    """The SwiGLU weight gradient: rows of the interleaved w1 | w2 stack land in parameter order."""
    du = rnd((M, 2 * f), 1, BF16); x = rnd((M, K), 2, BF16); g0 = rnd((2 * f, K), 3)

    def fn(o, du, x, gw):
        o.gemm(du, x, gw, layout=1, epi=3, splits=0, row_interleave=f)
    cu = twice(fn, [du, x, g0])
    cpu = emu(fn, [du, x, g0])
    close(cu[2], cpu[2], "interleaved wgrad", 1e-4)
    ref = g0.double().index_add(0, R.interleaved_to_natural(f), R.matmul(du, x, 1))
    bound = torch.zeros_like(ref).index_add(0, R.interleaved_to_natural(f), _dot_bound(du, x, 1, M, R.matmul(du, x, 1)))
    reassoc(cu[2], ref, bound + 4 * U * ref.abs(), f"interleaved wgrad M{M} f{f} K{K}")


def test_split_k_falls_back_when_partials_do_not_fit():
    """4 splits of a 512 x 512 output need 4 MiB of partials: with the 1 MiB minimum workspace the reduction runs
    un-split -- still correct, still bit-reproducible."""
    M = N = 512
    K = 2048
    assert 4 * M * N * 4 > MIN_WS
    A = rnd((K, M), 1, BF16); B = rnd((K, N), 2, BF16); C0 = rnd((M, N), 3)

    def f(o, A, B, C):
        o.gemm(A, B, C, layout=1, epi=3, splits=4)
    cu = twice(f, [A, B, C0], ws=MIN_WS)
    ref = R.gemm(A, B, 1, accumulate=C0)
    close(cu[2], emu(f, [A, B, C0])[2], "un-split fallback", 1e-4)
    reassoc(cu[2], ref, _dot_bound(A, B, 1, K, ref), "un-split fallback")


# ------------------------------------------------------------------------------------------------ LayerNorm / gate
@pytest.mark.parametrize("rows,D,T,xbf", [(256, 1024, 64, False), (154, 768, 77, False), (96, 128, 32, True),
                                          (40, 192, 8, False), (1024, 768, 256, False), (210, 512, 35, True)])
def test_ln_bwd(rows, D, T, xbf):
    ns = rows // T
    x = rnd((rows, D), 1, BF16 if xbf else F32, 2.0) + 0.5
    gamma = 1 + 0.1 * rnd((D,), 2); mod = rnd((ns, 6 * D), 3, scale=0.5)
    _, mu, rs, _ = R.ln_fwd(x, T=T)
    mean, rstd = mu.float(), rs.float()
    dy = rnd((rows, D), 4, BF16); dx0 = rnd((rows, D), 5); yn = rnd((rows, D), 6, BF16)
    dg0 = rnd((D,), 7); dmod0 = rnd((ns, 6 * D), 8)
    dyn = torch.zeros(rows, D, dtype=BF16)

    def b(o, dy, x, gamma, mod, mean, rstd, dx, dg, dmod, yn, dyn):
        o.ln_bwd(dy, x, mean, rstd, gamma=gamma, scale=mod[:, 3 * D:4 * D], T=T, dx=dx, dx_mode=0, dgamma=dg,
                 dshift=dmod[:, :D], dscale=dmod[:, 2 * D:3 * D], dy_next=dyn, y_next=yn, gate_next=mod[:, 5 * D:],
                 dgate_next=dmod[:, 4 * D:5 * D])
    args = [dy, x, gamma, mod, mean, rstd, dx0, dg0, dmod0, yn, dyn]
    cu = twice(b, args)
    cpu = emu(b, args)
    close(cu[6], cpu[6], "ln dx", 1e-4); close(cu[7], cpu[7], "dgamma", 1e-4); close(cu[8], cpu[8], "dmod", 1e-4)
    close(cu[10], cpu[10], "dy_next")
    # the reduced quantities against float64
    sc = mod[:, 3 * D:4 * D]
    rdx, rdg, rdsh, rdsc = R.ln_bwd(dy, x, gamma=gamma, scale=sc, T=T)
    xd = x.double()
    xh = (xd - mu[:, None]) * rs[:, None]
    xerr = 8 * U * (xd.abs() + mu.abs()[:, None]) * rs[:, None]       # xhat from the fp32 x, mean, rstd
    d = dy.double()
    s1 = 1 + R._per_row(sc, T, rows)
    tag = f"{rows}x{D} T{T}"
    reassoc(cu[8][:, :D], dmod0.double()[:, :D] + rdsh, 2 * U * (T * d.abs().reshape(ns, T, D).sum(1) + dmod0.double()[:, :D].abs()),
            f"dshift {tag}")
    reassoc(cu[8][:, 2 * D:3 * D], dmod0.double()[:, 2 * D:3 * D] + rdsc,
            (2 * U * T * (d * xh).abs().reshape(ns, T, D).sum(1) + (d.abs() * xerr).reshape(ns, T, D).sum(1))
            * gamma.double().abs() + 2 * U * (dmod0.double()[:, 2 * D:3 * D].abs() + rdsc.abs()), f"dscale {tag}")
    reassoc(cu[7], dg0.double() + rdg, 2 * U * rows * (d * xh * s1).abs().sum(0) + (d.abs() * xerr * s1.abs()).sum(0)
            + 2 * U * dg0.double().abs(), f"dgamma {tag}")
    # d gate of the fused tail: sum_t dx_total * y_next, dx_total from the kernel itself (its own rounding is in dy_next)
    dxt = cu[6].double()
    ref_dg = dmod0.double()[:, 4 * D:5 * D] + (dxt * yn.double()).reshape(ns, T, D).sum(1)
    reassoc(cu[8][:, 4 * D:5 * D], ref_dg, 2 * U * (T * (dxt * yn.double()).abs().reshape(ns, T, D).sum(1) + ref_dg.abs()),
            f"dgate_next {tag}")


@pytest.mark.parametrize("rows,D,T", [(192, 768, 64), (154, 256, 77), (1024, 1024, 256)])
def test_gate_bwd(rows, D, T):
    dres = rnd((rows, D), 1); y = rnd((rows, D), 2, BF16); mod = rnd((rows // T, 4 * D), 3)
    dy = torch.zeros(rows, D, dtype=BF16); dmod0 = rnd((rows // T, 4 * D), 4)

    def f(o, dres, y, mod, dy, dmod):
        o.gate_bwd(dres, dy, y=y, gate=mod[:, D:2 * D], dgate=dmod[:, 2 * D:3 * D], T=T)
    cu = twice(f, [dres, y, mod, dy, dmod0])
    cpu = emu(f, [dres, y, mod, dy, dmod0])
    close(cu[3], cpu[3], "dy"); close(cu[4], cpu[4], "dgate", 1e-4)
    _, rdg = R.gate_bwd(dres, y=y, T=T)
    ref = dmod0.double()[:, 2 * D:3 * D] + rdg
    t = (dres.double() * y.double()).abs().reshape(-1, T, D).sum(1)
    reassoc(cu[4][:, 2 * D:3 * D], ref, 2 * U * (T * t + ref.abs()), f"dgate {rows}x{D}")


# ------------------------------------------------------------------------------------------------ column / norm sums
@pytest.mark.parametrize("rows,N,dtype", [(700, 200, BF16), (4096, 1152, BF16), (231, 96, F32)])
def test_colsum(rows, N, dtype):
    x = rnd((rows, N), 1, dtype); c0 = rnd((N,), 2)
    cu = twice(lambda o, x, c: o.colsum(x, c), [x, c0])
    close(cu[1], emu(lambda o, x, c: o.colsum(x, c), [x, c0])[1], "colsum", 1e-4)
    ref = c0.double() + R.colsum(x)
    reassoc(cu[1], ref, 2 * U * (rows * x.double().abs().sum(0) + ref.abs()), f"colsum {rows}x{N}")


@pytest.mark.parametrize("n", [100003, 1 << 24])
def test_sumsq(n):
    """At n = 2^24 the grid is at its cap (2112 blocks): the partials still fit the 1 MiB minimum workspace."""
    v = rnd((n,), 1); s0 = torch.tensor([0.25])
    for ws in (WS, MIN_WS):
        cu = twice(lambda o, v, s: o.sumsq(v, s), [v, s0], ws=ws)
        ref = 0.25 + R.sumsq(v)
        reassoc(cu[1], ref.reshape(1), 2 * U * n * ref.reshape(1), f"sumsq n={n} ws={ws >> 20} MiB")


@pytest.mark.parametrize("B,T,E,cap,D", [(3, 64, 8, 2.0, 256), (2, 256, 8, 2.0, 768), (2, 100, 4, 1.0, 128),
                                          (3, 67, 8, 2.0, 1024), (1, 33, 16, 2.0, 512), (64, 256, 8, 2.0, 1024)])
def test_moe_gate_wgrad(B, T, E, cap, D):
    rows = B * T
    ds = rnd((rows, E), 1, scale=0.1); x = rnd((rows, D), 2, BF16); w0 = rnd((E, D), 3)
    cu = twice(lambda o, ds, x, w: o.moe_gate_wgrad(ds, x, w), [ds, x, w0])
    close(cu[2], emu(lambda o, ds, x, w: o.moe_gate_wgrad(ds, x, w), [ds, x, w0])[2], "dwg", 1e-3)
    ref = R.moe_gate_wgrad(ds, x, w0)
    reassoc(cu[2], ref, 2 * U * (rows * (ds.double().abs().t() @ x.double().abs()) + ref.abs()), f"dwg rows={rows} D{D}")


@pytest.mark.parametrize("B,C,H,p,masked,f16", [(4, 4, 32, 2, True, True), (2, 16, 16, 2, False, True), (3, 4, 64, 2, True, False)])
def test_edm_loss_fwd(B, C, H, p, masked, f16):
    T = (H // p) ** 2
    Tk = T // 4 if masked else T
    lat = rnd((B, C, H, H), 1, torch.float16 if f16 else F32, 0.8); eps = rnd((B, C, H, H), 2)
    xn, _, coef = R.edm_prepare(lat, eps, p, rnd=rnd((B,), 3), p_mean=-0.6, p_std=1.2, sigma_data=0.9)
    xn, coef = xn.float(), coef.float()
    kr = None
    if masked:
        kr = torch.stack([torch.randperm(T, generator=g(5))[:Tk] + b * T for b in range(B)]).reshape(-1).to(I32)
    ftok = rnd((B * Tk, C * p * p), 4)

    def f(o, ftok, kr, lat, xn, coef, ps, loss):
        o.edm_loss_fwd(ftok, kr, lat, xn, coef, ps, loss, p, Tk)
    args = [ftok, kr, lat, xn, coef, torch.zeros(B), torch.tensor([0.5])]
    cu = twice(f, args)
    cpu = emu(f, args)
    close(cu[5], cpu[5], "per-sample loss", 1e-5); close(cu[6], cpu[6], "loss", 1e-5)
    rps, rloss = R.edm_loss_fwd(ftok, lat, xn, coef, p, Tk, kr)
    n = Tk * C * p * p
    # every term is a weighted square (>= 0): sum|t| is the sum itself; the residual's own rounding adds 8 u |terms|
    reassoc(cu[5], rps, (2 * n + 16) * U * rps, f"per-sample loss B{B}")
    reassoc(cu[6], 0.5 + rloss.reshape(1), (2 * n + 16 + 2 * B) * U * (0.5 + rloss.reshape(1)), f"loss B{B}")


# ------------------------------------------------------------------------------------------------ workspace too small
def _too_small(call):
    from micro_diffusion_b200._lib import MicroditLibraryError
    ops = _ops()
    _arm(ops, MIN_WS)
    with pytest.raises(MicroditLibraryError, match="deterministic workspace too small"):
        call(ops)
    torch.cuda.synchronize()


def test_ln_bwd_refuses_a_workspace_too_small():
    T, ns, D = 4, 300, 1024                   # d gamma partials: ns * D * 4 = 1.2 MB
    assert ns * D * 4 > MIN_WS
    rows = T * ns
    x = torch.randn(rows, D, device=DEV); dy = torch.randn(rows, D, device=DEV).to(BF16)
    mean = torch.zeros(rows, device=DEV); rstd = torch.ones(rows, device=DEV)
    _too_small(lambda o: o.ln_bwd(dy, x, mean, rstd, T=T, dx=torch.zeros_like(x), dgamma=torch.zeros(D, device=DEV)))


def test_colsum_refuses_a_workspace_too_small():
    rows, N = 256 * 300, 1024                 # slab partials: 300 * N * 4 = 1.2 MB
    assert math.ceil(rows / 256) * N * 4 > MIN_WS
    x = torch.ones(rows, N, dtype=BF16, device=DEV)
    _too_small(lambda o: o.colsum(x, torch.zeros(N, device=DEV)))


def test_moe_gate_wgrad_refuses_a_workspace_too_small():
    E, D = 8, 1024
    rows = 264 * 64                           # 264 slabs of 64 rows: the grid cap; partials 264 * E * D * 4 = 8.6 MB
    assert 264 * E * D * 4 > MIN_WS
    ds = torch.zeros(rows, E, device=DEV); x = torch.zeros(rows, D, dtype=BF16, device=DEV)
    _too_small(lambda o: o.moe_gate_wgrad(ds, x, torch.zeros(E, D, device=DEV)))


def test_edm_loss_fwd_refuses_a_workspace_too_small():
    B = (MIN_WS // 4) + 1                     # one partial per sample: B * 4 bytes > 1 MiB
    lat = torch.zeros(B, 1, 1, 1, device=DEV); ftok = torch.zeros(B, 1, device=DEV)
    coef = torch.ones(6, B, device=DEV)
    _too_small(lambda o: o.edm_loss_fwd(ftok, None, lat, lat, coef, torch.zeros(B, device=DEV), torch.zeros(1, device=DEV),
                                        1, 1))
