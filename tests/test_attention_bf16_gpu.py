"""Every bf16 attention kernel element by element against softmax attention in float64, and row by row against the
systematic errors an indexing or masking bug leaves.

The inputs q, k, v, dO are bf16, so every product is exact; the references are tests/f64_reference.py's attn_fwd /
attn_bwd.  The backward gets the exact o rounded to bf16 and the exact lse rounded to fp32, as it would from a forward
that met its contract.  eps = 2^-8 is the bf16 unit roundoff: bf16 carries 8 significant bits, so a rounding is off by
at most 2^-8 relative (at a mantissa just above a power of two), not 2^-9.

Element bounds.  The fp32 arithmetic of the kernels (scores, exp2, the key / query sums, delta) is the quadrature model
of md_attn_*_f32 (_attn_bounds in tests/test_high_precision_ops_gpu.py).  The bf16 contract adds its rounding points,
each independent, zero-mean and at most eps relative, summed in quadrature with the same tail factor 8:

* forward: P is rounded for the PV product: 8 eps sqrt(sum_k p_k^2 v_k^2).  o is stored in bf16: eps |o|.  lse stays
  fp32, so its bound is the fp32 one.
* backward: P is rounded for dV: 8 eps sqrt(sum_q p_qk^2 dO_q^2); dS = P (dP - delta) is rounded for dQ and dK:
  8 eps sqrt(sum_k dS_qk^2 k_k^2) / sqrt(hd) and 8 eps sqrt(sum_q dS_qk^2 q_q^2) / sqrt(hd).  delta = sum dO o read from
  the bf16 o is off by dd_q = sum dO_q (bf16(o_q) - o_q), which is known exactly: it moves dS by -P dd and dq / dk by
  e_dq = -dd (P K) / sqrt(hd) and e_dk = -(P dd)^T Q / sqrt(hd); the bound adds |e|.  (The fused few-key kernels take
  delta as sum_k P dP instead, which has no such term; the bound covers both.)  dq, dk, dv are stored in bf16: eps |x|.

Row statistic.  Rounding errors are zero-mean; indexing and masking bugs are not.  For every (sample, head, query) row
of o and dq and every key row of dk and dv, c = <got - ref, ref> must stay within KSIG = 6 standard deviations of what
the rounding points predict for it, plus the projection of the fp32 bound and of e (both taken as worst cases).  A
bf16 rounding with a log-uniform mantissa m has relative error of variance 2^-14 E[1/m^2] / 12 = 2^-14 3 / (96 ln 2)
(VREL).  Hence var <err, o> = VREL (sum_k p_k^2 (v_k . o)^2 + sum_d o_d^4) and likewise for the backward
(sum_k dS_qk^2 (k_k . dq)^2 / hd for dq, sum_q dS_qk^2 (q_q . dk)^2 / hd for dk, sum_q p_qk^2 (dO_q . dv)^2 for dv, plus
the store).  One rounding alone cannot exceed 2^-8 / sqrt(VREL) = 2.4 deviations, so 6 is never reached by rounding,
while a padded key let into the softmax shifts a whole row by ~1/Tk: an element bound on a bf16 output cannot see
that, this statistic does.

Every case runs each entry point (ops.attn_tc = None / True / False), asserts which C entry point ran and, from a
torch.profiler trace, which kernel instantiations ran (route() mirrors the dispatch table of csrc/attn.cu and
csrc/attn_wgmma.cu); test_matrix_reaches_every_kernel checks that SHAPES x MODES reaches all of them.  Operands use
the engine's layouts (q a column slice of a wider qkv buffer, k / v the halves of a kv buffer); every output starts
as a sentinel, and the columns around the written slices must keep it.  Each case prints its worst error / bound
and its worst row |z|.

MD_TEST_DRYRUN=1 runs the same cases on oracle.emu_ops.EmuOps("cpu") (the bf16 contract with its rounding points):
the references, the model and the statistic are exercised without a GPU.  The entry-point and kernel assertions and
the rejection tests are skipped there.  tests/test_attention_bf16_model_cpu.py runs these cases on emulations with
one injected fault each, to show that the bounds catch them.
"""
import math
import os
import re
import time

import pytest
import torch

from tests import f64_reference as R
from tests.test_high_precision_ops_gpu import _attn_bounds

pytestmark = pytest.mark.gpu
DRY = bool(os.environ.get("MD_TEST_DRYRUN"))
DEV = "cuda:0"
BF16 = torch.bfloat16
EPS = 2.0 ** -8
VREL = 2.0 ** -14 * 3 / (96 * math.log(2.0))
KSIG = 6.0
QUAD = 8.0
SENT = -768.0      # exact in bf16 and far outside any output here
PAD = 8            # sentinel columns on each side of o (16 bytes: the slice stays aligned)
MODES = (None, True, False)


# ------------------------------------------------------------------------------------------------ cases and model
class Case:
    """Seeded bf16 operands of one shape, the float64 results, their element bounds and the row-statistic terms."""

    def __init__(self, B, H, Tq, Tk, hd, seed=1):
        self.B, self.H, self.Tq, self.Tk, self.hd = B, H, Tq, Tk, hd
        hsz = self.hsz = H * hd
        g = torch.Generator().manual_seed(seed)
        self.qkv = torch.randn(B * Tq, 3 * hsz + 64, generator=g).to(BF16)   # q = columns [hsz, 2 hsz)
        self.kv = torch.randn(B * Tk, 2 * hsz, generator=g).to(BF16)         # k | v
        self.do = torch.randn(B * Tq, hsz, generator=g).to(BF16)
        q, k, v = self.q, self.kv[:, :hsz], self.kv[:, hsz:]
        self.o, self.lse = R.attn_fwd(q, k, v, B, H, Tq, Tk, hd)
        self.o_in, self.lse_in = self.o.float().to(BF16), self.lse.float()   # what the backward is given
        self.dq, self.dk, self.dv = R.attn_bwd(self.do, q, k, v, B, H, Tq, Tk, hd)
        self._model(q, k, v)

    @property
    def q(self):
        return self.qkv[:, self.hsz:2 * self.hsz]

    def tag(self):
        return f"B{self.B} H{self.H} {self.Tq}/{self.Tk} hd{self.hd}"

    def _model(self, q, k, v):
        B, H, Tq, Tk, hd = self.B, self.H, self.Tq, self.Tk, self.hd
        bo32, bl32, bdq32, bdk32, bdv32 = _attn_bounds(q, k, v, self.do, B, H, Tq, Tk, hd)
        hq, hk = (lambda t: R._heads(t, B, Tq, H, hd)), (lambda t: R._heads(t, B, Tk, H, hd))
        qh, kh, vh, doh = hq(q), hk(k), hk(v), hq(self.do)
        sc = 1.0 / math.sqrt(hd)
        P = torch.softmax(qh @ kh.mT * sc, -1)
        o, dq, dk, dv = hq(self.o), hq(self.dq), hk(self.dk), hk(self.dv)
        ds = P * (doh @ vh.mT - (doh * o).sum(-1, keepdim=True))
        dd = (doh * (hq(self.o_in) - o)).sum(-1, keepdim=True)
        e_dq, e_dk = -sc * dd * (P @ kh), -sc * (P * dd).mT @ qh
        P2, ds2 = P ** 2, ds ** 2

        def store(pre, ref):
            return pre + EPS * (ref.abs() + pre)

        bound = {"o": store(hq(bo32) + QUAD * EPS * (P2 @ vh ** 2).sqrt(), o),
                 "dq": store(hq(bdq32) + QUAD * EPS * sc * (ds2 @ kh ** 2).sqrt() + e_dq.abs(), dq),
                 "dk": store(hk(bdk32) + QUAD * EPS * sc * (ds2.mT @ qh ** 2).sqrt() + e_dk.abs(), dk),
                 "dv": store(hk(bdv32) + QUAD * EPS * (P2.mT @ doh ** 2).sqrt(), dv)}
        self.bound = {n: R._unheads(b) for n, b in bound.items()}
        self.bound["lse"] = bl32

        def row(ref, mix, b32, e=None):
            det = (b32 * ref.abs()).sum(-1)
            if e is not None:
                det = det + (e * ref).sum(-1).abs()
            return VREL * (mix + (ref ** 4).sum(-1)), det

        self.row = {"o": row(o, (P2 * (o @ vh.mT) ** 2).sum(-1), hq(bo32)),
                    "dq": row(dq, sc ** 2 * (ds2 * (dq @ kh.mT) ** 2).sum(-1), hq(bdq32), e_dq),
                    "dk": row(dk, sc ** 2 * (ds2 * (qh @ dk.mT) ** 2).sum(-2), hk(bdk32), e_dk),
                    "dv": row(dv, (P2 * (doh @ dv.mT) ** 2).sum(-2), hk(bdv32))}


def _dev(ops):
    return "cpu" if getattr(ops, "is_emulation", False) else DEV


def run_fwd(ops, c):
    """o (inside a sentinel-filled buffer with PAD columns either side) and lse."""
    dev, hsz = _dev(ops), c.hsz
    qkv, kv = c.qkv.to(dev), c.kv.to(dev)
    obuf = torch.full((c.B * c.Tq, hsz + 2 * PAD), SENT, dtype=BF16, device=dev)
    lse = torch.full((c.B, c.H, c.Tq), SENT, device=dev)
    ops.attn_fwd(qkv[:, hsz:2 * hsz], kv[:, :hsz], kv[:, hsz:], obuf[:, PAD:PAD + hsz], lse, c.B, c.H, c.Tq, c.Tk, c.hd)
    return obuf.cpu(), lse.cpu()


def run_bwd(ops, c):
    """dq (the q columns of a sentinel-filled dqkv buffer) and dk | dv (a dkv buffer with PAD spare columns)."""
    dev, hsz = _dev(ops), c.hsz
    qkv, kv = c.qkv.to(dev), c.kv.to(dev)
    dqkv = torch.full(c.qkv.shape, SENT, dtype=BF16, device=dev)
    dkv = torch.full((c.B * c.Tk, 2 * hsz + PAD), SENT, dtype=BF16, device=dev)
    delta = torch.full((c.B, c.H, c.Tq), float("nan"), device=dev)
    ops.attn_bwd(c.do.to(dev), qkv[:, hsz:2 * hsz], kv[:, :hsz], kv[:, hsz:], c.o_in.to(dev), c.lse_in.to(dev), delta,
                 dqkv[:, hsz:2 * hsz], dkv[:, :hsz], dkv[:, hsz:2 * hsz], c.B, c.H, c.Tq, c.Tk, c.hd)
    return dqkv.cpu(), dkv.cpu()


def _elem(got, ref, bound):
    r = (got.double() - ref).abs() / bound.clamp_min(1e-300)
    return float(torch.nan_to_num(r, nan=math.inf).max()) if r.numel() else 0.0


def _rowz(got, ref, var, det):
    """max over rows of (|<got - ref, ref>| - det) / sqrt(var), in units of KSIG."""
    num = ((got.double() - ref) * ref).sum(-1).abs()
    z = (num - det).clamp_min(0) / var.sqrt().clamp_min(1e-300)
    return float(torch.nan_to_num(z, nan=math.inf).max()) / KSIG


def _kept(buf, cols):
    keep = torch.ones(buf.shape[1], dtype=torch.bool)
    keep[cols] = False
    return 0.0 if bool((buf[:, keep].float() == SENT).all()) else math.inf


def metrics(c, fwd, bwd):
    """{check: worst error as a fraction of what it may be}: <= 1 passes."""
    B, H, Tq, Tk, hd, hsz = c.B, c.H, c.Tq, c.Tk, c.hd, c.hsz
    hq, hk = (lambda t: R._heads(t, B, Tq, H, hd)), (lambda t: R._heads(t, B, Tk, H, hd))
    out = {}
    if fwd is not None:
        obuf, lse = fwd
        o = obuf[:, PAD:PAD + hsz]
        out["o"] = _elem(o, c.o, c.bound["o"])
        out["o row"] = _rowz(hq(o), hq(c.o), *c.row["o"])
        out["lse"] = _elem(lse, c.lse, c.bound["lse"])
        out["o pad"] = _kept(obuf, slice(PAD, PAD + hsz))
    if bwd is not None:
        dqkv, dkv = bwd
        for n, got, ref, h in (("dq", dqkv[:, hsz:2 * hsz], c.dq, hq), ("dk", dkv[:, :hsz], c.dk, hk),
                               ("dv", dkv[:, hsz:2 * hsz], c.dv, hk)):
            out[n] = _elem(got, ref, c.bound[n])
            out[n + " row"] = _rowz(h(got), h(ref), *c.row[n])
        out["dqkv pad"] = _kept(dqkv, slice(hsz, 2 * hsz))
        out["dkv pad"] = _kept(dkv, slice(0, 2 * hsz))
    return out


def report(what, m):
    worst = {n: v for n, v in m.items() if "pad" not in n}
    print(f"\n[{what}] " + " ".join(f"{n} {v * (KSIG if 'row' in n else 1):.3g}" for n, v in worst.items()), end="")


# ------------------------------------------------------------------------------------------------ routes
def _fwd_mma(hd, Tk):
    return f"attn_fwd_kernel<{hd}, {80 if 64 < Tk <= 80 else 64}>"


def route(mode, Tq, Tk, hd):
    """(forward entry point, its kernels, backward entry point, its kernels) for ops.attn_tc = mode."""
    tc_fwd = (hd == 64 and Tk <= 256) or hd == 128
    wg_fwd = "attn_fwd_wgmma128_kernel" if hd == 128 else "attn_fwd_wgmma_kernel"
    if mode is False:
        fe, fk = "md_attn_fwd_mma", {_fwd_mma(hd, Tk)}
    else:
        fe = "md_attn_fwd_tc" if (mode and tc_fwd) else "md_attn_fwd"
        fk = {wg_fwd if tc_fwd else _fwd_mma(hd, Tk)}
    be = "md_attn_bwd_mma" if mode is False else ("md_attn_bwd_tc" if (mode and hd == 64) else "md_attn_bwd")
    if hd == 64 and (mode is True or (mode is None and Tk > 128)):
        bk = {"attn_delta_kernel<64>", "attn_bwd_wgmma_kernel"}
    elif hd != 128 and Tk <= 80:
        bk = {f"attn_bwd_{'small' if Tq <= 64 else 'cross'}_kernel<{hd}, {80 if Tk > 64 else 64}>"}
    else:
        bk = {f"attn_delta_kernel<{hd}>", f"attn_bwd_dkdv_kernel<{hd}>", f"attn_bwd_dq_kernel<{hd}>"}
    return fe, fk, be, bk


ALL_KERNELS = {"attn_fwd_wgmma_kernel", "attn_fwd_wgmma128_kernel", "attn_bwd_wgmma_kernel"} \
    | {f"attn_fwd_kernel<{hd}, {kt}>" for hd in (32, 64, 128) for kt in (64, 80)} \
    | {f"attn_bwd_{kind}_kernel<{hd}, {kt}>" for kind in ("small", "cross") for hd in (32, 64) for kt in (64, 80)} \
    | {f"attn_{kind}_kernel<{hd}>" for kind in ("delta", "bwd_dkdv", "bwd_dq") for hd in (32, 64, 128)}


def _patterns(kid):
    """A kernel id as it shows in a trace: demangled (attn_fwd_kernel<64, 80>) or mangled (attn_fwd_kernelILi64ELi80EE)."""
    m = re.fullmatch(r"(\w+)<([\d, ]+)>", kid)
    if not m:
        return (kid + "(", kid + "P", kid + "E", kid + "v")
    args = [a.strip() for a in m.group(2).split(",")]
    return (kid, m.group(1) + "I" + "".join(f"Li{a}E" for a in args) + "E")


def _kernel_ids(names):
    ids, unknown = set(), []
    for n in names:
        hit = {kid for kid in ALL_KERNELS if any(p in n for p in _patterns(kid))}
        ids |= hit
        if not hit:
            unknown.append(n)
    return ids, unknown


def _ops(mode):
    if DRY:
        from oracle.emu_ops import EmuOps
        return EmuOps("cpu")
    from micro_diffusion_b200.ops import CudaOps
    ops = CudaOps(torch.device(DEV))
    ops.attn_tc = mode
    return ops


def _traced(ops, fn, want, attempts=4, keep="attn", ids=_kernel_ids):
    """fn()'s result, the C entry points it called and the kernels it launched whose names contain one of `keep`
    (a string or a tuple of strings); ids(names) maps them to (kernel ids, unrecognised names).  A short profiler
    session now and then loses kernel records of a call that did run (a few of ~500 sessions per run, sometimes two in
    a row).  fn has no effect beyond its fresh outputs, so a session whose kernels are not `want` is traced again, up
    to `attempts` times, and printed with what it did record; a dispatch that really differs fails every attempt."""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    orig = ops._call
    for attempt in range(attempts):
        calls = []

        def rec(name, *a, **k):
            calls.append(name)
            return orig(name, *a, **k)
        ops._call = rec
        try:
            with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
                out = fn()
                torch.cuda.synchronize()
        finally:
            ops._call = orig
        # the raw kernel records, not prof.events(): nothing here needs them matched to the CPU ops that launched them
        device = [e.name() for e in prof.profiler.kineto_results.events() if e.device_type() == DeviceType.CUDA]
        names = {n for n in device if any(k in n for k in ((keep,) if isinstance(keep, str) else keep))}
        if ids(names) == (want, []) or attempt == attempts - 1:
            return out, calls, names
        print(f"\n[trace {attempt}: {calls}, {sorted(names)} among {len(device)} device records]", end="")
        time.sleep(0.2)


# ------------------------------------------------------------------------------------------------ the matrix
# (B, H, Tq, Tk, hd).  Every key count of the tile edges (1 16 33 63 64 65 77 80 81 127 128 129 200 255 256 257 513
# 1000 1024) and query count (1 50 63 64 65 130 256 1000 1024); grids above 132 CTAs; H * hd = 2048 (the delta pass's
# limit) at hd 32, 64 and 128; the MicroDiT_XL_2 shapes at res 256 / 512 (64 / 256 / 1024 tokens, 77 caption tokens,
# head_dim 64, 16 heads at the widest block); and every shape of the relative-L2 checks in tests/test_attn_tc_gpu.py and
# tests/test_hd128_gpu.py, here at every entry point and against float64.
SHAPES_64 = [(2, 3, 128, 128, 64), (1, 1, 128, 64, 64), (2, 2, 256, 256, 64), (3, 4, 64, 64, 64), (2, 5, 256, 77, 64),
             (2, 3, 100, 200, 64), (1, 2, 64, 77, 64), (2, 2, 1024, 77, 64), (2, 3, 64, 64, 64), (2, 2, 77, 77, 64),
             (3, 2, 50, 33, 64), (40, 8, 256, 256, 64), (64, 16, 64, 77, 64), (37, 6, 130, 16, 64), (1, 1, 128, 128, 64),
             (1, 2, 512, 77, 64), (20, 8, 256, 256, 64), (40, 16, 64, 64, 64), (2, 2, 300, 144, 64),
             (1, 2, 1024, 1024, 64), (2, 3, 300, 1000, 64), (3, 2, 128, 513, 64),
             (2, 3, 1, 1, 64), (2, 2, 63, 1, 64), (2, 2, 63, 80, 64), (2, 3, 65, 81, 64), (2, 2, 64, 127, 64),
             (2, 2, 130, 129, 64), (2, 2, 1, 255, 64), (1, 2, 64, 257, 64), (2, 2, 1000, 65, 64), (1, 32, 64, 200, 64),
             (2, 16, 64, 64, 64), (2, 16, 256, 256, 64), (1, 16, 1024, 1024, 64), (2, 16, 64, 77, 64),
             (2, 16, 256, 77, 64), (1, 16, 1024, 77, 64)]
SHAPES_128 = [(2, 2, 64, 64, 128), (2, 3, 64, 77, 128), (2, 2, 64, 120, 128), (2, 2, 256, 256, 128),
              (1, 2, 1024, 1024, 128), (2, 3, 256, 77, 128), (1, 2, 1024, 77, 128), (2, 2, 256, 120, 128),
              (2, 2, 1024, 256, 128), (3, 2, 130, 33, 128), (3, 2, 50, 200, 128), (2, 3, 100, 1000, 128),
              (40, 8, 64, 77, 128), (64, 16, 64, 64, 128), (4, 16, 256, 256, 128), (1, 1, 64, 1024, 128),
              (1, 2, 1, 1, 128), (2, 2, 63, 81, 128), (1, 2, 65, 255, 128), (1, 2, 1, 257, 128), (1, 1, 1000, 513, 128),
              (2, 2, 64, 16, 128), (2, 1, 1024, 1, 128), (1, 16, 130, 200, 128)]
SHAPES_32 = [(2, 2, 1, 1, 32), (2, 2, 63, 63, 32), (2, 2, 65, 65, 32), (2, 2, 64, 80, 32), (2, 2, 50, 16, 32),
             (2, 2, 130, 64, 32), (2, 2, 63, 81, 32), (1, 2, 1000, 127, 32), (2, 2, 65, 200, 32), (1, 64, 64, 129, 32),
             (40, 8, 256, 77, 32)]
SHAPES = SHAPES_64 + SHAPES_128 + SHAPES_32


def test_matrix_reaches_every_kernel():
    """The union of ROUTES over SHAPES x MODES is every bf16 attention kernel instantiation; each case below asserts
    that its route is what ran, so together they reach all of them."""
    reached = set()
    for (B, H, Tq, Tk, hd) in SHAPES:
        for mode in MODES:
            _, fk, _, bk = route(mode, Tq, Tk, hd)
            reached |= fk | bk
    assert reached == ALL_KERNELS, (sorted(ALL_KERNELS - reached), sorted(reached - ALL_KERNELS))
    assert all(_kernel_ids([f"void md::{k}(int)"])[0] == {k} for k in ALL_KERNELS)


@pytest.mark.parametrize("B,H,Tq,Tk,hd", SHAPES)
def test_bf16_attention_within_error_model(B, H, Tq, Tk, hd):
    c = Case(B, H, Tq, Tk, hd)
    failed = []
    for mode in ((None,) if DRY else MODES):
        ops = _ops(mode)
        if DRY:
            fwd, bwd = run_fwd(ops, c), run_bwd(ops, c)
        else:
            fe, fk, be, bk = route(mode, Tq, Tk, hd)
            fwd, calls, names = _traced(ops, lambda: run_fwd(ops, c), fk)
            ids, unknown = _kernel_ids(names)
            assert calls == [fe] and ids == fk and not unknown, (mode, calls, sorted(names), fe, fk)
            bwd, calls, names = _traced(ops, lambda: run_bwd(ops, c), bk)
            ids, unknown = _kernel_ids(names)
            assert calls == [be] and ids == bk and not unknown, (mode, calls, sorted(names), be, bk)
        m = metrics(c, fwd, bwd)
        report(f"{c.tag()} attn_tc={mode}", m)
        failed += [(mode, n, round(v, 3)) for n, v in m.items() if not v <= 1.0]
    assert not failed, failed


# ------------------------------------------------------------------------------------------------ argument checks
def _lib_error():
    from micro_diffusion_b200._lib import MicroditLibraryError
    return MicroditLibraryError


@pytest.mark.skipif(DRY, reason="argument checks of the C entry points")
@pytest.mark.parametrize("mode", MODES)
def test_misaligned_operands_are_rejected(mode):
    """Every kernel moves head rows in 16-byte pieces: a q (or o) view that is only 8-byte aligned is MD_ERR_INVALID at
    every entry point (md_attn_fwd / _tc / _mma, md_attn_bwd / _tc / _mma), before anything launches."""
    B, H, Tq, Tk, hd = 1, 2, 64, 200, 64
    hsz = H * hd
    qkv = torch.zeros(B * Tq, 3 * hsz + 64, dtype=BF16, device=DEV)
    kv = torch.zeros(B * Tk, 2 * hsz, dtype=BF16, device=DEV)
    q8 = qkv[:, 4:4 + hsz]                        # element offset 4: 8-byte aligned, pitch a multiple of 8
    o = torch.zeros(B * Tq, hsz, dtype=BF16, device=DEV); lse = torch.zeros(B, H, Tq, device=DEV)
    dq = torch.zeros_like(o); dkv = torch.zeros_like(kv)
    ops = _ops(mode)
    err = _lib_error()
    with pytest.raises(err, match="16-byte aligned"):
        ops.attn_fwd(q8, kv[:, :hsz], kv[:, hsz:], o, lse, B, H, Tq, Tk, hd)
    for qv, ov in ((q8, o), (qkv[:, hsz:2 * hsz], qkv[:, 4:4 + hsz])):
        with pytest.raises(err, match="16-byte aligned"):
            ops.attn_bwd(o, qv, kv[:, :hsz], kv[:, hsz:], ov, lse, None, dq, dkv[:, :hsz], dkv[:, hsz:], B, H, Tq, Tk, hd)
    torch.cuda.synchronize()


@pytest.mark.skipif(DRY, reason="argument checks of the C entry points")
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("H,hd", [(33, 64), (17, 128), (65, 32)])
def test_backward_beyond_2048_columns_is_rejected(mode, H, hd):
    """The delta pass holds one token row of every head in a warp (H * hd <= 2048).  Every backward route that runs it
    -- the generic split and the wgmma backward -- returns MD_ERR_UNSUPPORTED beyond that instead of leaving the last
    heads' delta unwritten."""
    B, Tq, Tk = 1, 64, 200
    hsz = H * hd
    x = torch.zeros(B * Tq, hsz, dtype=BF16, device=DEV)
    kv = torch.zeros(B * Tk, 2 * hsz, dtype=BF16, device=DEV); dkv = torch.zeros_like(kv)
    lse = torch.zeros(B, H, Tq, device=DEV)
    with pytest.raises(_lib_error(), match="H\\*hd must be <= 2048"):
        _ops(mode).attn_bwd(x, x, kv[:, :hsz], kv[:, hsz:], x, lse, None, torch.zeros_like(x), dkv[:, :hsz], dkv[:, hsz:],
                            B, H, Tq, Tk, hd)
    torch.cuda.synchronize()
