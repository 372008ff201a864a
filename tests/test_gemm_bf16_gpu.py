"""Every bf16 GEMM epilogue of md_gemm_bf16 element by element against float64 (tests/f64_reference.py), on every path
through the kernel: the four instantiations gemm_wgmma_kernel<BLOCK_N, kMN> (BLOCK_N 128 / 256, NT / TN), the interior
epilogue, the guarded epilogue with pair accesses and with scalar accesses, and the deterministic split-K reduction.

Error model.  The operands are bf16, so every product a_k b_k is exact in fp32.  u = 2^-24, S = sqrt(sum_k a_k^2 b_k^2),
v = fl(fl(alpha acc) + bias) is the fp32 value every tail starts from, v_ref its exact value.  The fp32 accumulation is
the quadrature model of the high-precision tests (tests/test_high_precision_ops_gpu.py) at depth K:

    delta_v = |alpha| 8 sqrt(K) u S + u (|alpha acc| + |v|)

(the second term: the alpha scale and the bias add, one rounding each).

* bf16 outputs of v -- EPI_BF16, the ACT_DUAL pre-activation, the RESID side copy C2 and the SwiGLU u -- must lie in
  the rounding bracket [rn(v_ref - delta_v), rn(v_ref + delta_v)] (rn: round to nearest even in bf16).  delta_v is far
  below half a bf16 ulp, so the bracket is one value for most elements and the check is exact there.  Each case
  reports the share of single-value brackets and asserts SINGLE_FLOOR = 0.85.  The share depends only on the
  reference and delta_v, not on the kernel; the smallest the MD_TEST_DRYRUN run of this matrix gives is 0.898 (ACT_GRAD
  at K = 4000).  A store that rounds toward zero misses about half of the single-value brackets.
* Math tails are taken from the kernel's own stored bf16 inputs, because that is what the kernel computes from: the
  ACT_DUAL output from the stored pre-activation, SwiGLU h from the stored u (act_dual_tail and swiglu_tail round
  first).  The gradient tails take aux / u as given and v with delta_v.  Each output must lie in [rn(y - e), rn(y + e)]
  with y the float64 result and e the fp32 evaluation error below.  ulp errors are turned into relative ones with
  1 ulp <= 2^-23 |x| = 2u |x|.  Written sources only:
    - erf by Abramowitz-Stegun 7.1.26: |error| <= 1.5e-7 (absolute);
    - __expf(x): at most 2 + floor(|1.173 x|) ulp; __fdividef(x, y): 2 ulp for |y| in [2^-126, 2^126] (CUDA C++
      Programming Guide, intrinsic functions);
    - every other fp32 operation: one rounding, u relative to its result.
  Carried through the formulas of csrc/gemm_wgmma.cu (first order; every e is multiplied by 1 + 2^-10 for the products
  of two such terms):
    - sigmoid s = 1 / (1 + E), E = __expf(-a): eps_s = E / (1 + E) eps_E + u + 4u, eps_E = (2 + floor(1.173 |a|)) 2u.
    - SwiGLU h = (a s) b: e = |h| (eps_s + 2u).
    - SwiGLU' du2 = (d u1) s: e = |du2| (eps_s + 2u) + delta_v |u1 s|; du1 = (d u2) (s t), t = fma(a, 1 - s, 1):
      err(1 - s) = s eps_s + u |1 - s|, err t = |a| err(1 - s) + u |t|, err(s t) = |t| s eps_s + s err t + u |s t|,
      e = |d u2| (err(s t) + 2u |s t|) + delta_v |u2 s t|.
    - gelu-erf: z = |x| / sqrt2, q = fma(p, z, 1) (2u), t = __fdividef(1, q) (eps_t = 2u + 4u), the Horner polynomial
      P(t) t = sum_i a_i t^i with 4 fma roundings and the error of t: err(P t) = 6u (Q + Q1), Q = sum |a_i| t^i,
      Q1 = sum i |a_i| t^i.  zz = z z (3u), E = __expf(-zz): eps_E = (2 + floor(1.173 zz)) 2u + 3u zz.
      err erf = 1.5e-7 + E err(P t) + |P t| E (eps_E + u) + u.  gelu = (x / 2)(1 + erf): e = |x| / 2 (err erf + 2u)
      + u |gelu|.  gelu' = (1 + erf) / 2 + fma(x / sqrt(2 pi), E, .): e = (err erf + 2u) / 2 + |x E| / sqrt(2 pi)
      (eps_E + 2u) + u |gelu'|.
    - gelu-tanh: w = 2 k0 fma(k1 x, x x, x) (6u, the constants' own rounding included), E = __expf(w): eps_E =
      (2 + floor(1.173 |w|)) 2u + 6u |w|; d = __fdividef(2, E + 1): eps_d = E / (1 + E) eps_E + u + 4u; th = 1 - d:
      err th = |d| eps_d + u |th|.  gelu = (x / 2)(1 + th): e = |x| / 2 (err th + u |1 + th|) + u |gelu|.
      gelu' = (1 + th) / 2 + (x / 2)(1 - th^2) k0 m, m = fma(3 k1 x, x, 1): e = (err th + 2u) / 2 + |x k0 m| / 2
      (2 |th| err th + 2u) + 10u |B| + u |gelu'| with B the second term.
    - ACT_GRAD C = v gelu'(aux): e = delta_v |gelu'| + |v_ref| e(gelu') + u |C|.
* fp32 outputs: EPI_F32 within delta_v.  RESID: |g| delta_v + u (|g v| + |ref|) (the gate multiply and the residual
  add).  ATOMIC: |alpha| 8 sqrt(K) u S + u |alpha acc| + (splits + 1) u (|C0| + |alpha| sum_k |a_k b_k|), the split
  partials being reassociated fp32 adds onto C0.  Each of these bounds must reject a bf16 rounding of the reference by
  at least 2x.
* Writes outside the result: every output lives in a sentinel-filled buffer with rows below M and columns on both
  sides; the offset of the result is 16 bytes (32 for SwiGLU) where the case wants the pair path and one element where
  it wants the scalar path.  Every sentinel must survive.

Every case asserts, from a torch.profiler trace, that the gemm_wgmma_kernel<BLOCK_N, kMN> that route() -- a copy of the
host logic of md_gemm_bf16 -- predicts ran, and splitk_reduce_kernel in deterministic split cases.  In a long process
whose earlier tests started the profiler and then ran the DiT training tests, CUDA tracing can stop delivering kernel
records, and a late record of an earlier session can show up in a later one: so a trace that holds no GEMM kernel in
any attempt is printed instead of asserted, and a trace that holds some must contain every predicted kernel.
test_matrix_reaches_every_path (tests/test_gemm_bf16_model_cpu.py) checks that the matrix reaches every allowed
combination of instantiation, epilogue, path, activation and gate, and that it holds every GEMM signature the engine
issues.  Each case prints its worst error / bound per output and its smallest share of single-value brackets.

MD_TEST_DRYRUN=1 runs the same cases on the CPU contract (tests.bias_common.BiasEmuOps: oracle.emu_ops.EmuOps with the
SwiGLU bias in the header's natural order); the route and kernel assertions and the rejection tests are skipped there.
tests/test_gemm_bf16_model_cpu.py runs these cases on emulations with one injected fault each.
"""
import dataclasses
import math
import os
import re

import pytest
import torch

from oracle.emu_ops import (EPI_ACT_DUAL, EPI_ACT_GRAD, EPI_ATOMIC, EPI_BF16, EPI_F32, EPI_RESID, EPI_SWIGLU,
                            EPI_SWIGLU_GRAD, NT, TN)
from tests import f64_reference as R
from tests.test_attention_bf16_gpu import _traced

pytestmark = pytest.mark.gpu
DRY = bool(os.environ.get("MD_TEST_DRYRUN"))
DEV = "cuda:0"
BF16, F32, D64 = torch.bfloat16, torch.float32, torch.float64
U = 2.0 ** -24
SENT = -768.0           # exact in bf16 and far outside any output here
BELOW = 3               # sentinel rows below M
SINGLE_FLOOR = 0.85
SECOND_ORDER = 1.0 + 2.0 ** -10
DET_WS = 256 << 20      # deterministic workspace of the split cases; SMALL_WS forces the un-split fallback
SMALL_WS = 1 << 20
EPI_NAME = {EPI_BF16: "BF16", EPI_F32: "F32", EPI_RESID: "RESID", EPI_ATOMIC: "ATOMIC", EPI_ACT_DUAL: "ACT_DUAL",
            EPI_ACT_GRAD: "ACT_GRAD", EPI_SWIGLU: "SWIGLU", EPI_SWIGLU_GRAD: "SWIGLU_GRAD"}


# ------------------------------------------------------------------------------------------------ the cases
@dataclasses.dataclass(frozen=True)
class Spec:
    epi: int
    layout: int
    M: int
    N: int                   # the GEMM's N (SWIGLU_GRAD: f, its output has 2f columns)
    K: int
    batch: int = 1
    act: int = 0
    alpha: float = 1.0
    bias: str = ""           # "", "shared" ([N]) or "batched" ([batch, N] rows of a wider buffer)
    rows_per_gate: int = 0   # > 0: RESID gate [ceil(M / rows_per_gate), N], a column slice of a wider buffer
    res_mod: int = 0
    inplace: bool = False    # RESID with res = C
    c2: bool = False         # RESID side copy
    scalar: bool = False     # outputs one element off the 16-byte grid (SWIGLU: the bias instead)
    splits: int = 1
    interleave: bool = False  # ATOMIC row_interleave = M / 2
    sm_limit: int = 0
    modes: tuple = (None,)   # deterministic workspace per run (None: mode off)
    seed: int = 1

    def tag(self):
        s = f"{EPI_NAME[self.epi]} {'TN' if self.layout else 'NT'} {self.M}x{self.N}x{self.K}"
        s += f" b{self.batch}" if self.batch > 1 else ""
        for k, v in (("act", self.act), ("a", self.alpha), ("bias", self.bias), ("rpg", self.rows_per_gate),
                     ("rmod", self.res_mod), ("inplace", self.inplace), ("c2", self.c2), ("scalar", self.scalar),
                     ("s", self.splits if self.splits != 1 else 0), ("il", self.interleave), ("sm", self.sm_limit)):
            if v and not (k == "a" and v == 1.0):
                s += f" {k}{'' if v is True else v}"
        return s


def _rup(x, m):
    return (x + m - 1) // m * m


def _matrix():
    """Every (layout, BLOCK_N, epilogue[, act | gate]) on a ragged shape with the pair path (interior and guarded
    tiles) and on the scalar path, cycling K, alpha, batch and bias kinds; then the edges and the engine's calls."""
    out = []
    Ks = [8, 72, 16, 200, 72, 4000]
    alphas = [1.0, 0.05, 0.0]
    i = 0
    for layout in (NT, TN):
        for bn in (128, 256):
            sm = 0 if bn == 128 else 5   # 256-wide tiles on a small shape only win when few SMs are allowed
            variants = [(EPI_BF16, {}), (EPI_F32, {"bias": "shared"}), (EPI_RESID, {"bias": "shared"}),
                        (EPI_RESID, {"rows_per_gate": 77, "res_mod": 64}), (EPI_ATOMIC, {"splits": 4, "modes": (None, DET_WS)})]
            if layout == NT:
                variants += [(EPI_ACT_DUAL, {"act": 0, "bias": "shared"}), (EPI_ACT_DUAL, {"act": 1}),
                             (EPI_ACT_GRAD, {"act": 0}), (EPI_ACT_GRAD, {"act": 1}),
                             (EPI_SWIGLU, {"bias": "shared"}), (EPI_SWIGLU_GRAD, {})]
            for epi, kw in variants:
                N = {EPI_SWIGLU: {128: 192, 256: 1024}, EPI_SWIGLU_GRAD: {128: 160, 256: 512}}.get(epi, {128: 200, 256: 1000})[bn]
                for scalar in (False, True):
                    if epi == EPI_SWIGLU_GRAD and scalar:
                        continue     # every pointer and pitch it takes is 32-byte / 16-element aligned: never scalar
                    K = Ks[i % len(Ks)]
                    if epi in (EPI_ACT_GRAD, EPI_SWIGLU_GRAD) or (epi == EPI_SWIGLU and scalar):
                        kw = dict(kw, bias=kw.get("bias", "shared") if epi == EPI_SWIGLU else "")
                    batch = 2 if i % 4 == 3 else 1
                    kk = dict(kw)
                    if batch > 1 and kk.get("bias") == "shared" and epi != EPI_SWIGLU:
                        kk["bias"] = "batched"
                    out.append(Spec(epi, layout, 129 if scalar else 257, N, K, batch=batch, alpha=alphas[i % 3],
                                    scalar=scalar, sm_limit=sm, seed=i, **kk))
                    i += 1
    out += [
        # tiny and sub-k-block shapes
        Spec(EPI_BF16, NT, 1, 8, 8), Spec(EPI_F32, TN, 7, 16, 16, bias="shared", alpha=0.05),
        Spec(EPI_RESID, NT, 127, 72, 200, rows_per_gate=64, res_mod=64, c2=True),
        Spec(EPI_ACT_DUAL, NT, 7, 72, 16, act=1, bias="shared", scalar=True),
        # N = 130: ldc2 = N / 2 is odd, so pair accesses are off for every tile (vec2 = 0) although every pointer is aligned
        Spec(EPI_BF16, NT, 256, 130, 72, bias="shared"), Spec(EPI_RESID, TN, 256, 130, 200, c2=True, rows_per_gate=64),
        # the 256 -> 128 fallback (15 wide tiles do not fill the machine) at K = 4000
        Spec(EPI_F32, NT, 384, 1096, 4000, bias="shared"),
        # enough 256-wide tiles for the whole machine (9 x 16 = 144)
        Spec(EPI_BF16, NT, 1152, 4096, 16, bias="shared"), Spec(EPI_F32, TN, 1152, 4096, 72, alpha=0.05),
        Spec(EPI_RESID, NT, 1152, 4096, 8, c2=True, rows_per_gate=256, res_mod=77),
        # interior-only shapes (multiples of the tile), batched with per-batch bias, in-place residual
        Spec(EPI_RESID, NT, 512, 256, 200, batch=2, bias="batched", rows_per_gate=256, inplace=True),
        Spec(EPI_BF16, TN, 256, 512, 72, batch=3, bias="batched", sm_limit=5),
        Spec(EPI_ACT_DUAL, NT, 256, 1024, 200, batch=2, bias="batched", sm_limit=5),
        Spec(EPI_SWIGLU, NT, 384, 1024, 72, batch=2, bias="batched", sm_limit=5),
        Spec(EPI_SWIGLU_GRAD, NT, 256, 256, 200, batch=2),
        # gated residual whose gate changes mid-tile, with a side copy and a wrapped residual, many tiles per CTA
        Spec(EPI_RESID, NT, 300, 1000, 200, bias="shared", rows_per_gate=77, res_mod=77, c2=True, sm_limit=5),
        Spec(EPI_RESID, TN, 257, 300, 72, batch=3, bias="batched", rows_per_gate=64, sm_limit=1),
        # split-K: empty splits (K = 64, 4 splits; kb_total = 9, 4 splits), the auto split, one CTA for everything, and
        # the deterministic reduction and its un-split fallback (4 x 256 x 512 x 4 bytes > 1 MiB)
        Spec(EPI_ATOMIC, NT, 200, 136, 64, splits=4, modes=(None, DET_WS)),
        Spec(EPI_ATOMIC, TN, 136, 200, 576, splits=4, alpha=0.05, modes=(None, DET_WS)),
        Spec(EPI_ATOMIC, TN, 256, 512, 4000, splits=0, modes=(None, DET_WS)),
        Spec(EPI_ATOMIC, NT, 300, 200, 4000, batch=2, splits=0, modes=(None, DET_WS)),
        Spec(EPI_ATOMIC, TN, 257, 300, 520, batch=3, splits=4, sm_limit=1, modes=(None, DET_WS)),
        Spec(EPI_ATOMIC, TN, 256, 512, 200, splits=4, modes=(SMALL_WS,)),
        # the weight gradient of a 32-row-interleaved SwiGLU stack (M = 2f)
        Spec(EPI_ATOMIC, TN, 192, 200, 300, splits=0, interleave=True, modes=(None, DET_WS)),
        Spec(EPI_ATOMIC, TN, 256, 72, 64, splits=4, interleave=True, modes=(None, DET_WS)),
        # the GEMM signatures the engine issues that the loops above do not already have
        Spec(EPI_BF16, NT, 300, 256, 72, batch=3), Spec(EPI_F32, NT, 129, 200, 72),
        Spec(EPI_RESID, NT, 256, 200, 72), Spec(EPI_RESID, NT, 256, 200, 72, bias="shared", res_mod=64),
        Spec(EPI_RESID, NT, 256, 200, 72, inplace=True),
        Spec(EPI_ATOMIC, NT, 256, 200, 520, splits=0), Spec(EPI_ATOMIC, TN, 256, 200, 520, batch=2, splits=0),
        Spec(EPI_ACT_DUAL, NT, 256, 200, 72, batch=2), Spec(EPI_ACT_GRAD, NT, 256, 200, 72, batch=2),
        Spec(EPI_SWIGLU, NT, 256, 192, 72),
    ]
    return out


SPECS = _matrix()


class Case:
    """Seeded bf16 operands and side inputs of one Spec in padded / sentinel-filled buffers, and the float64 results
    with their error terms."""

    def __init__(self, s: Spec, reference=True):
        self.s = s
        g = torch.Generator().manual_seed(1000 + s.seed)
        b, M, N, K = s.batch, s.M, s.N, s.K
        self.Nc = 2 * N if s.epi == EPI_SWIGLU_GRAD else N
        swig = s.epi in (EPI_SWIGLU, EPI_SWIGLU_GRAD)
        self.off = 16 if swig else (1 if s.scalar else 8)
        W = _rup(self.off + self.Nc + 8, 16) + (1 if s.scalar and not swig else 0)
        bufs = {}
        # operands: row pitch padded past K (NT) or M / N (TN); the padding holds random values the kernel must not read
        if s.layout == NT:
            bufs["A"] = torch.randn(b, M, _rup(K, 8) + 8, generator=g) * (1.5 / math.sqrt(K))
            bufs["B"] = torch.randn(b, N, _rup(K, 8) + 8, generator=g)
        else:
            bufs["A"] = torch.randn(b, K, _rup(M, 8) + 8, generator=g) * (1.5 / math.sqrt(K))
            bufs["B"] = torch.randn(b, K, _rup(N, 8) + 8, generator=g)
        bufs["A"], bufs["B"] = bufs["A"].to(BF16), bufs["B"].to(BF16)
        cdt = F32 if s.epi in (EPI_F32, EPI_RESID, EPI_ATOMIC) else BF16
        bufs["C"] = torch.full((b, M + BELOW, W), SENT, dtype=cdt)
        if s.epi == EPI_SWIGLU:
            bufs["C2"] = torch.full((b, M + BELOW, _rup(N // 2 + 32, 16)), SENT, dtype=BF16)
        elif s.epi == EPI_ACT_DUAL or (s.epi == EPI_RESID and s.c2):
            bufs["C2"] = torch.full((b, M + BELOW, W), SENT, dtype=BF16)
        if s.bias:
            boff = 1 if s.scalar else 2
            shape = (N + 2 * boff + 4,) if s.bias == "shared" else (b, N + 2 * boff + 4)
            bufs["bias"] = torch.randn(*shape, generator=g)
        if s.epi == EPI_RESID and not s.inplace:
            bufs["res"] = torch.randn(b, M + BELOW, W, generator=g)
        if s.rows_per_gate:
            bufs["gate"] = torch.randn((M + s.rows_per_gate - 1) // s.rows_per_gate, N + 12, generator=g)
        if s.epi in (EPI_ACT_GRAD, EPI_SWIGLU_GRAD):
            bufs["aux"] = (torch.randn(b, M + BELOW, W, generator=g) * 2).to(BF16)
        v = self.views(bufs)
        if s.epi == EPI_ATOMIC or s.inplace:   # C0, or the residual read from C itself
            v["C"].copy_(torch.randn(v["C"].shape, generator=g))
        self.bufs = bufs
        if reference:
            self._reference(v)

    # ---------------------------------------------------------------- geometry
    def views(self, bufs):
        """The GEMM's arguments as views of the buffers (on whatever device they are)."""
        s, M, N, K, off = self.s, self.s.M, self.s.N, self.s.K, self.off
        one = (lambda t: t[0]) if s.batch == 1 else (lambda t: t)
        v = {}
        if s.layout == NT:
            v["A"], v["B"] = one(bufs["A"][:, :, :K]), one(bufs["B"][:, :, :K])
        else:
            v["A"], v["B"] = one(bufs["A"][:, :, :M]), one(bufs["B"][:, :, :N])
        v["C"] = one(bufs["C"][:, :M, off:off + self.Nc])
        if "C2" in bufs:
            v["C2"] = one(bufs["C2"][:, :M, 16:16 + N // 2]) if s.epi == EPI_SWIGLU else one(bufs["C2"][:, :M, off:off + N])
        if "bias" in bufs:
            boff = 1 if s.scalar else 2
            v["bias"] = bufs["bias"][..., boff:boff + N]
        if s.epi == EPI_RESID:
            v["res"] = v["C"] if s.inplace else one(bufs["res"][:, :M, off:off + N])
        if "gate" in bufs:
            v["gate"] = bufs["gate"][:, 6:6 + N]
        if "aux" in bufs:
            v["aux"] = one(bufs["aux"][:, :M, off:off + self.Nc])
        return v

    def kwargs(self, v):
        s = self.s
        return dict(layout=s.layout, epi=s.epi, C2=v.get("C2"), bias=v.get("bias"), res=v.get("res"), gate=v.get("gate"),
                    rows_per_gate=s.rows_per_gate, res_mod=s.res_mod, splits=s.splits, act=s.act, alpha=s.alpha,
                    aux=v.get("aux"), row_interleave=s.M // 2 if s.interleave else 0)

    def vec2(self):
        """md_gemm_bf16's pair-access rule: 8-byte aligned pointers and even pitches everywhere, including the
        dev.ldc2 = N / 2 default of the epilogues that have no C2 pitch."""
        s, v = self.s, self.views(self.bufs)
        C3 = v["C"] if s.batch > 1 else v["C"].unsqueeze(0)
        ptrs = [t.data_ptr() for k, t in v.items() if k in ("C", "C2", "bias", "res", "gate", "aux")]
        ldc2 = v["C2"].stride(-2) if s.epi == EPI_SWIGLU else s.N // 2
        strideC2 = v["C2"].stride(0) if s.epi == EPI_SWIGLU and s.batch > 1 else 0
        sbias = v["bias"].stride(0) if "bias" in v and v["bias"].dim() == 2 else 0
        ldgate = v["gate"].stride(0) if "gate" in v else 0
        pitches = s.N | C3.stride(1) | C3.stride(0) | ldc2 | strideC2 | sbias | ldgate
        return all(p % 8 == 0 for p in ptrs) and pitches % 2 == 0

    # ---------------------------------------------------------------- float64 results and error terms
    def _reference(self, v):
        s = self.s
        A, B = v["A"], v["B"]
        a = abs(s.alpha) if s.alpha else 1.0
        acc = R.matmul(A, B, s.layout)
        bias = v.get("bias")
        if bias is not None and s.epi == EPI_SWIGLU:   # natural [b1 | b2] -> the interleaved columns
            bias = bias.index_select(-1, R.interleaved_to_natural(s.N // 2))
        self.v = R.gemm(A, B, s.layout, alpha=s.alpha, bias=bias)
        self.sq = R.matmul(A.double() ** 2, B.double() ** 2, s.layout).sqrt()
        self.quad = a * 8.0 * math.sqrt(s.K) * U * self.sq
        self.dv = self.quad + U * (a * acc.abs() + self.v.abs())
        self.absacc = a * R.matmul(A.double().abs(), B.double().abs(), s.layout)
        self.acc = a * acc
        if s.epi == EPI_RESID:
            self.res = R.f64(v["res"]).clone()
            self.ref = R.gemm(A, B, s.layout, alpha=s.alpha, bias=bias, res=self.res, res_mod=s.res_mod,
                              gate=v.get("gate"), rows_per_gate=s.rows_per_gate)
            self.g = R._per_row(v["gate"], s.rows_per_gate, s.M).abs() if "gate" in v else torch.ones(())
        elif s.epi == EPI_ATOMIC:
            self.c0 = R.f64(v["C"]).clone()
        elif s.epi == EPI_ACT_GRAD:
            x = R.f64(v["aux"])
            self.ref = R.gemm(A, B, s.layout, alpha=s.alpha, aux=x, act=s.act)
            gp = R.gelu_grad(x, s.act)
            self.bound = self.dv * gp.abs() + self.v.abs() * _gelu_err(x, s.act, grad=True) + U * self.ref.abs()
        elif s.epi == EPI_SWIGLU_GRAD:
            u = R.f64(v["aux"])
            perm = R.interleaved_to_natural(s.N)
            nat = torch.empty_like(u)
            nat[..., perm] = u
            rows = nat.reshape(-1, 2 * s.N)
            du = R.swiglu_bwd(self.v.reshape(-1, s.N), rows).reshape(u.shape)
            self.ref = du[..., perm]
            a1, a2 = nat[..., :s.N], nat[..., s.N:]
            sg = torch.sigmoid(a1)
            es = _sig_err(a1)
            t = 1.0 + a1 * (1.0 - sg)
            e_q = sg * es + U * (1.0 - sg).abs()
            e_t = a1.abs() * e_q + U * t.abs()
            e_st = t.abs() * sg * es + sg * e_t + U * (sg * t).abs()
            d = self.v
            e1 = (d * a2).abs() * (e_st + 2 * U * (sg * t).abs()) + self.dv * (a2 * sg * t).abs()
            e2 = (d * a1 * sg).abs() * (es + 2 * U) + self.dv * (a1 * sg).abs()
            self.bound = torch.cat([e1, e2], -1)[..., perm] * SECOND_ORDER

    # ---------------------------------------------------------------- checks
    def metrics(self, outs, splits):
        """{check: worst error as a fraction of what it may be (<= 1 passes)}, {output: share of single-value brackets},
        {fp32 output: how far a bf16 rounding of the reference misses its bound}."""
        s = self.s
        v = self.views({**self.bufs, **outs})
        m, share, teeth = {}, {}, {}

        def brk(name, got, ref, d):
            m[name], share[name] = bracket(got, ref, d)

        def fp32(name, got, ref, bound):
            m[name] = _ratio(R.f64(got), ref, bound)
            teeth[name] = _ratio(rn_bf16(ref), ref, bound)

        C = v["C"]
        if s.epi == EPI_BF16:
            brk("C", C, self.v, self.dv)
        elif s.epi == EPI_F32:
            fp32("C", C, self.v, self.dv)
        elif s.epi == EPI_RESID:
            bound = self.g * self.dv + U * ((self.g * self.v).abs() + self.ref.abs())
            fp32("C", C, self.ref, bound)
            if "C2" in v:
                brk("C2", v["C2"], self.v, self.dv)
        elif s.epi == EPI_ATOMIC:
            part = self.quad + U * self.acc.abs() + (splits + 1) * U * self.absacc
            ref = self.c0.clone()
            if s.interleave:   # GEMM row p is output row perm[p]
                perm = R.interleaved_to_natural(s.M // 2)
                ref[..., perm, :] += self.v
                part = part.clone()
                part[..., perm, :] = part.clone()
            else:
                ref = ref + self.v
            fp32("C", C, ref, part + (splits + 1) * U * self.c0.abs())
        elif s.epi == EPI_ACT_DUAL:
            brk("C", C, self.v, self.dv)
            pre = R.f64(C)
            brk("C2", v["C2"], R.gelu(pre, s.act), _gelu_err(pre, s.act))
        elif s.epi == EPI_ACT_GRAD:
            brk("C", C, self.ref, self.bound)
        elif s.epi == EPI_SWIGLU:
            brk("C", C, self.v, self.dv)
            u = R.f64(C)
            perm = R.interleaved_to_natural(s.N // 2)
            nat = torch.empty_like(u)
            nat[..., perm] = u
            h = R.swiglu_fwd(nat.reshape(-1, s.N)).reshape(u.shape[:-1] + (s.N // 2,))
            a1 = nat[..., :s.N // 2]
            brk("C2", v["C2"], h, h.abs() * (_sig_err(a1) + 2 * U) * SECOND_ORDER)
        elif s.epi == EPI_SWIGLU_GRAD:
            brk("C", C, self.ref, self.bound)
        for name, buf in outs.items():
            m[name + " outside"] = _outside(self, name, buf)
        return m, share, teeth


def rn_bf16(x):
    """Round float64 to the nearest bf16 (ties to even) in one step -- a float64 -> bf16 cast goes through fp32 and can
    round twice."""
    x = x.double()
    _, e = torch.frexp(x)
    scale = torch.exp2((8 - e).double())
    return torch.round(x * scale) / scale


def bracket(got, ref, d):
    """(worst |got - ref| / |bracket end on got's side - ref|, share of single-value brackets) for the rounding bracket
    [rn(ref - d), rn(ref + d)]: <= 1 means every element is inside."""
    got = R.f64(got)
    lo, hi = rn_bf16(ref - d), rn_bf16(ref + d)
    side = torch.where(got >= ref, hi, lo)
    num = (got - ref).abs()
    r = torch.where(num == 0, torch.zeros_like(num), num / (side - ref).abs())
    worst = float(torch.nan_to_num(r, nan=math.inf).max()) if r.numel() else 0.0
    return worst, float((lo == hi).double().mean()) if r.numel() else 1.0


def _ratio(got, ref, bound):
    r = (got - ref).abs() / bound.clamp_min(1e-300)
    return float(torch.nan_to_num(r, nan=math.inf).max()) if r.numel() else 0.0


def _outside(c, name, buf):
    """0 if every element of buf outside the GEMM's view still holds the sentinel, else inf."""
    mark = torch.zeros(buf.shape, dtype=torch.bool)
    c.views({**{k: torch.zeros(t.shape, dtype=torch.bool) for k, t in c.bufs.items()}, name: mark})[name].fill_(True)
    return 0.0 if bool((buf[~mark].double() == SENT).all()) else math.inf


def _sig_err(a):
    """Relative error of the kernel's sigmoid 1 / (1 + __expf(-a)) (module docstring)."""
    E = torch.exp(-a)
    eps_e = (2 + torch.floor(1.173 * a.abs())) * 2 * U
    return torch.where(torch.isfinite(E), E / (1 + E), torch.ones_like(E)) * eps_e + U + 4 * U


_AS = (0.254829592, -0.284496736, 1.421413741, -1.453152027, 1.061405429)


def _gelu_err(x, act, grad=False):
    """Absolute fp32 evaluation error of gelu_erf_fast / gelu_tanh_fast (grad: their derivatives) at x (module
    docstring)."""
    x = R.f64(x)
    if act == 0:
        z = x.abs() / math.sqrt(2.0)
        t = 1.0 / (1.0 + 0.3275911 * z)
        Q = sum(abs(c) * t ** (i + 1) for i, c in enumerate(_AS))
        Q1 = sum((i + 1) * abs(c) * t ** (i + 1) for i, c in enumerate(_AS))
        pt = sum(c * t ** (i + 1) for i, c in enumerate(_AS))
        zz = z * z
        E = torch.exp(-zz)
        eps_e = (2 + torch.floor(1.173 * zz)) * 2 * U + 3 * U * zz
        e_erf = 1.5e-7 + E * 6 * U * (Q + Q1) + pt.abs() * E * (eps_e + U) + U
        if grad:
            val = R.gelu_grad(x, 0)
            e = (e_erf + 2 * U) / 2 + (x * E).abs() / math.sqrt(2 * math.pi) * (eps_e + 2 * U) + U * val.abs()
        else:
            e = x.abs() / 2 * (e_erf + 2 * U) + U * R.gelu(x, 0).abs()
    else:
        k0, k1 = math.sqrt(2.0 / math.pi), 0.044715
        w = 2 * k0 * (x + k1 * x ** 3)
        E = torch.exp(w)
        eps_e = (2 + torch.floor(1.173 * w.abs())) * 2 * U + 6 * U * w.abs()
        frac = torch.where(torch.isfinite(E), E / (1 + E), torch.ones_like(E))
        d = 2.0 / (1.0 + E)
        th = torch.tanh(w / 2)
        e_th = d * (frac * eps_e + 5 * U) + U * th.abs()
        if grad:
            mm = 1 + 3 * k1 * x * x
            Bt = 0.5 * x * (1 - th * th) * k0 * mm
            e = (e_th + 2 * U) / 2 + (x * k0 * mm).abs() / 2 * (2 * th.abs() * e_th + 2 * U) + 10 * U * Bt.abs() \
                + U * R.gelu_grad(x, 1).abs()
        else:
            e = x.abs() / 2 * (e_th + U * (1 + th).abs()) + U * R.gelu(x, 1).abs()
    return e * SECOND_ORDER


# ------------------------------------------------------------------------------------------------ route
@dataclasses.dataclass(frozen=True)
class Route:
    block_n: int
    kmn: bool
    splits: int
    vec2: bool
    interior: int
    guarded: int
    reduce: bool

    def kernels(self):
        k = {f"gemm_wgmma_kernel<{self.block_n}, {'true' if self.kmn else 'false'}>"}
        return k | {"splitk_reduce_kernel"} if self.reduce else k


def route(s: Spec, vec2: bool, sm_count: int, det_ws=None):
    """The host logic of md_gemm_bf16: tile width (the use256 rule and its fallback when 256-wide tiles do not fill the
    machine), layout, effective splits (the splits == 0 cost model and the deterministic workspace fallback), pair
    accesses and how many tiles take the interior and the guarded epilogue."""
    M, N, K, b = s.M, s.N, s.K, s.batch
    mb, kb = -(-M // 128), -(-K // 64)

    def tiles_for(bn):
        return b * mb * -(-N // bn)
    use256 = N >= 256 and (-(-N // 256) * 256 - N) * 5 <= N
    sp = s.splits if s.splits > 0 else 1
    if s.splits == 0 and s.epi == EPI_ATOMIC:
        t = tiles_for(256 if use256 else 128)
        smax = min(kb // 8, 64) if kb // 8 > 0 else 1
        best = 1e30
        for c in range(1, smax + 1):
            cost = -(-(t * c) // sm_count) * (-(-kb // c) + 10.0)
            if cost < best - 1e-9:
                best, sp = cost, c
    elif use256 and tiles_for(256) * sp < sm_count and tiles_for(128) * sp > tiles_for(256) * sp:
        use256 = False
    bn = 256 if use256 else 128
    reduce = det_ws is not None and s.epi == EPI_ATOMIC and sp > 1
    if reduce and 4 * sp * b * M * N > det_ws:
        sp, reduce = 1, False
    interior = b * (M // 128) * (N // bn) if vec2 and s.epi != EPI_ATOMIC else 0
    return Route(bn, s.layout == TN, sp, vec2, interior, tiles_for(bn) * sp - interior, reduce)


def paths(s, r):
    """The (instantiation, epilogue, path, act, gated) combinations a run of s along route r reaches."""
    inst = (r.block_n, r.kmn)
    act = s.act if s.epi in (EPI_ACT_DUAL, EPI_ACT_GRAD) else 0
    gated = bool(s.rows_per_gate)
    out = set()
    if r.interior:
        out.add((inst, s.epi, "interior", act, gated))
    if r.guarded:
        out.add((inst, s.epi, "guarded vec" if r.vec2 else "guarded scalar", act, gated))
    return out


def signature(s):
    """(layout, epi, act, bias kind, gate, res_mod, C2, aux, splits, row_interleave, batched) of a Spec: the GEMM call
    signature tests/test_gemm_bf16_model_cpu.py records from the engine."""
    return (s.layout, s.epi, s.act if s.epi in (EPI_ACT_DUAL, EPI_ACT_GRAD) else 0,
            {"": None, "shared": 1, "batched": 2}[s.bias], bool(s.rows_per_gate), s.res_mod > 0,
            s.epi in (EPI_ACT_DUAL, EPI_SWIGLU) or s.c2, s.epi in (EPI_ACT_GRAD, EPI_SWIGLU_GRAD), s.splits,
            s.interleave, s.batch > 1)


GEMM_KERNELS = {f"gemm_wgmma_kernel<{bn}, {m}>" for bn in (128, 256) for m in ("false", "true")} | {"splitk_reduce_kernel"}


def _gemm_ids(names):
    """Kernel ids of trace names, demangled (gemm_wgmma_kernel<128, false>) or mangled (gemm_wgmma_kernelILi128ELb0EE)."""
    ids, unknown = set(), []
    for n in names:
        hit = set()
        for kid in GEMM_KERNELS:
            m = re.fullmatch(r"(\w+)<(\d+), (\w+)>", kid)
            pats = (kid + "(", kid + "P") if not m else \
                (kid, f"{m.group(1)}ILi{m.group(2)}ELb{int(m.group(3) == 'true')}E")
            if any(p in n for p in pats):
                hit.add(kid)
        ids |= hit
        if not hit:
            unknown.append(n)
    return ids, unknown


# ------------------------------------------------------------------------------------------------ running
def _dev(ops):
    return "cpu" if getattr(ops, "is_emulation", False) else DEV


def _ops():
    if DRY:
        from tests.bias_common import BiasEmuOps
        return BiasEmuOps("cpu")
    from micro_diffusion_b200.ops import CudaOps
    return CudaOps(torch.device(DEV))


def sm_count(sm_limit=0):
    """SMs a persistent GEMM grid may use: the device's count, capped by ops.sm_limit (132 on a dry run: an H100 SXM)."""
    n = 132 if DRY else torch.cuda.get_device_properties(DEV).multi_processor_count
    return min(n, sm_limit) if sm_limit > 0 else n


def run(ops, c, det_ws=None):
    """One md_gemm_bf16 call on fresh device copies of the case's buffers; returns the output buffers on the host."""
    dev = _dev(ops)
    bufs = {k: t.to(dev, copy=True) for k, t in c.bufs.items()}
    v = c.views(bufs)
    ops.gemm(v["A"], v["B"], v["C"], **c.kwargs(v))
    return {k: bufs[k].cpu() for k in ("C", "C2") if k in bufs}


def _set_det(ops, det_ws):
    if DRY:
        return
    from micro_diffusion_b200 import ops as O
    ws = O._DET_WORKSPACE.get("ws")
    if ws is not None and (det_ws is None or ws.numel() != det_ws):
        ops.set_deterministic(False)
    if det_ws is not None:
        ops.set_deterministic(True, workspace_bytes=det_ws)


@pytest.fixture(autouse=True)
def _deterministic_mode_is_switched_off_again():
    """The switch is process-wide: whatever a test does, later tests of the same process run in the default mode."""
    try:
        yield
    finally:
        if not DRY:
            _ops().set_deterministic(False)


def report(tag, m, share):
    worst = {n: v for n, v in m.items() if "outside" not in n}
    print(f"\n[{tag}] " + " ".join(f"{n} {v:.3g}" for n, v in worst.items())
          + (f" single {min(share.values()):.3f}" if share else ""), end="")


def check(c, outs, sp):
    """Failures of one run: error / bound above 1, a sentinel overwritten, too few single-value brackets, an fp32 bound
    that would pass a bf16 rounding of the reference."""
    m, share, teeth = c.metrics(outs, sp)
    failed = [(n, round(v, 3)) for n, v in m.items() if not v <= 1.0]
    failed += [(n + " single", round(v, 3)) for n, v in share.items() if v < SINGLE_FLOOR]
    failed += [(n + " teeth", round(v, 3)) for n, v in teeth.items() if v < 2.0]
    return m, share, failed


@pytest.mark.parametrize("spec", SPECS, ids=lambda s: s.tag().replace(" ", "-"))
def test_bf16_gemm_within_error_model(spec):
    c = Case(spec)
    failed = []
    for det_ws in spec.modes:
        ops = _ops()
        if not DRY:
            ops.sm_limit = spec.sm_limit
        _set_det(ops, det_ws)
        r = route(spec, c.vec2(), sm_count(ops.sm_limit if not DRY else spec.sm_limit), det_ws)
        if DRY:
            outs = run(ops, c, det_ws)
        else:
            want = r.kernels()
            outs, _, names = _traced(ops, lambda: run(ops, c, det_ws), want, keep=("gemm_wgmma", "splitk_reduce"),
                                     ids=_gemm_ids)
            ids, unknown = _gemm_ids(names)
            if not names:
                print("\n[kernel trace unavailable: no GEMM kernel recorded in any attempt]", end="")
            else:
                assert want <= ids and not unknown, (sorted(names), want, r)
        m, share, f = check(c, outs, r.splits)
        report(f"{spec.tag()} det={det_ws} {'/'.join(sorted(r.kernels()))} splits {r.splits} "
               f"tiles {r.interior}i+{r.guarded}{'v' if r.vec2 else 's'}", m, share)
        failed += [(det_ws, *x) for x in f]
    assert not failed, failed


# ------------------------------------------------------------------------------------------------ argument checks
def _lib_error():
    from micro_diffusion_b200._lib import MicroditLibraryError
    return MicroditLibraryError


@pytest.mark.skipif(DRY, reason="argument checks of the C entry point")
@pytest.mark.parametrize("precision", ["bf16", "high"])
@pytest.mark.parametrize("det", [False, True])
@pytest.mark.parametrize("splits", [1, 4, 0])
def test_bias_on_the_accumulate_epilogue_is_rejected(splits, det, precision):
    """MD_EPI_ATOMIC_F32 is C += alpha*acc: a bias would be added once per split (and not at all by the deterministic
    partials), so md_gemm_bf16 returns MD_ERR_INVALID for one, before anything launches."""
    from micro_diffusion_b200.ops import CudaOps
    ops = CudaOps(torch.device(DEV), precision=precision)
    if det:
        ops.set_deterministic(True, workspace_bytes=DET_WS)
    M, N, K = 256, 512, 4000
    lowp = F32 if precision == "high" else BF16
    A = torch.randn(K, M, device=DEV).to(lowp)
    B = torch.randn(K, N, device=DEV).to(lowp)
    C = torch.full((M, N), 3.0, device=DEV)
    bias = torch.ones(N, device=DEV)
    with pytest.raises(_lib_error(), match="accumulate epilogue takes no bias"):
        ops.gemm(A, B, C, layout=TN, epi=EPI_ATOMIC, bias=bias, splits=splits)
    torch.cuda.synchronize()
    assert bool((C == 3.0).all()), "C changed by a rejected call"


@pytest.mark.skipif(DRY, reason="argument checks of the host wrapper")
@pytest.mark.parametrize("epi", [EPI_RESID, EPI_ACT_DUAL])
@pytest.mark.parametrize("layout_kind", ["contiguous C2 beside a column-slice C", "batched C2 with its own batch stride"])
def test_c2_laid_out_unlike_c_is_rejected(epi, layout_kind):
    """The kernel writes C2 at C's offsets (batch stride, row pitch).  A C2 with other strides raises before anything
    launches.  The C2 here is the head of an allocation as large as C's, so that a call that did launch could not write
    outside it."""
    from micro_diffusion_b200.ops import CudaOps
    ops = CudaOps(torch.device(DEV))
    M, N, K = 130, 256, 72
    cdt = F32 if epi == EPI_RESID else BF16
    if layout_kind.startswith("contiguous"):
        A = torch.randn(M, K, device=DEV).to(BF16)
        B = torch.randn(N, K, device=DEV).to(BF16)
        cbuf = torch.full((M, N + 64), SENT, dtype=cdt, device=DEV)
        C = cbuf[:, 32:32 + N]
        store = torch.full((M * cbuf.shape[1],), SENT, dtype=BF16, device=DEV)
        C2 = store[:M * N].view(M, N)
    else:
        A = torch.randn(2, M, K, device=DEV).to(BF16)
        B = torch.randn(2, N, K, device=DEV).to(BF16)
        cbuf = torch.full((2, M + 3, N), SENT, dtype=cdt, device=DEV)
        C = cbuf[:, :M]
        store = torch.full((cbuf.numel(),), SENT, dtype=BF16, device=DEV)
        C2 = store[:2 * M * N].view(2, M, N)
    # a residual laid out like C (res must share C's pitch), so that only C2's layout is wrong
    res = (torch.zeros_like(cbuf)[:, 32:32 + N] if cbuf.dim() == 2 else torch.zeros_like(cbuf)[:, :M]) \
        if epi == EPI_RESID else None
    launches = ops.launches
    with pytest.raises(AssertionError):
        ops.gemm(A, B, C, epi=epi, C2=C2, res=res)
    torch.cuda.synchronize()
    assert ops.launches == launches and bool((cbuf == SENT).all()) and bool((store == SENT).all())
