"""The bf16 GEMM error model of tests/test_gemm_bf16_gpu.py has teeth, and its matrix reaches what it claims to.

* Its cases, run on emulations of the bf16 contract (tests.bias_common.BiasEmuOps) with one injected fault each, fail
  -- each fault at least one case -- while the unmodified contract passes everywhere.  Each fault prints the margin
  by which its worst case missed (error / bound, inf for an overwritten sentinel).
* The matrix reaches every allowed combination of kernel instantiation x epilogue x {interior, guarded with pair
  accesses, guarded scalar} x activation x gate, and the deterministic split-K reduction, on an H100 SXM (132 SMs) and
  PCIe (114 SMs).
* Every GEMM call signature the engine issues in a training step of the S, S16, SB and H configs is in the matrix.
"""
import functools

import pytest
import torch
import torch.nn.functional as F

from oracle.emu_ops import (EPI_ACT_DUAL, EPI_ACT_GRAD, EPI_ATOMIC, EPI_BF16, EPI_F32, EPI_RESID, EPI_SWIGLU,
                            EPI_SWIGLU_GRAD, NT, TN, EmuOps, interleave_perm)
from tests import bias_common as bc
from tests import hd128_common as hc
from tests import parity_common as pc
from tests.test_gemm_bf16_gpu import DET_WS, SMALL_WS, SPECS, Case, check, paths, route, run, signature

# the cases small enough for a quick CPU run, and the wrapped-residual ones (res_mod 77: the only residual map that a
# per-tile row wrap changes)
MODEL_SPECS = [s for s in SPECS if s.M * s.N * s.K <= 20_000_000 or (s.res_mod == 77 and s.M * s.N * s.K < 10 ** 8)]


@functools.lru_cache(maxsize=None)
def _case(spec):
    return Case(spec)


def _fp32(ops, A, B, Cm, kw, bias_il=False):
    """fp32 v = alpha acc + bias of the same call (bias mapped to the interleaved columns for SwiGLU)."""
    tmp = torch.empty(Cm.shape)
    bias = kw.get("bias")
    if bias is not None and bias_il:
        bias = bias.index_select(-1, interleave_perm(bias.shape[-1] // 2))
    EmuOps.gemm(ops, A, B, tmp, layout=kw.get("layout", NT), epi=EPI_F32, bias=bias, alpha=kw.get("alpha", 1.0))
    return tmp


class RoundTowardZero(bc.BiasEmuOps):
    """The bf16 store of EPI_BF16 truncates instead of rounding to nearest."""

    def gemm(self, A, B, Cm, **kw):
        if kw.get("epi", EPI_BF16) != EPI_BF16:
            return super().gemm(A, B, Cm, **kw)
        tmp = _fp32(self, A, B, Cm, kw)
        Cm.copy_((tmp.view(torch.int32) & -65536).view(torch.float32))


class DropKTail(bc.BiasEmuOps):
    """The last K % 64 columns of the reduction are dropped."""

    def gemm(self, A, B, Cm, **kw):
        nt = kw.get("layout", NT) == NT
        K = A.shape[-1] if nt else A.shape[-2]
        k = K - K % 64
        if nt:
            A, B = A[..., :k], B[..., :k]
        else:
            A, B = A[..., :k, :], B[..., :k, :]
        return super().gemm(A, B, Cm, **kw)


class Batch0Bias(bc.BiasEmuOps):
    """Batch entry 0's bias is used for every batch entry."""

    def gemm(self, A, B, Cm, **kw):
        b = kw.get("bias")
        if b is not None and b.dim() == 2:
            kw = dict(kw, bias=b[:1].expand(b.shape))
        return super().gemm(A, B, Cm, **kw)


class GateRowMod(bc.BiasEmuOps):
    """The gate row is row % rows_per_gate instead of row / rows_per_gate."""

    def gemm(self, A, B, Cm, **kw):
        g, rpg = kw.get("gate"), kw.get("rows_per_gate", 0)
        if g is not None:
            idx = torch.arange(Cm.shape[-2]) % rpg % g.shape[0]
            kw = dict(kw, gate=g[idx], rows_per_gate=1)
        return super().gemm(A, B, Cm, **kw)


class ResidRowPerTile(bc.BiasEmuOps):
    """The residual row is (row % 128) % res_mod: the wrap restarts with every 128-row tile."""

    def gemm(self, A, B, Cm, **kw):
        rm = kw.get("res_mod", 0)
        if kw.get("epi") == EPI_RESID and rm > 0:
            idx = (torch.arange(Cm.shape[-2]) % 128) % rm
            kw = dict(kw, res=kw["res"][..., idx, :].clone(), res_mod=0)
        return super().gemm(A, B, Cm, **kw)


class AlphaAfterBias(bc.BiasEmuOps):
    """alpha scales the bias too: alpha (acc + bias)."""

    def gemm(self, A, B, Cm, **kw):
        a, b = kw.get("alpha", 1.0), kw.get("bias")
        if b is not None and a not in (0.0, 1.0):
            kw = dict(kw, bias=b * a)
        return super().gemm(A, B, Cm, **kw)


class ActOnFp32(bc.BiasEmuOps):
    """ACT_DUAL's activation is taken on the fp32 pre-activation, not on the stored bf16 one."""

    def gemm(self, A, B, Cm, **kw):
        super().gemm(A, B, Cm, **kw)
        if kw.get("epi") == EPI_ACT_DUAL:
            kw["C2"].copy_(F.gelu(_fp32(self, A, B, Cm, kw), approximate="tanh" if kw.get("act") == 1 else "none"))


class SwigluHFromFp32(bc.BiasEmuOps):
    """SwiGLU h is taken from the fp32 u, not from the stored bf16 one."""

    def gemm(self, A, B, Cm, **kw):
        super().gemm(A, B, Cm, **kw)
        if kw.get("epi") == EPI_SWIGLU:
            u = _fp32(self, A, B, Cm, kw, bias_il=True)
            ub = u.reshape(u.shape[:-1] + (u.shape[-1] // 64, 2, 32))
            kw["C2"].copy_((F.silu(ub[..., 0, :]) * ub[..., 1, :]).reshape(kw["C2"].shape))


class ErfTanhSwapped(bc.BiasEmuOps):
    """ACT_GRAD differentiates the other GELU (erf <-> tanh)."""

    def gemm(self, A, B, Cm, **kw):
        if kw.get("epi") == EPI_ACT_GRAD:
            kw = dict(kw, act=1 - kw.get("act", 0))
        return super().gemm(A, B, Cm, **kw)


class RowInterleaveIgnored(bc.BiasEmuOps):
    """row_interleave is ignored: the weight gradient lands in the interleaved row order."""

    def gemm(self, A, B, Cm, **kw):
        return super().gemm(A, B, Cm, **dict(kw, row_interleave=0))


class ResidC2Gated(bc.BiasEmuOps):
    """RESID's side copy C2 stores the gated value gate * v instead of v."""

    def gemm(self, A, B, Cm, **kw):
        super().gemm(A, B, Cm, **kw)
        if kw.get("epi") == EPI_RESID and kw.get("C2") is not None and kw.get("gate") is not None:
            v = _fp32(self, A, B, Cm, kw)
            g = kw["gate"].float().repeat_interleave(kw["rows_per_gate"], dim=0)[:Cm.shape[-2]]
            kw["C2"].copy_(v * g)


class EdgeLastRowUnstored(bc.BiasEmuOps):
    """The last row of an edge tile (M % 128 != 0) is never stored."""

    def gemm(self, A, B, Cm, **kw):
        M = Cm.shape[-2]
        outs = [t for t in (Cm, kw.get("C2")) if t is not None]
        kept = [t[..., M - 1, :].clone() for t in outs]
        super().gemm(A, B, Cm, **kw)
        if M % 128:
            for t, k in zip(outs, kept):
                t[..., M - 1, :] = k


FAULTS = [RoundTowardZero, DropKTail, Batch0Bias, GateRowMod, ResidRowPerTile, AlphaAfterBias, ActOnFp32,
          SwigluHFromFp32, ErfTanhSwapped, RowInterleaveIgnored, ResidC2Gated, EdgeLastRowUnstored]


def _worst(ops_cls):
    """(largest failing metric over every case, its case and check, number of failing cases)."""
    best, nfail = (0.0, None, None), 0
    for spec in MODEL_SPECS:
        c = _case(spec)
        m, share, failed = check(c, run(ops_cls("cpu"), c), spec.splits if spec.splits > 0 else 1)
        if failed:
            nfail += 1
            n, v = max(m.items(), key=lambda kv: kv[1])
            if v <= 1.0:   # failed on its single-value share or on teeth
                n, v = failed[0][0], float("inf")
            if v > best[0]:
                best = (v, spec.tag(), n)
    return best, nfail


@pytest.mark.parametrize("fault", FAULTS, ids=lambda f: f.__name__)
def test_injected_fault_fails_a_case(fault):
    (v, tag, n), nfail = _worst(fault)
    print(f"\n[{fault.__name__}] fails {nfail} of {len(MODEL_SPECS)} cases; worst: {n} at {v:.3g}x its bound ({tag})",
          end="")
    assert nfail > 0, f"{fault.__name__} passes every case"


def test_contract_passes():
    worst, nfail = 0.0, 0
    for spec in MODEL_SPECS:
        c = _case(spec)
        m, share, failed = check(c, run(bc.BiasEmuOps("cpu"), c), spec.splits if spec.splits > 0 else 1)
        assert not failed, (spec.tag(), failed)
        worst = max(worst, max(m.values()))
    print(f"\n[contract] {len(MODEL_SPECS)} cases, worst error / bound {worst:.3g}", end="")


# ------------------------------------------------------------------------------------------------ coverage
ACT_EPIS = (EPI_ACT_DUAL, EPI_ACT_GRAD)
ALL_EPIS = (EPI_BF16, EPI_F32, EPI_RESID, EPI_ATOMIC, EPI_ACT_DUAL, EPI_ACT_GRAD, EPI_SWIGLU, EPI_SWIGLU_GRAD)


def allowed():
    """What the host rules of md_gemm_bf16 let a call reach.  The math tails need NT; ATOMIC never takes the interior
    epilogue; SWIGLU_GRAD's guarded loop moves pairs whatever vec2 says (its operands are 32-byte aligned with pitches
    % 16 == 0), so it has no scalar path."""
    out = set()
    for inst in ((128, False), (256, False), (128, True), (256, True)):
        for epi in ALL_EPIS:
            if inst[1] and epi in (EPI_ACT_DUAL, EPI_ACT_GRAD, EPI_SWIGLU, EPI_SWIGLU_GRAD):
                continue
            for path in ("interior", "guarded vec", "guarded scalar"):
                if (epi == EPI_ATOMIC and path == "interior") or (epi == EPI_SWIGLU_GRAD and path == "guarded scalar"):
                    continue
                for act in ((0, 1) if epi in ACT_EPIS else (0,)):
                    for gated in ((False, True) if epi == EPI_RESID else (False,)):
                        out.add((inst, epi, path, act, gated))
    return out


@pytest.mark.parametrize("sm_count", [132, 114])
def test_matrix_reaches_every_path(sm_count):
    reached, reduce, fallback = set(), False, False
    for s in SPECS:
        vec2 = Case(s, reference=False).vec2()
        for det_ws in s.modes:
            r = route(s, vec2, min(sm_count, s.sm_limit) if s.sm_limit else sm_count, det_ws)
            reached |= paths(s, r)
            reduce |= r.reduce
            fallback |= det_ws == SMALL_WS and s.splits > 1 and r.splits == 1
    want = allowed()
    assert reached == want, (sorted(want - reached), sorted(reached - want))
    assert reduce and fallback
    assert DET_WS > SMALL_WS


def _recording(base, sigs):
    class Recording(base):
        def gemm(self, A, B, Cm, *, layout=NT, epi=EPI_BF16, C2=None, bias=None, res=None, gate=None, rows_per_gate=0,
                 res_mod=0, splits=1, act=0, alpha=1.0, aux=None, row_interleave=0):
            sigs.add((layout, epi, act if epi in ACT_EPIS else 0, None if bias is None else bias.dim(), gate is not None,
                      res_mod > 0, C2 is not None, aux is not None, splits, bool(row_interleave), A.dim() == 3))
            return super().gemm(A, B, Cm, layout=layout, epi=epi, C2=C2, bias=bias, res=res, gate=gate,
                                rows_per_gate=rows_per_gate, res_mod=res_mod, splits=splits, act=act, alpha=alpha,
                                aux=aux, row_interleave=row_interleave)
    return Recording


def test_matrix_holds_every_engine_gemm_signature():
    """(layout, epi, act, bias kind, gate, res_mod, C2, aux, splits, row_interleave, batched) of every ops.gemm call of
    one bf16 training step and sample of the S, S16 (tests/parity_common.py), SB (tests/bias_common.py) and H
    (tests/hd128_common.py) configs, on the CPU contract."""
    sigs = set()
    for name, mod, base in (("S", pc, bc.BiasEmuOps), ("S16", pc, bc.BiasEmuOps), ("SB", bc, bc.BiasEmuOps),
                            ("H", hc, hc.Emu)):
        mod.product_run(name, ops_factory=lambda d, b=base: _recording(b, sigs)(d, exact=False))
    have = {signature(s) for s in SPECS}
    assert sigs and not sigs - have, sorted(sigs - have)
    assert any(s[1] == EPI_SWIGLU for s in sigs) and any(s[9] for s in sigs) and any(s[0] == TN for s in sigs)
