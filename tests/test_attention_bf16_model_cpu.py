"""The bf16 attention error model of tests/test_attention_bf16_gpu.py has teeth: its cases, run on emulations of the
bf16 contract (oracle.emu_ops.EmuOps) with one injected fault each, fail -- each fault at least one case -- while the
unmodified contract and one that skips the bf16 rounding of P pass everywhere.  Each fault prints by how much its
worst case missed (the largest error as a fraction of its bound, or row |z| / 6)."""
import functools
import math

import pytest
import torch

from oracle.emu_ops import EmuOps
from tests.test_attention_bf16_gpu import Case, metrics, run_bwd, run_fwd

# ragged query tiles (100, 130, 65), ragged key tiles (200, 33, 81, 77), more than one key tile (200, 81), 2+ heads
SHAPES = [(2, 3, 100, 200, 64), (2, 2, 130, 33, 32), (2, 2, 65, 81, 64), (2, 3, 64, 77, 32), (1, 2, 130, 200, 128)]


@functools.lru_cache(maxsize=None)
def _case(shape):
    return Case(*shape)


def _per_sample(x, B, T, keep):
    """rows [b*T + t for t in keep] of every sample b, as a [B*len(keep), cols] tensor."""
    return x.reshape(B, T, -1)[:, keep].reshape(-1, x.shape[1])


class PaddedKey(EmuOps):
    """The key mask of a ragged last key tile lets one zero-padded key (score 0, value 0) into the softmax."""

    def attn_fwd(self, q, k, v, o, lse, B, H, Tq, Tk, hd):
        if Tk % 64 == 0:
            return super().attn_fwd(q, k, v, o, lse, B, H, Tq, Tk, hd)
        pad = lambda x: torch.cat([x.reshape(B, Tk, -1), torch.zeros(B, 1, x.shape[1], dtype=x.dtype)], 1).reshape(-1, x.shape[1])
        super().attn_fwd(q, pad(k), pad(v), o, lse, B, H, Tq, Tk + 1, hd)


class DroppedKey(EmuOps):
    """The last key of every sample is masked out."""

    def attn_fwd(self, q, k, v, o, lse, B, H, Tq, Tk, hd):
        if Tk == 1:
            return super().attn_fwd(q, k, v, o, lse, B, H, Tq, Tk, hd)
        keep = slice(0, Tk - 1)
        super().attn_fwd(q, _per_sample(k, B, Tk, keep), _per_sample(v, B, Tk, keep), o, lse, B, H, Tq, Tk - 1, hd)


class UnwrittenRow(EmuOps):
    """The last row of a ragged query tile is never stored."""

    def attn_fwd(self, q, k, v, o, lse, B, H, Tq, Tk, hd):
        rows = [b * Tq + Tq - 1 for b in range(B)] if Tq % 64 else []
        kept = o[rows].clone()
        super().attn_fwd(q, k, v, o, lse, B, H, Tq, Tk, hd)
        o[rows] = kept


class NaturalLse(EmuOps):
    """lse stored in natural-log units instead of log2."""

    def attn_fwd(self, q, k, v, o, lse, B, H, Tq, Tk, hd):
        super().attn_fwd(q, k, v, o, lse, B, H, Tq, Tk, hd)
        lse.mul_(math.log(2.0))


class LastHeadLeft(EmuOps):
    """The last head's output is written one head to the left; its own columns stay unwritten."""

    def attn_fwd(self, q, k, v, o, lse, B, H, Tq, Tk, hd):
        before = o.clone()
        super().attn_fwd(q, k, v, o, lse, B, H, Tq, Tk, hd)
        if H > 1:
            last = o[:, (H - 1) * hd:H * hd].clone()
            o[:, (H - 1) * hd:H * hd] = before[:, (H - 1) * hd:H * hd]
            o[:, (H - 2) * hd:(H - 1) * hd] = last


class WrongHeadDelta(EmuOps):
    """The backward's delta = sum dO o is taken from the un-rounded o of the next head."""

    def attn_bwd(self, dout, q, k, v, o, lse, delta, dq, dk, dv, B, H, Tq, Tk, hd):
        o32, l32 = torch.zeros(B * Tq, H * hd), torch.zeros(B, H, Tq)
        EmuOps("cpu", exact=True).attn_fwd(q.float(), k.float(), v.float(), o32, l32, B, H, Tq, Tk, hd)
        wrong = o32.reshape(-1, H, hd).roll(-1, dims=1).reshape(-1, H * hd)
        super().attn_bwd(dout, q, k, v, wrong, lse, delta, dq, dk, dv, B, H, Tq, Tk, hd)


class DqMissesLastKeyTile(EmuOps):
    """dq leaves out the keys of the last 64-key tile."""

    def attn_bwd(self, dout, q, k, v, o, lse, delta, dq, dk, dv, B, H, Tq, Tk, hd):
        super().attn_bwd(dout, q, k, v, o, lse, delta, dq, dk, dv, B, H, Tq, Tk, hd)
        if Tk > 64:
            kt = 64 * ((Tk - 1) // 64)
            ks, vs = _per_sample(k, B, Tk, slice(0, kt)), _per_sample(v, B, Tk, slice(0, kt))
            scratch = torch.zeros(B * kt, ks.shape[1], dtype=dk.dtype)
            super().attn_bwd(dout, q, ks, vs, o, lse, delta.clone(), dq, scratch, scratch.clone(), B, H, Tq, kt, hd)


class InvLBf16(EmuOps):
    """1/l is rounded to bf16 before it normalises the row (a rounding point the contract does not have)."""

    def attn_fwd(self, q, k, v, o, lse, B, H, Tq, Tk, hd):
        qh, kh, vh = self._heads(q, B, Tq, H, hd), self._heads(k, B, Tk, H, hd), self._heads(v, B, Tk, H, hd)
        s = qh @ kh.mT / math.sqrt(hd)
        m = s.amax(-1, keepdim=True)
        p = torch.exp(s - m)
        l = p.sum(-1, keepdim=True)
        out = (self._r(p) @ vh) * self._r(1.0 / l)
        o[:, :H * hd].copy_(out.permute(0, 2, 1, 3).reshape(B * Tq, H * hd))
        lse.copy_(((m + l.log()) * 1.4426950408889634)[..., 0])


class NoPRounding(EmuOps):
    """Control: P (and dS) not rounded to bf16 before their products; only the stored outputs are bf16."""

    def _r(self, t):
        return t


def _worst(ops_cls):
    """Largest metric over every case, and the case and check it came from."""
    best = (-1.0, None, None)
    for shape in SHAPES:
        c = _case(shape)
        ops = ops_cls("cpu")
        m = metrics(c, run_fwd(ops, c), run_bwd(ops, c))
        n, v = max(m.items(), key=lambda kv: kv[1])
        if v > best[0]:
            best = (v, c.tag(), n)
    return best


@pytest.mark.parametrize("fault", [PaddedKey, DroppedKey, UnwrittenRow, NaturalLse, LastHeadLeft, WrongHeadDelta,
                                   DqMissesLastKeyTile, InvLBf16], ids=lambda f: f.__name__)
def test_injected_fault_fails_a_case(fault):
    v, tag, n = _worst(fault)
    print(f"\n[{fault.__name__}] worst: {n} at {v:.3g}x its bound ({tag})", end="")
    assert v > 1.0, f"{fault.__name__} passes every case (worst {n} {v:.3g})"


@pytest.mark.parametrize("control", [EmuOps, NoPRounding], ids=lambda f: f.__name__)
def test_contract_and_unrounded_p_pass(control):
    v, tag, n = _worst(control)
    print(f"\n[{control.__name__}] worst: {n} at {v:.3g} of its bound ({tag})", end="")
    assert v <= 1.0, (n, v, tag)
