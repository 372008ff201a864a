"""Shared pieces of the weight-EMA tests: the CPU contracts of md_adamw_ema / md_swap_f32 and the plain torch
restatement of the EMA schedule."""
import math

import torch

from oracle.emu_ops import EmuOps


class EMAEmuOps(EmuOps):
    """EmuOps plus the CPU contracts of md_adamw_ema and md_swap_f32."""

    def adamw_ema(self, p, g, m, v, sumsq, clip, lr, beta1, beta2, eps, wd, step, ema, smoothing, nonfinite=None):
        """adamw(...) then ema = s * ema + (1 - s) * p_new; a non-finite sumsq writes nothing and raises the flag."""
        if sumsq is not None and not math.isfinite(float(sumsq[0])):
            self.launches += 1
            if nonfinite is not None:
                nonfinite.fill_(1)
            return
        self.adamw(p, g, m, v, sumsq, clip, lr, beta1, beta2, eps, wd, step, nonfinite)
        ema.copy_(ema_update(ema, p, smoothing))

    def swap(self, a, b):
        self.launches += 1
        assert a.numel() == b.numel() and a.dtype == b.dtype == torch.float32
        pa, pb, nbytes = a.data_ptr(), b.data_ptr(), 4 * a.numel()
        if pa == pb or (pa < pb + nbytes and pb < pa + nbytes):
            raise RuntimeError("md_swap_f32: the two ranges overlap")
        t = a.clone()
        a.copy_(b)
        b.copy_(t)


def ema_update(ema, p, s):
    """One EMA update as written in torch: s * ema + (1 - s) * p."""
    return s * ema + (1.0 - s) * p


def ema_reference(weights, smoothing, ema_start, update_interval):
    """The EMA after the last of `weights` (weights[i] = the flat weights after batch i + 1), or None if it has not
    started: copy at the first batch >= ema_start, then an update at every later batch divisible by update_interval."""
    ema = None
    for i, w in enumerate(weights):
        b = i + 1
        if ema is None:
            if b >= ema_start:
                ema = w.clone()
        elif b % update_interval == 0:
            ema = ema_update(ema, w, smoothing)
    return ema


def ulp_bound(ema_prev, p_new, s):
    """One fp32 ulp of the largest of |s * ema|, |(1 - s) * p| and the result, elementwise: the tolerance of an EMA
    update whose FMA contraction may differ from torch's.  The two terms can cancel, so an ulp of the result alone is too
    tight; and a same-sign sum can round up into the next binade, where an ulp of the larger term is half the step."""
    big = torch.maximum((s * ema_prev).abs(), ((1.0 - s) * p_new).abs())
    big = torch.maximum(big, ema_update(ema_prev, p_new, s).abs())
    return torch.nextafter(big, torch.full_like(big, math.inf)) - big
