"""Exponential moving average of the DiT weights (the `algorithms.ema` of configs/res_512_pretrain.yaml:3-9 and
res_512_finetune.yaml:3-9), kept in one fp32 buffer laid out like `ParamStore.flat`.

The update rides inside the optimizer step: `FlatAdamW.step(lr, reducer, ema)` launches `md_adamw_ema` instead of
`md_adamw` when an update is due, which writes ema = s * ema + (1 - s) * p_new from the registers that already hold the
new weights.  Schedule, after the optimizer step that brings the batch count to b:

* b < ema_start: nothing;
* the first b >= ema_start: ema <- p (a copy: the buffer is uninitialised before);
* afterwards, every b with b % update_interval == 0: the fused update.

With a sharded optimizer (train_step.GradReducer with `shard`) only this rank's owned shares of the buffer are valid,
exactly as for FlatAdamW.m / v; `gather_state()` completes it for checkpoints.
"""
from __future__ import annotations

import contextlib
from typing import Optional

import torch


class FlatEMA:
    """EMA of every DiT parameter.  Exactly one of `smoothing` (per update) and `half_life` (in batches, '<n>ba') is set;
    a half-life h gives smoothing = 2 ** (-update_interval / h)."""

    def __init__(self, dit, smoothing: Optional[float] = None, half_life=None, update_interval="1ba", ema_start="0ba"):
        from .trainer import parse_batches
        if (smoothing is None) == (half_life is None):
            raise ValueError("EMA: set exactly one of smoothing and half_life")
        self.update_interval = parse_batches(update_interval)
        self.ema_start = parse_batches(ema_start)
        if self.update_interval < 1 or self.ema_start < 0:
            raise ValueError(f"EMA: update_interval must be >= 1ba and ema_start >= 0ba, got {update_interval!r}, "
                             f"{ema_start!r}")
        if half_life is not None:
            hl = parse_batches(half_life)
            if hl <= 0:
                raise ValueError(f"EMA: half_life must be positive, got {half_life!r}")
            smoothing = 2.0 ** (-self.update_interval / hl)
        smoothing = float(smoothing)
        if not 0.0 <= smoothing <= 1.0:
            raise ValueError(f"EMA: smoothing must lie in [0, 1], got {smoothing}")
        self.smoothing = smoothing
        self.dit = dit
        self.ema = torch.empty_like(dit.store.flat)  # undefined until the EMA starts
        self.started = False
        self.sharded_by = None  # the GradReducer whose owned shares are the valid part of `ema` (None: all of it)

    def due(self, batch: int) -> bool:
        """Whether the optimizer step that brings the batch count to `batch` runs the fused EMA update."""
        return self.started and batch % self.update_interval == 0

    @torch.no_grad()
    def after_step(self, batch: int, segments, reducer=None) -> None:
        """Called by FlatAdamW.step after the update of `segments` (the owned shares when sharded): starts the EMA
        at the first batch >= ema_start by copying the new weights."""
        if reducer is not None:
            self.sharded_by = reducer
        if self.started or batch < self.ema_start:
            return
        flat = self.dit.store.flat
        for a, b in segments:
            self.ema[a:b].copy_(flat[a:b])
        self.started = True

    @torch.no_grad()
    def gather_state(self) -> None:
        """Make `ema` complete on every rank (checkpoints): all-gather of the owned shares."""
        if self.started and self.sharded_by is not None:
            self.sharded_by.gather_buffer(self.ema)

    def _exchange(self, ops, st) -> None:
        red = self.sharded_by
        if red is None:  # one rank, or replicated ranks: both buffers are complete
            ops.swap(st.flat, self.ema)
            return
        for a, b in red.owned:  # each rank parks its share of the other set in its own `ema`
            ops.swap(st.flat[a:b], self.ema[a:b])
        red.gather_params(st)
        if red.stream is not None:
            torch.cuda.current_stream(st.device).wait_stream(red.stream)

    @contextlib.contextmanager
    def applied(self):
        """Inside the block the model's weights are the EMA weights (evaluation, sampling, export); on exit the training
        weights are back, bit for bit.  Does nothing before the EMA has started.  Sharded: the owned shares are swapped
        and `flat` is all-gathered, so every rank holds the full EMA weights without a full-size copy of anything."""
        if not self.started:
            yield self
            return
        dit = self.dit
        st, ops = dit.store, dit.engine.ops
        for part in list(st.param_ready):  # a parameter all-gather may still be in flight
            torch.cuda.current_stream(st.device).wait_event(st.param_ready.pop(part))
        with torch.no_grad():
            self._exchange(ops, st)
        dit.mark_weights_dirty()
        try:
            yield self
        finally:
            with torch.no_grad():
                self._exchange(ops, st)
            dit.mark_weights_dirty()

    def state_tensors(self):
        """{"dit.<param>": EMA value (host)} in the layout's parameter order; call gather_state() first when sharded."""
        return {f"dit.{name}": self.ema[off:off + _numel(shape)].view(shape).cpu()
                for name, (off, shape) in self.dit.store.layout.slots.items()}

    @torch.no_grad()
    def load_tensors(self, weights: dict) -> bool:
        """Inverse of state_tensors(); False (and nothing loaded) unless every parameter is present with its shape."""
        slots = self.dit.store.layout.slots
        for name, (_, shape) in slots.items():
            t = weights.get(f"dit.{name}")
            if not torch.is_tensor(t) or tuple(t.shape) != tuple(shape):
                return False
        for name, (off, shape) in slots.items():
            self.ema[off:off + _numel(shape)].copy_(weights[f"dit.{name}"].reshape(-1))
        self.started = True
        self.sharded_by = None  # complete on every rank
        return True


def _numel(shape) -> int:
    n = 1
    for d in shape:
        n *= d
    return n
