"""A Composer-free training step over the drop-in model: microbatching, data-parallel gradient mean over NCCL,
global-norm clipping and AdamW -- what composer.Trainer does around `model(batch)` in the reference
(train.py:103-123; configs/res_256_pretrain.yaml:6-8 clip 0.25, :50-57 AdamW, :111 microbatch 256, :117-118
FSDP SHARD_GRAD_OP: gradient reduce-scatter, optimizer step on the local shard, parameter all-gather).

Default with more than one rank ("sharded", the SHARD_GRAD_OP arithmetic on replicated weights): the flat gradient
buffer (params.ParamStore.grad) is REDUCE-SCATTERED (mean) in a few contiguous ranges on a side stream -- the backbone
ranges from inside the last microbatch's backward, as soon as they are final, so that they overlap the patch-mixer and
stem backward -- each rank runs clip + AdamW on its 1/N of every range, and the updated fp32 parameters are ALL-GATHERED
on the side stream: the front range (stem, patch mixer) first, the backbone range under the next step's patch-mixer
forward (params.ParamStore.refresh_copies waits per part).  The path shards by batch: no activation traffic.
MD_SHARD_OPT=0 (or a world size that does not divide the range alignment) falls back to the replicated form: one
all-reduce (mean) per range and the full AdamW on every rank.
"""
from __future__ import annotations

import os
from typing import Dict, Iterable, List, Optional

import torch
import torch.distributed as dist


class FlatAdamW:
    """Clip-by-global-norm + AdamW over the flat parameter buffer: two kernel launches per step."""

    def __init__(self, dit, lr=2.4e-4, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.1, clip_norm: Optional[float] = 0.25):
        self.dit = dit
        self.lr, self.betas, self.eps, self.wd, self.clip = lr, betas, eps, weight_decay, clip_norm
        st = dit.store
        self.m = torch.zeros_like(st.flat)
        self.v = torch.zeros_like(st.flat)
        self.sumsq = torch.zeros(1, dtype=torch.float32, device=st.device)
        self.nonfinite = torch.zeros(1, dtype=torch.int32, device=st.device)  # set by md_adamw when it skipped a step
        self.t = 0

    @torch.no_grad()
    def step(self, lr: Optional[float] = None, reducer: Optional["GradReducer"] = None, ema=None):
        """`reducer` with `shard` set: the gradient is only valid on this rank's shares (reduce-scatter), so clip + AdamW
        run on those segments -- the squared norm is summed over ranks -- and the updated parameters are all-gathered.
        `ema` (ema.FlatEMA): when an EMA update is due at this step, md_adamw_ema replaces md_adamw on the same segments;
        otherwise the launches are those of a step without EMA."""
        eng = self.dit.engine
        st, o = eng.store, eng.ops
        self.t += 1
        sharded = reducer is not None and reducer.shard
        segs = reducer.owned if sharded else [(0, st.flat.numel())]
        # the squared gradient norm is always taken: it scales the clip AND guards the update -- a non-finite norm
        # (NaN / Inf loss, callbacks.py:47-64) makes md_adamw leave weights and moments untouched and raise `nonfinite`
        self.sumsq.zero_()
        for a, b in segs:
            o.sumsq(st.grad[a:b], self.sumsq)
        if sharded:
            dist.all_reduce(self.sumsq, op=dist.ReduceOp.SUM, group=reducer.group)
        elif reducer is not None and reducer.world > 1:
            # replicated form: every rank holds the same gradient, but md_sumsq adds its block partials atomically, so the
            # norm can differ in the last bit from rank to rank -- and with it the clip factor and every updated weight.
            # Rank 0's value is the value: replicas stay bit-identical (there is no parameter broadcast to repair drift).
            dist.broadcast(self.sumsq, src=0, group=reducer.group)
        fused = ema is not None and ema.due(self.t)
        for a, b in segs:
            if fused:
                o.adamw_ema(st.flat[a:b], st.grad[a:b], self.m[a:b], self.v[a:b], self.sumsq, float(self.clip or 0.0),
                            float(lr if lr is not None else self.lr), self.betas[0], self.betas[1], self.eps, self.wd,
                            self.t, ema.ema[a:b], ema.smoothing, nonfinite=self.nonfinite)
            else:
                o.adamw(st.flat[a:b], st.grad[a:b], self.m[a:b], self.v[a:b], self.sumsq, float(self.clip or 0.0),
                        float(lr if lr is not None else self.lr), self.betas[0], self.betas[1], self.eps, self.wd, self.t,
                        nonfinite=self.nonfinite)
        if ema is not None:
            ema.after_step(self.t, segs, reducer if sharded else None)  # the start copy reads this rank's new weights
        if sharded:
            reducer.gather_params(st)
            self.sharded_by = reducer
        self.dit.mark_weights_dirty()

    sharded_by = None  # the GradReducer whose shares the moments m / v are valid on (None: valid everywhere)

    @torch.no_grad()
    def gather_state(self):
        """Make m / v complete on every rank (checkpoints): all-gather of the owned shares."""
        if self.sharded_by is not None:
            self.sharded_by.gather_buffer(self.m)
            self.sharded_by.gather_buffer(self.v)

    def zero_grad(self):
        self.dit.store.grad.zero_()


class GradReducer:
    """Data-parallel mean of the flat gradient over the default process group (NCCL on GPUs, gloo in CPU tests).

    The flat layout ends with blocks.* and final_layer.* (params.ParamLayout keeps the reference order for them), and
    backward finishes those first.  `early_ranges` (element ranges that are final once the backbone backward is done)
    are therefore all-reduced on a side stream while the patch-mixer and stem backward still run; `reduce()` then
    handles the remainder and joins the streams."""

    def __init__(self, store, buckets: int = 4, group=None, ops=None, reserve_sms: Optional[int] = None,
                 overlap: Optional[bool] = None, shard: Optional[bool] = None):
        """`ops` (the model's CudaOps) + `reserve_sms`: while the early all-reduce is in flight the persistent GEMM grids
        leave that many SMs to NCCL's CTAs -- a statically scheduled one-CTA-per-SM grid whose last CTAs cannot become resident
        until the collective's CTAs retire would otherwise run its tail at half speed."""
        self.store = store
        self.ops = ops
        self.reserve = int(os.environ.get("MD_DDP_SM_RESERVE", "16")) if reserve_sms is None else int(reserve_sms)
        self.overlap = (os.environ.get("MD_DDP_OVERLAP", "1") != "0") if overlap is None else bool(overlap)
        self.sm_count = (torch.cuda.get_device_properties(store.grad.device).multi_processor_count
                         if store.grad.is_cuda else 0)
        self.grad = store.grad
        self.group = group
        self.world = dist.get_world_size(group) if dist.is_available() and dist.is_initialized() else 1
        lay = store.layout
        n = self.grad.numel()
        # early part 1: everything from the first blocks.* parameter to the end of the buffer
        first = min(off for name, (off, _) in lay.slots.items()
                    if (name.startswith("blocks.") or name.startswith("final_layer."))
                    and not name.endswith("adaLN_modulation.1.weight") and not name.endswith("adaLN_modulation.1.bias")
                    and not name.endswith("cross_attn.kv_linear.weight") and not name.endswith("cross_attn.kv_linear.bias"))
        self.early = [(first, n)]
        if lay.kv_back is not None:  # part 2: the stacked backbone K/V projection, its bias stack included
            self.early.append(lay.kv_back)
        # late = the complement
        cuts = sorted(self.early)
        self.late, pos = [], 0
        for a, b in cuts:
            if a > pos:
                self.late.append((pos, a))
            pos = max(pos, b)
        if pos < n:
            self.late.append((pos, n))
        self.buckets = buckets
        self.stream = torch.cuda.Stream(device=self.grad.device) if self.grad.is_cuda else None
        self._early_done = False
        self.rank = dist.get_rank(group) if self.world > 1 else 0
        ra = lay.RANGE_ALIGN
        can_shard = (self.world > 1 and ra % (8 * self.world) == 0 and n % ra == 0
                     and all(a % ra == 0 and b % ra == 0 for a, b in self.early + self.late))
        want = (os.environ.get("MD_SHARD_OPT", "1") != "0") if shard is None else bool(shard)
        self.shard = bool(want and can_shard)
        # this rank's share of every bucket: [a + r * (b - a) / W, a + (r + 1) * (b - a) / W)
        self.owned = [self._mine(a, b) for a, b in self._split(self.early) + self._split(self.late)] if self.shard else []

    def _mine(self, a, b):
        ch = (b - a) // self.world
        return (a + self.rank * ch, a + (self.rank + 1) * ch)

    def _split(self, ranges):
        out = []
        for a, b in ranges:
            per = max(1, (b - a + self.buckets - 1) // self.buckets)
            per = (per + 1023) // 1024 * 1024
            out += [(i, min(b, i + per)) for i in range(a, b, per)]
        return out

    def _allreduce(self, ranges):
        """Mean over ranks of every bucket of `ranges`: all-reduce, or (sharded) reduce-scatter in place -- afterwards
        only this rank's share of each bucket holds the mean, the rest of the bucket is scratch."""
        if self.stream is None:  # gloo (CPU tests): no AVG, no reduce_scatter_tensor -- same arithmetic through all_reduce
            for a, b in self._split(ranges):
                dist.all_reduce(self.grad[a:b], op=dist.ReduceOp.SUM, group=self.group)
                if self.shard:
                    ma, mb = self._mine(a, b)
                    mine = self.grad[ma:mb] / self.world
                    self.grad[a:b].fill_(float("nan"))  # what a reduce-scatter leaves undefined must not be read
                    self.grad[ma:mb] = mine
                else:
                    self.grad[a:b].div_(self.world)
            return
        self.stream.wait_stream(torch.cuda.current_stream(self.grad.device))
        with torch.cuda.stream(self.stream):
            for a, b in self._split(ranges):
                if self.shard:
                    ma, mb = self._mine(a, b)
                    dist.reduce_scatter_tensor(self.grad[ma:mb], self.grad[a:b], op=dist.ReduceOp.AVG, group=self.group)
                else:
                    dist.all_reduce(self.grad[a:b], op=dist.ReduceOp.AVG, group=self.group)

    def gather_buffer(self, buf):
        """All-gather the owned shares of a flat buffer laid out like the gradient (optimizer moments), in place."""
        for a, b in self._split(self.early) + self._split(self.late):
            ma, mb = self._mine(a, b)
            dist.all_gather_into_tensor(buf[a:b], buf[ma:mb].clone(), group=self.group)

    def gather_params(self, store):
        """All-gather the updated parameters: front ranges first, then the backbone ranges; on the side stream, with one
        event per part that ParamStore.refresh_copies waits on -- the backbone part travels under the next step's
        patch-mixer forward."""
        flat = store.flat
        parts = (("front", self._split(self.late)), ("back", self._split(self.early)))
        if self.stream is None:
            for _, subs in parts:
                for a, b in subs:
                    ma, mb = self._mine(a, b)
                    dist.all_gather_into_tensor(flat[a:b], flat[ma:mb].clone(), group=self.group)
            return
        self.stream.wait_stream(torch.cuda.current_stream(flat.device))
        with torch.cuda.stream(self.stream):
            for part, subs in parts:
                for a, b in subs:
                    ma, mb = self._mine(a, b)
                    dist.all_gather_into_tensor(flat[a:b], flat[ma:mb], group=self.group)  # in place (NCCL allows it)
                ev = torch.cuda.Event()
                ev.record(self.stream)
                store.param_ready[part] = ev

    def reduce_early(self):
        """Called from inside the LAST microbatch's backward once the backbone gradients are final."""
        if self.world == 1 or not self.overlap:
            return
        self._allreduce(self.early)
        self._early_done = True
        if self.ops is not None and self.reserve > 0 and self.sm_count > self.reserve:
            self.ops.sm_limit = self.sm_count - self.reserve

    def reduce(self):
        """All-reduce (mean) whatever has not been reduced yet and make the result visible to the compute stream."""
        if self.world == 1:
            return
        self._allreduce(self.late if self._early_done else [(0, self.grad.numel())])
        self._early_done = False
        if self.stream is not None:
            torch.cuda.current_stream(self.grad.device).wait_stream(self.stream)
        if self.ops is not None:
            self.ops.sm_limit = 0


def train_step(model, batch: Dict[str, torch.Tensor], optimizer: FlatAdamW, reducer: Optional[GradReducer] = None,
               microbatch: int = 256, lr: Optional[float] = None, ema=None) -> torch.Tensor:
    """One optimisation step over `batch` (this rank's share of the global batch) at learning rate `lr` (default: the
    optimizer's base rate), with the weight EMA `ema` (ema.FlatEMA) if given: returns the mean loss (device)."""
    B = batch["image_latents"].shape[0]
    total = None
    eng = model.dit.engine
    starts = list(range(0, B, microbatch))
    for s in starts:
        mb = {k: v[s:s + microbatch] for k, v in batch.items()}
        n = mb["image_latents"].shape[0]
        loss = model(mb)[0]
        last = s == starts[-1]
        eng.on_backbone_grads_ready = reducer.reduce_early if (reducer is not None and last) else None
        (loss * (n / B)).backward()  # Composer's microbatch loss scaling
        eng.on_backbone_grads_ready = None
        total = loss.detach() * (n / B) if total is None else total + loss.detach() * (n / B)
    if reducer is not None:
        reducer.reduce()
    optimizer.step(lr, reducer, ema)
    optimizer.zero_grad()
    return total
