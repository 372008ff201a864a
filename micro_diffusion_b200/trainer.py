"""Composer-free step driver (SURVEY.md §8 f-2): what `composer.Trainer` does around the hot path in the
reference's four YAML configs, and nothing more.

* learning-rate schedule `composer.optim.CosineAnnealingWithWarmupScheduler(t_warmup, alpha_f)`
  (configs/res_256_pretrain.yaml:58-61): linear 0 -> 1 over `t_warmup` batches, then cosine from 1 to `alpha_f`
  over the remaining `max_duration - t_warmup` batches (Composer's `scale_warmup=False` default);
* `device_train_microbatch_size` (configs/res_256_pretrain.yaml:111) via train_step.train_step;
* `NaNCatcher.after_loss` (micro_diffusion/models/callbacks.py:45-65);
* checkpoints in Composer's nesting (`state/model/dit.<key>`, `state/optimizers`, `state/timestamp`) with
  `load_weights_only`, `load_strict_model_weights` and `load_ignore_keys` glob semantics
  (configs/res_512_pretrain.yaml:117-123 drops `state/model/dit.pos_embed` when going 256 -> 512).

train.py:28-38 halves the learning rate of parameters whose NAME contains "moe"; no MicroDiT parameter name does
(the expert banks are `blocks.N.mlp.{w1,w2,gate.weight}`), so the reference trains every parameter at one rate and
so does FlatAdamW.
"""
from __future__ import annotations

import fnmatch
import math
import os
import time
from typing import Callable, Dict, Iterable, List, Optional, Sequence

import torch

from .ema import FlatEMA
from .train_step import FlatAdamW, GradReducer, train_step


def parse_batches(duration) -> int:
    """'2500ba' -> 2500 (the only time unit the reference's configs use)."""
    if isinstance(duration, int):
        return duration
    s = str(duration).strip()
    if not s.endswith("ba"):
        raise ValueError(f"only batch durations ('<n>ba') are supported, got {duration!r}")
    return int(s[:-2])


def cosine_with_warmup(step: int, t_warmup: int, t_max: int, alpha_f: float = 0.0) -> float:
    """LR multiplier at optimizer step `step` (0-based count of completed batches)."""
    if t_warmup > 0 and step < t_warmup:
        return step / t_warmup
    span = max(1, t_max - t_warmup)
    frac = min(1.0, max(0.0, (step - t_warmup) / span))
    return alpha_f + (1.0 - alpha_f) * 0.5 * (1.0 + math.cos(math.pi * frac))


def lr_multiplier(kind: str, step: int, t_warmup: int, t_max: int, alpha: float = 1.0, alpha_f: float = 0.0) -> float:
    """The three Composer schedulers the reference's configs name (configs/res_256_pretrain.yaml:58-61,
    res_256_finetune.yaml:58-60, res_512_pretrain.yaml:63-66), as LR multipliers at optimizer step `step`."""
    if kind == "cosine_with_warmup":
        return cosine_with_warmup(step, t_warmup, t_max, alpha_f)
    if kind == "constant":
        return alpha
    if kind == "constant_with_warmup":
        return alpha * (step / t_warmup) if (t_warmup > 0 and step < t_warmup) else alpha
    raise ValueError(f"unknown LR schedule {kind!r}")


SCHEDULERS = {"CosineAnnealingWithWarmupScheduler": "cosine_with_warmup", "ConstantScheduler": "constant",
              "ConstantWithWarmupScheduler": "constant_with_warmup"}


# ------------------------------------------------------------------------------------------ checkpoints
def _flatten(tree, prefix=""):
    for k, v in tree.items():
        path = f"{prefix}/{k}" if prefix else k
        if isinstance(v, dict):
            yield from _flatten(v, path)
        else:
            yield path, v


def _drop_ignored(tree: dict, patterns: Sequence[str]) -> List[str]:
    """Composer's `load_ignore_keys`: '/'-separated glob paths into the checkpoint dict; matches are deleted."""
    dropped = []
    for path, _ in list(_flatten(tree)):
        if any(fnmatch.fnmatchcase(path, pat) for pat in patterns):
            node = tree
            parts = path.split("/")
            # keys themselves may contain '/'-free dots only, so a plain walk is enough
            for p in parts[:-1]:
                node = node[p]
            del node[parts[-1]]
            dropped.append(path)
    return dropped


def _rng_state(device) -> dict:
    st = {"torch": torch.get_rng_state()}
    if torch.device(device).type == "cuda":
        st["cuda"] = torch.cuda.get_rng_state(device)
    return st


_EMA_KEYS = ("ema_weights", "started", "smoothing", "update_interval", "ema_start")


def save_checkpoint(path: str, model, optimizer: Optional[FlatAdamW], batch: int, rank: int = 0, loader=None,
                    world: int = 1, keep: Optional[int] = None, ema: Optional[FlatEMA] = None) -> None:
    """Rank 0 writes; parameters are replicated so there is nothing to gather except the per-rank RNG states
    (every rank calls this).  `loader.state_dict()` (epoch, batch in epoch) and the RNG states are what Composer's
    checkpoint restores so that a resumed run continues the sample / noise / mask streams instead of replaying them.
    `keep` = Composer's save_num_checkpoints_to_keep (configs/res_256_pretrain.yaml:112): older ba*.pt are removed.
    `ema`: its weights go to state["algorithms"]["EMA"]["ema_weights"] ("dit.<param>" keys, empty before the EMA has
    started); state["model"] stays the training weights."""
    rng = [_rng_state(model.dit.store.device)]
    if optimizer is not None:
        optimizer.gather_state()  # sharded optimizer: every rank takes part in completing the moments
    if ema is not None:
        ema.gather_state()
    if world > 1:
        import torch.distributed as dist
        gathered = [None] * world
        dist.all_gather_object(gathered, rng[0])
        rng = gathered
    if rank != 0:
        return
    for ev in list(model.dit.store.param_ready.values()):  # a parameter all-gather may still be in flight
        ev.synchronize()
    sd = {f"dit.{k}": v.detach().cpu() for k, v in model.dit.state_dict().items()}
    state = {"model": sd, "timestamp": {"batch": int(batch)}}
    if loader is not None and hasattr(loader, "state_dict"):
        state["dataset_state"] = loader.state_dict()
    if optimizer is not None:
        state["optimizers"] = {"FlatAdamW": {"exp_avg": optimizer.m.cpu(), "exp_avg_sq": optimizer.v.cpu(),
                                             "step": optimizer.t,
                                             "layout": list(model.dit.store.layout.slots.keys())}}
    if ema is not None:
        state["algorithms"] = {"EMA": {"ema_weights": ema.state_tensors() if ema.started else {},
                                       "started": bool(ema.started), "smoothing": ema.smoothing,
                                       "update_interval": ema.update_interval, "ema_start": ema.ema_start}}
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    tmp = path + ".tmp"
    torch.save({"state": state, "rng": rng}, tmp)
    os.replace(tmp, path)
    if keep is not None and keep > 0:
        folder = os.path.dirname(os.path.abspath(path))
        olds = sorted((f for f in os.listdir(folder) if f.startswith("ba") and f.endswith(".pt") and f[2:-3].isdigit()),
                      key=lambda f: int(f[2:-3]))
        for f in olds[:-keep]:
            os.remove(os.path.join(folder, f))


def load_checkpoint(path: str, model, optimizer: Optional[FlatAdamW] = None, load_weights_only: bool = False,
                    load_strict_model_weights: bool = True, load_ignore_keys: Sequence[str] = (), loader=None,
                    rank: int = 0, ema: Optional[FlatEMA] = None) -> int:
    """Returns the batch count to resume from (0 with `load_weights_only`).  A full load also restores this rank's
    RNG state, the loader position and the EMA saved by `save_checkpoint` (dropped like any other entry by
    `load_ignore_keys`).  An EMA entry that is missing, incomplete (e.g. partly dropped) or not started leaves `ema`
    unstarted: it then starts again on its own schedule.  The schedule itself (smoothing, interval, start) is `ema`'s."""
    ckpt = torch.load(path, map_location="cpu", weights_only=False)
    if load_ignore_keys:
        _drop_ignored(ckpt, list(load_ignore_keys))
    sd = ckpt["state"]["model"]
    dit_sd = {k[len("dit."):]: v for k, v in sd.items() if k.startswith("dit.")}
    missing, unexpected = model.dit.load_state_dict(dit_sd, strict=False)
    if load_strict_model_weights and (missing or unexpected):
        raise RuntimeError(f"checkpoint does not match the model: missing {list(missing)}, unexpected {list(unexpected)}")
    model.dit.mark_weights_dirty()
    if load_weights_only:
        return 0
    opt = ckpt["state"].get("optimizers", {}).get("FlatAdamW")
    if optimizer is not None and opt is not None:
        if opt["layout"] != list(model.dit.store.layout.slots.keys()):
            raise RuntimeError("optimizer state was saved with a different parameter layout")
        optimizer.m.copy_(opt["exp_avg"])
        optimizer.v.copy_(opt["exp_avg_sq"])
        optimizer.t = int(opt["step"])
    if ema is not None:
        ema.started = False
        entry = _ema_entry(ckpt)
        if entry is not None:
            ema.load_tensors(entry["ema_weights"])
    ds_state = ckpt["state"].get("dataset_state")
    if loader is not None and ds_state is not None and hasattr(loader, "load_state_dict"):
        loader.load_state_dict(ds_state)
    rng = ckpt.get("rng")
    if isinstance(rng, list) and rank < len(rng) and rng[rank] is not None:
        torch.set_rng_state(rng[rank]["torch"])
        if "cuda" in rng[rank] and torch.device(model.dit.store.device).type == "cuda":
            torch.cuda.set_rng_state(rng[rank]["cuda"], model.dit.store.device)
    return int(ckpt["state"].get("timestamp", {}).get("batch", 0))


def _ema_entry(ckpt: dict) -> Optional[dict]:
    """state["algorithms"]["EMA"] if it holds started EMA weights and every schedule field, else None."""
    entry = (ckpt["state"].get("algorithms") or {}).get("EMA")
    if not isinstance(entry, dict) or any(k not in entry for k in _EMA_KEYS):
        return None
    if not entry["started"] or not isinstance(entry["ema_weights"], dict) or not entry["ema_weights"]:
        return None
    return entry


def ema_state_dict(path: str) -> dict:
    """A DiT state_dict of the checkpoint's EMA weights plus its buffers (pos_embed, ...), for
    `model.dit.load_state_dict(ema_state_dict(path))` -- sampling from the EMA.  Raises if the checkpoint holds no
    complete EMA entry."""
    ckpt = torch.load(path, map_location="cpu", weights_only=False)
    entry = _ema_entry(ckpt)
    if entry is None:
        raise ValueError(f"{path} holds no (complete) EMA weights")
    sd = {k[len("dit."):]: v for k, v in ckpt["state"]["model"].items() if k.startswith("dit.")}
    for k, v in entry["ema_weights"].items():
        name = k[len("dit."):]
        if name not in sd:
            raise ValueError(f"{path}: EMA weight {k} has no counterpart in the model state")
        sd[name] = v
    return sd


# ------------------------------------------------------------------------------------------ the loop
class Trainer:
    """fit() = for each batch: microbatched forward/backward, gradient mean, clip + AdamW at the scheduled LR.

    `train_dataloader` yields the reference's batch dict (latents_loader.py:43-70) with this rank's share of the
    global batch, on the host (pinned) or already on the device."""

    def __init__(self, model, train_dataloader: Iterable[Dict[str, torch.Tensor]], max_duration="50000ba",
                 lr: float = 2.4e-4, betas=(0.9, 0.999), eps: float = 1e-8, weight_decay: float = 0.1,
                 clip_norm: Optional[float] = 0.25, t_warmup="2500ba", alpha_f: float = 0.33,
                 scheduler: str = "cosine_with_warmup", alpha: float = 1.0,
                 device_train_microbatch_size: int = 256, save_folder: Optional[str] = None, save_interval="2500ba",
                 load_path: Optional[str] = None, load_weights_only: bool = False,
                 load_strict_model_weights: bool = True, load_ignore_keys: Sequence[str] = (),
                 log_every: int = 50, log_fn: Callable[[str], None] = print,
                 eval_dataloader: Optional[Iterable[Dict[str, torch.Tensor]]] = None, eval_interval="0ba",
                 save_num_checkpoints_to_keep: Optional[int] = None, ema_smoothing: Optional[float] = None,
                 ema_half_life=None, ema_update_interval="1ba", ema_start="0ba"):
        """`ema_smoothing` or `ema_half_life` (Composer's EMA arguments, configs/res_512_pretrain.yaml:3-9) keeps an
        exponential moving average of the weights (ema.FlatEMA) in `self.ema`; without either there is none."""
        import torch.distributed as dist
        self.model = model
        self.loader = train_dataloader
        self.t_max = parse_batches(max_duration)
        self.t_warmup = parse_batches(t_warmup)
        self.alpha_f = alpha_f
        self.scheduler, self.alpha = scheduler, alpha
        lr_multiplier(scheduler, 0, 1, 2)  # validate the name early
        self.microbatch = device_train_microbatch_size
        self.save_folder, self.save_interval = save_folder, parse_batches(save_interval)
        self.save_keep = save_num_checkpoints_to_keep if (save_num_checkpoints_to_keep or 0) > 0 else None
        self.log_every, self.log = log_every, log_fn
        self.eval_loader, self.eval_interval = eval_dataloader, parse_batches(eval_interval)
        self.last_eval_loss: Optional[float] = None
        self.rank = dist.get_rank() if dist.is_available() and dist.is_initialized() else 0
        self.world = dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1
        self.optimizer = FlatAdamW(model.dit, lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, clip_norm=clip_norm)
        self.reducer = GradReducer(model.dit.store, ops=model.dit.engine.ops) if self.world > 1 else None
        self.ema = (FlatEMA(model.dit, ema_smoothing, ema_half_life, ema_update_interval, ema_start)
                    if (ema_smoothing is not None or ema_half_life is not None) else None)
        self.batch = 0
        if load_path:
            self.batch = load_checkpoint(load_path, model, self.optimizer, load_weights_only,
                                         load_strict_model_weights, load_ignore_keys, loader=self.loader, rank=self.rank,
                                         ema=self.ema)

    def lr_at(self, batch: int) -> float:
        return self.optimizer.lr * lr_multiplier(self.scheduler, batch, self.t_warmup, self.t_max, self.alpha, self.alpha_f)

    @torch.no_grad()
    def evaluate(self) -> float:
        """Composer's eval pass over `eval_dataloader` (trainer.eval_interval, dataset.eval in the configs): mean over
        batches and ranks of `model.eval_forward(batch)`'s loss -- DistLoss (utils.py:598-613: sum of batch losses and a
        batch count, both sum-reduced across ranks).  The model runs in eval mode (no patch masking, model.py:115-118).
        This trainer's rule: once the EMA has started, the pass runs on the EMA weights (`ema.applied()`); the training
        weights are restored bit for bit afterwards."""
        if self.ema is not None:
            with self.ema.applied():
                return self._evaluate()
        return self._evaluate()

    def _evaluate(self) -> float:
        import torch.distributed as dist
        dev = self.model.dit.store.device
        was_training = self.model.training
        self.model.eval()
        total = torch.zeros(2, dtype=torch.float64, device=dev)  # [sum of batch losses, batches]
        for batch in self.eval_loader:
            batch = {k: (v.to(dev, non_blocking=True) if torch.is_tensor(v) else v) for k, v in batch.items()}
            # eval runs unmasked (4x the backbone tokens of training): split like training does so that the
            # reference's eval_batch_size fits beside the weights; the batch loss is the sample-weighted mean
            n = batch["image_latents"].shape[0]
            acc = torch.zeros((), dtype=torch.float64, device=dev)
            for s0 in range(0, n, self.microbatch):
                mb = {k: (v[s0:s0 + self.microbatch] if torch.is_tensor(v) else v) for k, v in batch.items()}
                nb = mb["image_latents"].shape[0]
                acc += self.model.eval_forward(mb)[0].detach().double() * (nb / n)
            total[0] += acc
            total[1] += 1
        if self.world > 1:
            dist.all_reduce(total)
        self.model.train(was_training)
        if float(total[1]) == 0:
            raise RuntimeError("eval_dataloader yielded no batches")
        self.last_eval_loss = float(total[0] / total[1])
        return self.last_eval_loss

    def _raise_if_nonfinite(self, loss: Optional[float] = None) -> None:
        """NaNCatcher.after_loss (callbacks.py:47-64) without a per-step host sync: md_adamw refuses to apply a step
        whose gradient norm is not finite and raises a device flag; the flag (and the loss, when it is read anyway) is
        checked at log and checkpoint time, so a poisoned update is never applied and never saved."""
        if (loss is not None and loss != loss) or int(self.optimizer.nonfinite.item()) != 0:
            raise RuntimeError("Train loss contains a NaN.")  # callbacks.py:52

    def fit(self, until: Optional[int] = None) -> float:
        """Train to `max_duration` (or stop early after batch `until`, schedule unchanged); returns the last logged loss."""
        stop = self.t_max if until is None else min(self.t_max, int(until))
        dev = self.model.dit.store.device
        self.model.train()
        last = float("nan")
        t0, n0 = time.perf_counter(), 0
        while self.batch < stop:
            progressed = False
            for batch in self.loader:
                progressed = True
                batch = {k: (v.to(dev, non_blocking=True) if torch.is_tensor(v) else v) for k, v in batch.items()}
                self.optimizer.lr_now = self.lr_at(self.batch)
                loss = train_step(self.model, batch, self.optimizer, self.reducer, self.microbatch,
                                  lr=self.optimizer.lr_now, ema=self.ema)
                self.batch += 1
                n0 += batch["image_latents"].shape[0] * self.world
                if self.batch % self.log_every == 0 or self.batch == stop:
                    last = float(loss)  # the only host sync of the loop
                    self._raise_if_nonfinite(last)
                    dt = time.perf_counter() - t0
                    if self.rank == 0:
                        self.log(f"batch {self.batch}/{self.t_max} loss {last:.4f} lr {self.optimizer.lr_now:.3e} "
                                 f"{n0 / dt:.0f} img/s")
                    t0, n0 = time.perf_counter(), 0
                if self.eval_loader is not None and self.eval_interval > 0 and self.batch % self.eval_interval == 0:
                    ev = self.evaluate()
                    if self.rank == 0:
                        self.log(f"batch {self.batch}/{self.t_max} eval loss {ev:.4f}")
                if self.save_folder and self.batch % self.save_interval == 0:
                    self._raise_if_nonfinite()  # never write a checkpoint after a skipped (NaN / Inf) step
                    save_checkpoint(os.path.join(self.save_folder, f"ba{self.batch}.pt"), self.model, self.optimizer,
                                    self.batch, self.rank, loader=self.loader, world=self.world, keep=self.save_keep,
                                    ema=self.ema)
                if self.batch >= stop:
                    break
            if not progressed:
                raise RuntimeError("train_dataloader yielded no batches")
        return last
