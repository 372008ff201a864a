"""Cost of the weight EMA on the training step, on one GPU.

    python tools/ema_bench.py [--batch 256] [--iters 10] [--warmup 3] [--rounds 3] [--out DIR]

MicroDiT_XL_2 at the C2 shape (res 256 -> 32x32x4 latents, mask 0.75), one train_step (microbatched forward +
backward, clip + AdamW) per iteration, with
  off  FlatAdamW alone (md_sumsq + md_adamw)
  on   the same with a FlatEMA updated every batch (md_adamw_ema in place of md_adamw; started before the timed steps)
Every leg runs in its own process; the legs alternate off, on, off, on, ... for `rounds` rounds, each timed with CUDA
events around `iters` steps after `warmup` untimed ones.  Per leg: ms / step, img/s, peak memory, and the time of the
optimizer step alone (events around `iters` further FlatAdamW.step calls); the `on` leg also times `iters`
`ema.applied()` enter + exit pairs.  Prints one JSON line with every leg, the medians, and the GPU name and power limit
read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = (s.strip() for s in q.split(","))
    except Exception:
        name, power = torch.cuda.get_device_name(0), "unknown"
    return name, power


def _timed(fn, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def leg(mode, B, iters, warmup):
    from micro_diffusion_b200.ema import FlatEMA
    from micro_diffusion_b200.models.dit import MicroDiT_XL_2
    from micro_diffusion_b200.models.model import LatentDiffusion, PrecomputedLatentStubs
    from micro_diffusion_b200.train_step import FlatAdamW, train_step
    dev = "cuda:0"
    ld = LatentDiffusion(MicroDiT_XL_2(input_size=32, in_channels=4).to(dev), *PrecomputedLatentStubs.make(),
                         train_mask_ratio=0.75, latent_res=32)
    ld.train()
    from oracle import weights
    batch = {k: v.to(dev) for k, v in weights.synth_batch(B, 4, 32, seed=0).items()}
    opt = FlatAdamW(ld.dit, lr=1e-4)
    ema = FlatEMA(ld.dit, smoothing=0.9999, ema_start="0ba") if mode == "on" else None

    def step():
        train_step(ld, batch, opt, None, B, ema=ema)

    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    ms = _timed(step, iters)
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    opt_ms = _timed(lambda: opt.step(None, None, ema), iters)
    res = {"mode": mode, "ms": round(ms, 3), "img_per_s": round(B / ms * 1e3, 1), "peak_gib": round(peak, 2),
           "optimizer_step_ms": round(opt_ms, 3), "params": ld.dit.store.flat.numel()}
    if ema is not None:
        assert ema.started and ema.due(opt.t + 1)

        def enter_exit():
            with ema.applied():
                pass
        enter_exit()
        res["applied_enter_exit_ms"] = round(_timed(enter_exit, iters), 3)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--leg", choices=("off", "on"), default=None, help=argparse.SUPPRESS)
    ap.add_argument("--out", default=None, help="also write the JSON line to DIR/ema_bench.json")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "ema_bench times the H100 path: it needs a GPU"
    if a.leg:
        print(json.dumps(leg(a.leg, a.batch, a.iters, a.warmup)))
        return
    legs = []
    for _ in range(a.rounds):
        for mode in ("off", "on"):
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--leg", mode, "--batch", str(a.batch),
                                "--iters", str(a.iters), "--warmup", str(a.warmup)], capture_output=True, text=True)
            if r.returncode != 0:
                raise RuntimeError(f"{mode} leg failed:\n{r.stdout}\n{r.stderr}")
            legs.append(json.loads(r.stdout.strip().splitlines()[-1]))
            print(legs[-1], file=sys.stderr)

    def med(key, mode):
        return statistics.median(l[key] for l in legs if l["mode"] == mode)
    res = {"model": "MicroDiT_XL_2", "shape": "C2 res256 mask0.75", "microbatch": a.batch, "iters": a.iters,
           "legs": legs, "median_ms": {m: med("ms", m) for m in ("off", "on")},
           "median_optimizer_step_ms": {m: med("optimizer_step_ms", m) for m in ("off", "on")},
           "median_applied_enter_exit_ms": med("applied_enter_exit_ms", "on"),
           "peak_gib": {m: max(l["peak_gib"] for l in legs if l["mode"] == m) for m in ("off", "on")}}
    res["ema_overhead_pct"] = round(100 * (res["median_ms"]["on"] / res["median_ms"]["off"] - 1), 2)
    res["gpu"], res["power_limit"] = gpu_info()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "ema_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
