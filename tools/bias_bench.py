"""Cost of use_bias=True on the training step, on one GPU.

    python tools/bias_bench.py [--batch 256] [--iters 10] [--warmup 3] [--rounds 3] [--out DIR]

The fused EDM loss step (forward + hand-derived backward) at the C2 shape (res 256 -> 32x32x4 latents, mask 0.75) for
  zoo   MicroDiT_XL_2 (use_bias=False)
  bias  the same architecture built as DiT(**micro_dit_xl_2_kwargs(), use_bias=True)
Both do not fit on one 80 GB device next to each other at microbatch 256, so every leg runs in its own process; the legs
alternate zoo, bias, zoo, bias, ... for `rounds` rounds, each timed with CUDA events around `iters` steps after `warmup`
untimed ones.  Per leg: ms / step, img/s, peak memory, kernel launches per step and the bytes the bias-gradient column
sums read per step (counted over one extra, untimed step).  Prints one JSON line with every leg, the per-arch medians,
the overhead of `bias` over `zoo`, and the GPU name and power limit read in the same run.
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


def leg(arch, B, iters, warmup):
    from micro_diffusion_b200.arch import micro_dit_xl_2_kwargs
    from micro_diffusion_b200.models.dit import DiT
    from micro_diffusion_b200.models.model import LatentDiffusion, PrecomputedLatentStubs
    dev, mask_ratio = "cuda:0", 0.75
    net = DiT(**{**micro_dit_xl_2_kwargs(input_size=32, in_channels=4), "use_bias": arch == "bias"})
    ld = LatentDiffusion(net.to(dev), *PrecomputedLatentStubs.make(), train_mask_ratio=mask_ratio, latent_res=32)
    ld.train()
    g = torch.Generator(device=dev).manual_seed(0)
    x = 0.8 * torch.randn(B, 4, 32, 32, device=dev, generator=g)
    y = torch.randn(B, 1, 77, 1024, device=dev, generator=g).half()
    rnd = torch.randn(B, device=dev, generator=g)
    eps = torch.randn(B, 4, 32, 32, device=dev, generator=g)
    noise = torch.rand(B, 256, device=dev, generator=g)

    def step():
        ld.edm_loss_with_draws(x, y, None, rnd, eps, noise, mask_ratio).backward()

    ops = ld.dit.engine.ops
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    n0 = ops.launches
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        step()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / iters
    launches = (ops.launches - n0) / iters
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    # bytes read by the bias-gradient column sums of one step (the adaLN / stem / patch-embed / final-layer biases exist in
    # both models; only the block, prompt-block and mixer-map biases are new)
    read = {"colsum": 0, "colsum_interleaved": 0}
    for nm in read:
        orig = getattr(ops, nm)

        def counted(x, *a, _nm=nm, _orig=orig, **k):
            read[_nm] += x.numel() * x.element_size()
            return _orig(x, *a, **k)
        setattr(ops, nm, counted)
    step()
    torch.cuda.synchronize()
    return {"arch": arch, "ms": round(ms, 3), "img_per_s": round(B / ms * 1e3, 1), "peak_gib": round(peak, 2),
            "launches_per_step": launches, "colsum_read_mb": round(sum(read.values()) / 2 ** 20, 1),
            "colsum_interleaved_read_mb": round(read["colsum_interleaved"] / 2 ** 20, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--leg", choices=("zoo", "bias"), default=None, help=argparse.SUPPRESS)
    ap.add_argument("--out", default=None, help="also write the JSON line to DIR/bias_bench.json")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bias_bench times the H100 path: it needs a GPU"
    if a.leg:
        print(json.dumps(leg(a.leg, a.batch, a.iters, a.warmup)))
        return
    legs = []
    for _ in range(a.rounds):
        for arch in ("zoo", "bias"):
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--leg", arch, "--batch", str(a.batch),
                                "--iters", str(a.iters), "--warmup", str(a.warmup)], capture_output=True, text=True)
            if r.returncode != 0:
                raise RuntimeError(f"{arch} leg failed:\n{r.stdout}\n{r.stderr}")
            legs.append(json.loads(r.stdout.strip().splitlines()[-1]))
            print(legs[-1], file=sys.stderr)
    med = {arch: statistics.median(l["ms"] for l in legs if l["arch"] == arch) for arch in ("zoo", "bias")}
    res = {"model": "MicroDiT_XL_2 vs the same with use_bias=True", "shape": "C2 res256 mask0.75", "microbatch": a.batch,
           "iters": a.iters, "legs": legs, "median_ms": med,
           "median_img_per_s": {k: round(a.batch / v * 1e3, 1) for k, v in med.items()},
           "bias_overhead_pct": round(100 * (med["bias"] / med["zoo"] - 1), 2)}
    res["gpu"], res["power_limit"] = gpu_info()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bias_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
