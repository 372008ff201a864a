"""Time the differentiable DiT.forward against the fused training step on one GPU.

    python tools/dit_vjp_bench.py [--batch 256] [--iters 10] [--warmup 3] [--out DIR]

MicroDiT_XL_2 at the C2 shape (res 256 -> 32x32x4 latents, mask 0.75), one microbatch, seeded inputs.  Three legs, each
timed with CUDA events around `iters` calls after `warmup` untimed ones:
  fused_loss_step  LatentDiffusion.edm_loss_with_draws(...).backward()  (forward + hand-derived backward, EDM loss)
  dit_vjp          F = DiT.forward(x, t, y, mask_ratio=0.75); F.backward(dF) with x, t, y and every parameter requiring
                   grad (forward + backward_output + the three input-gradient exits)
  dit_vjp_frozen   the same with every parameter frozen (input gradients only: no weight-gradient GEMMs)
Prints one JSON line with ms / step, img/s, peak memory, the GPU name and its power limit.
"""
from __future__ import annotations

import argparse
import json
import os
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


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters, torch.cuda.max_memory_allocated() / 2 ** 30


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON line to DIR/dit_vjp_bench.json")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "dit_vjp_bench times the H100 path: it needs a GPU"
    from micro_diffusion_b200.models.dit import MicroDiT_XL_2
    from micro_diffusion_b200.models.model import LatentDiffusion, PrecomputedLatentStubs
    from oracle import weights
    dev, B, mask_ratio = "cuda:0", a.batch, 0.75
    net = MicroDiT_XL_2(input_size=32, in_channels=4)
    net.load_state_dict(weights.synth_state_dict(net.state_dict(), seed=7))
    ld = LatentDiffusion(net.to(dev), *PrecomputedLatentStubs.make(), train_mask_ratio=mask_ratio, latent_res=32)
    ld.train()
    dit = ld.dit
    g = torch.Generator(device=dev).manual_seed(0)
    x = 0.8 * torch.randn(B, 4, 32, 32, device=dev, generator=g)
    y = torch.randn(B, 1, 77, 1024, device=dev, generator=g).half()
    rnd = torch.randn(B, device=dev, generator=g)
    eps = torch.randn(B, 4, 32, 32, device=dev, generator=g)
    noise = torch.rand(B, 256, device=dev, generator=g)
    t = 0.3 * torch.randn(B, device=dev, generator=g)
    dF = torch.randn(B, 4, 32, 32, device=dev, generator=g)
    yf = y.float()

    def loss_step():
        ld.edm_loss_with_draws(x, y, None, rnd, eps, noise, mask_ratio).backward()

    def vjp():
        xr, tr, yr = (v.detach().requires_grad_(True) for v in (x, t, yf))
        dit(xr, tr, yr, mask_ratio=mask_ratio)["sample"].backward(dF)

    res = {"model": "MicroDiT_XL_2", "shape": "C2 res256 mask0.75", "microbatch": B, "iters": a.iters}
    for leg, fn, frozen in (("fused_loss_step", loss_step, False), ("dit_vjp", vjp, False), ("dit_vjp_frozen", vjp, True)):
        dit.requires_grad_(not frozen)
        dit.zero_grad(set_to_none=True)
        ops = dit.engine.ops
        f0 = ops.gemm_flops
        ms, peak = timed(fn, a.iters, a.warmup)
        res[leg] = {"ms": round(ms, 3), "img_per_s": round(B / ms * 1e3, 1), "peak_gib": round(peak, 2),
                    "gemm_tflop_per_step": round((ops.gemm_flops - f0) / (a.iters + a.warmup) / 1e12, 3)}
    res["gpu"], res["power_limit"] = gpu_info()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "dit_vjp_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
