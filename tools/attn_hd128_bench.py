"""Attention at head_dim 128 on one GPU: every hd-128 kernel at the shapes a hd-128 model runs, next to hd 64 at the same
H * hd, and a full training step of MicroDiT_XL_2 widths at head_dim 128 against 64.

    python tools/attn_hd128_bench.py [--iters 20] [--warmup 3] [--step-iters 5] [--rounds 2] [--no-step] [--out DIR]

Kernels: MicroDiT_XL_2 built with head_dim=128 (backbone 1024 with 4 / 6 / 8 heads per block, mixer 768 = 6 heads,
cross-attention to 77 caption tokens) at
  C2  res 256 (1024 tokens of 2x2 patches of 32x32 latents -> 256 tokens), mask 0.75 (64 backbone tokens), microbatch 256
  C4  res 512 (1024 tokens), mask 0.75 (256 backbone tokens), microbatch 32
plus the T5 caption length (120 keys) and a ragged shape.  Per shape, CUDA-event µs per launch (mean over `iters` after
`warmup`): md_attn_fwd_tc (the chunked wgmma forward) and md_attn_fwd_mma at hd 128 -- the two candidates md_attn_fwd
chooses between --, what md_attn_fwd picks, the hd-128 backward (md_attn_bwd), and hd 64 with twice the heads through
md_attn_fwd / md_attn_bwd.
Step: the fused EDM loss step (forward + backward) of MicroDiT_XL_2 widths at C2, microbatch 256, head_dim 64 and 128,
every leg in its own process, alternating for `rounds` rounds.
Prints one JSON line, with the GPU name and power limit read in the same run.
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

# (label, B, H at hd 128, Tq, Tk)
SHAPES = [
    ("C2 mixer self", 256, 6, 256, 256), ("C2 mixer cross", 256, 6, 256, 77),
    ("C2 backbone self", 256, 4, 64, 64), ("C2 backbone self", 256, 8, 64, 64), ("C2 backbone cross", 256, 8, 64, 77),
    ("C4 mixer self", 32, 6, 1024, 1024), ("C4 mixer cross", 32, 6, 1024, 77),
    ("C4 backbone self", 32, 4, 256, 256), ("C4 backbone self", 32, 8, 256, 256), ("C4 backbone cross", 32, 8, 256, 77),
    ("T5 captions", 256, 8, 64, 120), ("T5 captions", 32, 8, 256, 120), ("ragged", 64, 8, 130, 200),
]


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = (s.strip() for s in q.split(","))
    except Exception:
        name, power = torch.cuda.get_device_name(0), "unknown"
    return name, power


def time_us(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return round(e0.elapsed_time(e1) * 1e3 / iters, 1)


def kernels(iters, warmup):
    from micro_diffusion_b200.ops import CudaOps
    dev = torch.device("cuda:0")
    ops = CudaOps(dev)
    rows = []
    for label, B, H, Tq, Tk in SHAPES:
        row = {"shape": label, "B": B, "H128": H, "Tq": Tq, "Tk": Tk}
        for hd, Hh in ((128, H), (64, 2 * H)):
            hsz = Hh * hd
            g = torch.Generator(device=dev).manual_seed(0)
            q = torch.randn(B * Tq, hsz, device=dev, generator=g).to(torch.bfloat16)
            kv = torch.randn(B * Tk, 2 * hsz, device=dev, generator=g).to(torch.bfloat16)
            do = torch.randn(B * Tq, hsz, device=dev, generator=g).to(torch.bfloat16)
            o = torch.empty(B * Tq, hsz, device=dev, dtype=torch.bfloat16)
            lse = torch.empty(B, Hh, Tq, device=dev)
            delta = torch.empty(B, Hh, Tq, device=dev)
            dq, dkv = torch.empty_like(q), torch.empty_like(kv)
            k, v, dk, dv = kv[:, :hsz], kv[:, hsz:], dkv[:, :hsz], dkv[:, hsz:]

            def fwd(name):
                return lambda: ops._call(name, q.data_ptr(), hsz, k.data_ptr(), 2 * hsz, v.data_ptr(), 2 * hsz,
                                         o.data_ptr(), hsz, lse.data_ptr(), B, Hh, Tq, Tk, hd)

            def bwd(name):
                return lambda: ops._call(name, do.data_ptr(), hsz, q.data_ptr(), hsz, k.data_ptr(), 2 * hsz,
                                         v.data_ptr(), 2 * hsz, o.data_ptr(), hsz, lse.data_ptr(), delta.data_ptr(),
                                         dq.data_ptr(), hsz, dk.data_ptr(), 2 * hsz, dv.data_ptr(), 2 * hsz, B, Hh, Tq,
                                         Tk, hd)
            if hd == 128:
                row["fwd_tc_us"] = time_us(fwd("md_attn_fwd_tc"), iters, warmup)
                row["fwd_mma_us"] = time_us(fwd("md_attn_fwd_mma"), iters, warmup)
                row["fwd_us"] = time_us(fwd("md_attn_fwd"), iters, warmup)
                row["fwd_tflops"] = round(4 * B * Hh * Tq * Tk * hd / min(row["fwd_tc_us"], row["fwd_mma_us"]) / 1e6, 1)
                row["bwd_us"] = time_us(bwd("md_attn_bwd"), iters, warmup)
                row["bwd_tflops"] = round(10 * B * Hh * Tq * Tk * hd / row["bwd_us"] / 1e6, 1)
            else:
                row["hd64_fwd_us"] = time_us(fwd("md_attn_fwd"), iters, warmup)
                row["hd64_bwd_us"] = time_us(bwd("md_attn_bwd"), iters, warmup)
            del q, kv, do, o, lse, delta, dq, dkv
        row["faster_fwd"] = "wgmma" if row["fwd_tc_us"] < row["fwd_mma_us"] else "mma.sync"
        rows.append(row)
        print(row, file=sys.stderr)
    return rows


def step_leg(hd, B, iters, warmup):
    from micro_diffusion_b200.arch import micro_dit_xl_2_kwargs
    from micro_diffusion_b200.models.dit import DiT
    from micro_diffusion_b200.models.model import LatentDiffusion, PrecomputedLatentStubs
    dev, mask_ratio = "cuda:0", 0.75
    net = DiT(**{**micro_dit_xl_2_kwargs(input_size=32, in_channels=4), "head_dim": hd})
    ld = LatentDiffusion(net.to(dev), *PrecomputedLatentStubs.make(), train_mask_ratio=mask_ratio, latent_res=32)
    ld.train()
    g = torch.Generator(device=dev).manual_seed(0)
    x = 0.8 * torch.randn(B, 4, 32, 32, device=dev, generator=g)
    y = torch.randn(B, 1, 77, 1024, device=dev, generator=g).half()
    rnd = torch.randn(B, device=dev, generator=g)
    eps = torch.randn(B, 4, 32, 32, device=dev, generator=g)
    noise = torch.rand(B, 256, device=dev, generator=g)
    ms = time_us(lambda: ld.edm_loss_with_draws(x, y, None, rnd, eps, noise, mask_ratio).backward(), iters, warmup) / 1e3
    return {"head_dim": hd, "ms": round(ms, 2), "img_per_s": round(B / ms * 1e3, 1),
            "peak_gib": round(torch.cuda.max_memory_allocated() / 2 ** 30, 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--step-iters", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--no-step", action="store_true")
    ap.add_argument("--leg", type=int, default=None, help=argparse.SUPPRESS)
    ap.add_argument("--out", default=None, help="also write the JSON line to DIR/attn_hd128_bench.json")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "attn_hd128_bench times the H100 path: it needs a GPU"
    if a.leg:
        print(json.dumps(step_leg(a.leg, a.batch, a.step_iters, a.warmup)))
        return
    res = {"kernels": kernels(a.iters, a.warmup)}
    if not a.no_step:
        legs = []
        for _ in range(a.rounds):
            for hd in (64, 128):
                r = subprocess.run([sys.executable, os.path.abspath(__file__), "--leg", str(hd), "--batch", str(a.batch),
                                    "--step-iters", str(a.step_iters), "--warmup", str(a.warmup)],
                                   capture_output=True, text=True)
                if r.returncode != 0:
                    raise RuntimeError(f"head_dim {hd} leg failed:\n{r.stdout}\n{r.stderr}")
                legs.append(json.loads(r.stdout.strip().splitlines()[-1]))
                print(legs[-1], file=sys.stderr)
        res["step"] = {"model": "MicroDiT_XL_2 widths", "shape": "C2 res256 mask0.75", "microbatch": a.batch,
                       "legs": legs, "median_ms": {hd: statistics.median(l["ms"] for l in legs if l["head_dim"] == hd)
                                                   for hd in (64, 128)}}
    res["gpu"], res["power_limit"] = gpu_info()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "attn_hd128_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
