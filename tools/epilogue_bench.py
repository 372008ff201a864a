"""Cost of the GEMM epilogue tails that read global memory, at the C2 launch shapes, on one GPU.

    python tools/epilogue_bench.py [--batch 256] [--iters 30] [--warmup 5] [--rounds 3] [--out DIR]

C2 is MicroDiT_XL_2 at res 256 (32 x 32 latents, 256 tokens; mask 0.75 leaves 64 in the backbone), 8 microbatches of
256 per step.  The shapes come from `arch.py`: every SwiGLU block runs MD_EPI_SWIGLU forward and MD_EPI_SWIGLU_GRAD in
the w3 dgrad, every expert block MD_EPI_ACT_DUAL forward and MD_EPI_ACT_GRAD in the dgrad of its second expert GEMM,
and the prompt block's SwiGLU runs over the 77 caption tokens.  Each distinct shape is timed with its real epilogue and
again with the plain bf16 store (MD_EPI_STORE_BF16) at the same M, N, K and batch; the difference is its "tail tax".
Timing: CUDA events around `iters` back-to-back launches after `warmup` untimed ones, the two variants alternating for
`rounds` rounds, median per variant.  Prints a table and one JSON line with the per-shape times, TFLOP/s and tail tax,
the tail tax summed over one C2 step (launches per microbatch x 8), and the GPU name and power limit read in the same
run.  The backward tails (SWIGLU_GRAD, ACT_GRAD) are summed separately from the forward ones, which are for information.
"""
from __future__ import annotations

import argparse
import collections
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from micro_diffusion_b200.arch import DiTConfig, micro_dit_xl_2_kwargs  # noqa: E402
from micro_diffusion_b200.ops import (EPI_ACT_DUAL, EPI_ACT_GRAD, EPI_BF16, EPI_SWIGLU,  # noqa: E402
                                      EPI_SWIGLU_GRAD, CudaOps)

NAMES = {EPI_SWIGLU: "SWIGLU", EPI_SWIGLU_GRAD: "SWIGLU_GRAD", EPI_ACT_DUAL: "ACT_DUAL", EPI_ACT_GRAD: "ACT_GRAD"}
MICROBATCHES = 8   # C2: global batch 2048 at microbatch 256
CAPTION_TOKENS = 77
TOKENS, MASK_RATIO = 256, 0.75


def c2_shapes(B):
    """{(epi, batch, M, N, K): launches per microbatch} of the reading tails and their forward partners."""
    cfg = DiTConfig(**micro_dit_xl_2_kwargs(input_size=32, in_channels=4))
    kept = int(TOKENS * (1 - MASK_RATIO))
    count = collections.Counter()
    for blocks, T in ((cfg.mixer_blocks, TOKENS), (cfg.blocks, kept)):
        for b in blocks:
            D, f = b.dim, b.ffn_dim
            if b.moe:
                E = cfg.num_experts
                rows = B * int(cfg.expert_capacity * T / E)
                count[(EPI_ACT_DUAL, E, rows, f, D)] += 1
                count[(EPI_ACT_GRAD, E, rows, f, D)] += 1
            else:
                count[(EPI_SWIGLU, 1, B * T, 2 * f, D)] += 1
                count[(EPI_SWIGLU_GRAD, 1, B * T, f, D)] += 1
    f = cfg.prompt_ffn_dim
    count[(EPI_SWIGLU, 1, B * CAPTION_TOKENS, 2 * f, cfg.dim)] += 1
    count[(EPI_SWIGLU_GRAD, 1, B * CAPTION_TOKENS, f, cfg.dim)] += 1
    return count


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = (s.strip() for s in q.split(","))
    except Exception:
        name, power = torch.cuda.get_device_name(0), "unknown"
    return name, power


def time_launches(fn, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / iters  # us per launch


def measure(ops, epi, batch, M, N, K, iters, warmup, rounds):
    dev = ops.device
    g = torch.Generator(device=dev).manual_seed(0)
    bshape = (lambda *s: (batch, *s)) if batch > 1 else (lambda *s: s)
    A = (torch.randn(bshape(M, K), device=dev, generator=g) * K ** -0.5).bfloat16()
    W = (torch.randn(bshape(N, K), device=dev, generator=g) * K ** -0.5).bfloat16()
    plain = torch.empty(bshape(M, N), device=dev, dtype=torch.bfloat16)
    if epi == EPI_SWIGLU:
        C, C2 = torch.empty(bshape(M, N), device=dev, dtype=torch.bfloat16), torch.empty(bshape(M, N // 2), device=dev, dtype=torch.bfloat16)
        real = lambda: ops.gemm(A, W, C, epi=EPI_SWIGLU, C2=C2)  # noqa: E731
    elif epi == EPI_SWIGLU_GRAD:
        C = torch.empty(bshape(M, 2 * N), device=dev, dtype=torch.bfloat16)
        aux = torch.randn(bshape(M, 2 * N), device=dev, generator=g).bfloat16()
        real = lambda: ops.gemm(A, W, C, epi=EPI_SWIGLU_GRAD, aux=aux)  # noqa: E731
    elif epi == EPI_ACT_DUAL:
        C, C2 = torch.empty_like(plain), torch.empty_like(plain)
        real = lambda: ops.gemm(A, W, C, epi=EPI_ACT_DUAL, C2=C2)  # noqa: E731
    else:
        C = torch.empty_like(plain)
        aux = torch.randn(bshape(M, N), device=dev, generator=g).bfloat16()
        real = lambda: ops.gemm(A, W, C, epi=EPI_ACT_GRAD, aux=aux)  # noqa: E731
    store = lambda: ops.gemm(A, W, plain, epi=EPI_BF16)  # noqa: E731
    for fn in (store, real):
        for _ in range(warmup):
            fn()
    torch.cuda.synchronize()
    t_store, t_real = [], []
    for _ in range(rounds):
        t_store.append(time_launches(store, iters))
        t_real.append(time_launches(real, iters))
    us_store, us_real = statistics.median(t_store), statistics.median(t_real)
    flop = 2.0 * batch * M * N * K
    return {"epilogue": NAMES[epi], "batch": batch, "M": M, "N": N, "K": K, "us": round(us_real, 1),
            "us_store_only": round(us_store, 1), "tflops": round(flop / us_real * 1e-6, 1),
            "tflops_store_only": round(flop / us_store * 1e-6, 1), "tail_tax_us": round(us_real - us_store, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256, help="microbatch")
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON line to DIR/epilogue_bench.json")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "epilogue_bench times the H100 kernels: it needs a GPU"
    assert a.iters >= 20, "at least 20 timed launches per shape"
    ops = CudaOps("cuda:0")
    shapes = c2_shapes(a.batch)
    rows = []
    for (epi, batch, M, N, K), n in sorted(shapes.items()):
        r = measure(ops, epi, batch, M, N, K, a.iters, a.warmup, a.rounds)
        r["launches_per_microbatch"] = n
        r["tail_tax_ms_per_step"] = round(r["tail_tax_us"] * n * MICROBATCHES * 1e-3, 2)
        rows.append(r)
        print(f"{r['epilogue']:>12} b={batch} M={M:6d} N={N:5d} K={K:5d} x{n:2d}: {r['us']:8.1f} us {r['tflops']:6.1f} TF/s | "
              f"store only {r['us_store_only']:8.1f} us {r['tflops_store_only']:6.1f} TF/s | tail tax {r['tail_tax_us']:7.1f} us, "
              f"{r['tail_tax_ms_per_step']:6.2f} ms/step", file=sys.stderr, flush=True)
    bwd = sum(r["tail_tax_ms_per_step"] for r in rows if r["epilogue"] in ("SWIGLU_GRAD", "ACT_GRAD"))
    fwd = sum(r["tail_tax_ms_per_step"] for r in rows if r["epilogue"] in ("SWIGLU", "ACT_DUAL"))
    res = {"model": "MicroDiT_XL_2", "shape": "C2 res256 mask0.75", "microbatch": a.batch, "microbatches_per_step": MICROBATCHES,
           "iters": a.iters, "rounds": a.rounds, "shapes": rows, "tail_tax_ms_per_step_backward": round(bwd, 1),
           "tail_tax_ms_per_step_forward": round(fwd, 1)}
    res["gpu"], res["power_limit"] = gpu_info()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "epilogue_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
