"""Eager Heun loop vs the CUDA-graph sampler (engine.SamplerGraph) on MicroDiT_XL_2, at the settings people sample with:
the README's (latent 64, 4 prompts, guidance 5, 30 steps), the image_monitor callback's (16 prompts, guidance 5, 30 steps,
latent 32 and 64) and one prompt at guidance 5.  Synthetic weights and precomputed caption tensors (the sampler's cost
does not depend on the weights, and the text encoder is frozen and outside the timed loop).

Per setting and path: ms per sampler run (host clock around runs that end in a device synchronise, median of --runs),
library launches per run (ctypes calls into libmicrodit_b200.so), CUDA-graph replays per run and peak device memory;
for the graph path also the GPU time of one replay of the full-step graph (CUDA events over --replays back-to-back
replays: two denoiser calls and the four stage launches), halved as the GPU time per denoiser call.  The two paths are
checked bit-identical on the timed inputs.  Prints one JSON line per setting and writes them to --out.

  python tools/sampler_bench.py [--runs 5] [--replays 20] [--only readme,monitor32,monitor64,single] [--out FILE]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

SETTINGS = {  # name: (latent, pos_interp_scale, prompts, guidance, steps)
    "readme": (64, 2.0, 4, 5.0, 30),
    "monitor32": (32, 1.0, 16, 5.0, 30),
    "monitor64": (64, 2.0, 16, 5.0, 30),
    "single": (64, 2.0, 1, 5.0, 30),
}


def gpu_info():
    try:
        q = "name,power.limit,clocks.sm,clocks.max.sm"
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return dict(zip(q.split(","), [s.strip() for s in out[0].split(",")])) if out else {}
    except Exception as e:  # the numbers are still reported, without the card's settings
        return {"error": str(e)}


def build(latent, scale):
    from micro_diffusion_b200.models.dit import MicroDiT_XL_2
    from micro_diffusion_b200.models.model import LatentDiffusion, PrecomputedLatentStubs
    from oracle import weights
    net = MicroDiT_XL_2(input_size=latent, in_channels=4, pos_interp_scale=scale)
    net.load_state_dict(weights.synth_state_dict(net.state_dict(), seed=7))
    vae, te, tok = PrecomputedLatentStubs.make()
    ld = LatentDiffusion(net.to("cuda"), vae, te, tok, latent_res=latent)
    ld.eval()
    return ld


def time_path(ld, x, y, steps, cfg, graph, runs):
    ld.sampler_graph = graph
    ops = ld.dit.engine.ops
    torch.manual_seed(0)
    out = ld.edm_sampler_loop(x, y, steps=steps, cfg=cfg)  # warm-up (and, on the graph path, the capture)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    times, launches = [], []
    for _ in range(runs):
        torch.manual_seed(0)
        l0 = ops.launches
        t0 = time.perf_counter()
        out = ld.edm_sampler_loop(x, y, steps=steps, cfg=cfg)
        torch.cuda.synchronize()
        times.append((time.perf_counter() - t0) * 1e3)
        launches.append(ops.launches - l0)
    return out, statistics.median(times), min(times), launches[-1], torch.cuda.max_memory_allocated()


def replay_ms(ld, B, cfg, shape, cap_shape, replays):
    sg = ld.dit.engine.sampler(B, cfg != 1.0, shape, cap_shape)
    g = sg.graphs["step"]
    sg.step.zero_()  # keep the index inside the table: every replay runs step 0 again
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    g.replay()
    sg.step.zero_()
    e0.record()
    for _ in range(replays):
        g.replay()
        sg.step.zero_()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / replays


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--replays", type=int, default=20)
    ap.add_argument("--only", default=",".join(SETTINGS))
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "sampler_bench measures on the GPU: no CUDA device found"
    info = gpu_info()
    lines = []
    models = {}
    for name in a.only.split(","):
        latent, scale, B, cfg, steps = SETTINGS[name]
        if (latent, scale) not in models:
            models.clear()
            torch.cuda.empty_cache()
            models[(latent, scale)] = build(latent, scale)
        ld = models[(latent, scale)]
        g = torch.Generator(device="cuda").manual_seed(1)
        x = torch.randn(B, 4, latent, latent, device="cuda", generator=g)
        y = torch.randn(B, 1, 77, 1024, device="cuda", generator=g).half()
        res = {}
        for graph in (False, True, False, True):  # alternating, so drift of the shared machine hits both paths
            out, med, best, launches, peak = time_path(ld, x, y, steps, cfg, graph, a.runs)
            r = res.setdefault(graph, {"out": out, "ms": [], "launches": launches, "peak_gib": 0.0})
            r["ms"].append(med)
            r["peak_gib"] = max(r["peak_gib"], peak / 2 ** 30)
        same = bool(torch.equal(res[True]["out"], res[False]["out"]))
        step_ms = replay_ms(ld, B, cfg, (4, latent, latent), (1, 77, 1024), a.replays)
        calls = 2 * steps - 1
        line = {"setting": name, "latent": latent, "prompts": B, "guidance": cfg, "steps": steps, "gpu": info,
                "eager_ms_per_run": [round(v, 1) for v in res[False]["ms"]],
                "graph_ms_per_run": [round(v, 1) for v in res[True]["ms"]],
                "speedup": round(min(res[False]["ms"]) / min(res[True]["ms"]), 3),
                "graph_gpu_ms_per_denoiser_call": round(step_ms / 2, 3),
                "eager_wall_ms_per_denoiser_call": round(min(res[False]["ms"]) / calls, 3),
                "eager_library_launches_per_run": res[False]["launches"],
                "graph_library_launches_per_run": res[True]["launches"], "graph_replays_per_run": steps + 1,
                "eager_peak_gib": round(res[False]["peak_gib"], 2), "graph_peak_gib": round(res[True]["peak_gib"], 2),
                "bit_identical": same}
        print(json.dumps(line), flush=True)
        lines.append(line)
        ld.dit.engine.release_sampler_graphs()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write("\n".join(json.dumps(v) for v in lines) + "\n")


if __name__ == "__main__":
    main()
