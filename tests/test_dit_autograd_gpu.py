"""Autograd through DiT.forward on the H100: the three adjoint kernels against their torch restatements, the CUDA VJP
against the fp32 oracle's autograd (bf16 bounds as tests/test_parity_gpu.py, 1e-3 in MD_PRECISION=high), the fused loss
against the same loss written over the differentiable model_forward_wrapper, bit-reproducibility in deterministic mode
and the release of the saved activations."""
import gc
import os

import pytest
import torch

from oracle import configs, port, weights
from tests import dit_vjp_common as vc
from tests import parity_common as pc

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
CASES = list(configs.PARITY_CONFIGS)
rel = pc.rel_l2


def _ops(prec):
    from micro_diffusion_b200.ops import CudaOps
    return CudaOps(DEV, precision="high" if prec else "bf16")


def _high_ops(device):
    from micro_diffusion_b200.ops import CudaOps
    return CudaOps(device, precision="high")


# ------------------------------------------------------------------------------------------------ 1. kernel contracts
@pytest.mark.parametrize("prec", [0, 1])
def test_adjoint_kernels_match_their_contracts(prec):
    ops = _ops(prec)
    emu = vc.VJPEmuOps(exact=True)
    g = torch.Generator().manual_seed(5)
    for C, p, H, masked in [(4, 2, 32, False), (4, 2, 32, True), (16, 2, 64, True), (4, 4, 32, False)]:
        B, T = 3, (H // p) ** 2
        Tk = T // 4 if masked else T
        keep = None
        if masked:
            keep = torch.empty(B * Tk, dtype=torch.int32)
            emu.mask_sort(torch.rand(B, T, generator=g), None, torch.empty(B, T, dtype=torch.int32), torch.empty(B, T), keep, Tk)
        dF = torch.randn(B, C, H, H, generator=g)
        out = ops.empty((B * Tk, p * p * C), torch.bfloat16)
        ops.unpatchify_bwd(dF.to(DEV), keep.to(DEV) if keep is not None else None, out, p, Tk)
        ref = torch.empty(B * Tk, p * p * C)
        emu.unpatchify_bwd(dF, keep, ref, p, Tk)
        assert torch.equal(out.cpu(), ref.to(out.dtype)), (C, p, masked)   # a permutation + one rounding
        scale = torch.rand(B, generator=g) + 0.5 if masked else None
        dp = torch.randn(B * T, C * p * p, generator=g)
        dx = torch.empty(B, C, H, H, device=DEV)
        ops.patchify_bwd(dp.to(DEV), scale.to(DEV) if scale is not None else None, dx, p)
        ref = torch.empty(B, C, H, H)
        emu.patchify_bwd(dp, scale, ref, p)
        assert torch.equal(dx.cpu(), ref), (C, p, masked)
    for dim in (256, 512):
        t = 2 * torch.randn(7, generator=g)
        cot = torch.randn(7, dim, generator=g)
        dt = torch.empty(7, device=DEV)
        ops.timestep_embed_bwd(cot.to(DEV), t.to(DEV), dt)
        td = t.double().requires_grad_(True)
        half = dim // 2
        a = td[:, None] * torch.exp(-torch.log(torch.tensor(10000.0, dtype=torch.float64)) * torch.arange(half) / half)
        (torch.cat([a.cos(), a.sin()], -1) * cot.double()).sum().backward()
        scale_ = float(cot.abs().sum(1).max())
        assert float((dt.cpu().double() - td.grad).abs().max()) < 1e-5 * scale_, dim


def test_adjoint_kernels_validate_their_arguments():
    from micro_diffusion_b200._lib import MicroditLibraryError
    ops = _ops(0)
    with pytest.raises(MicroditLibraryError, match="Tk"):
        ops._call("md_unpatchify_bwd", torch.zeros(1, device=DEV).data_ptr(), None, torch.zeros(1, device=DEV).data_ptr(),
                  1, 4, 8, 8, 2, 8)
    with pytest.raises(MicroditLibraryError, match="multiples of p"):
        ops._call("md_patchify_bwd", torch.zeros(1, device=DEV).data_ptr(), None, torch.zeros(1, device=DEV).data_ptr(),
                  1, 4, 9, 8, 2)
    with pytest.raises(MicroditLibraryError, match="null pointer"):
        ops._call("md_timestep_embed_bwd", None, None, None, 2, 256)


# ------------------------------------------------------------------------------------------------ 2. VJP parity
def _cuda_vs_port(name, mask_ratio, ops_factory=None):
    net = vc.build_dit(name, ops_factory=ops_factory, device=DEV)
    x, t, y, dF = vc.vjp_inputs(name, device=DEV)
    grid = configs.PARITY_CONFIGS[name]["ctor"]["input_size"] // configs.PARITY_CONFIGS[name]["ctor"]["patch_size"]
    noise = vc.mask_noise(x.shape[0], grid * grid, DEV).cpu() if mask_ratio > 0 else None
    F, dx, dt, dy, grads = vc.product_vjp(net, x, t, y, dF, mask_ratio)
    assert not net.engine.ops.is_emulation
    oF, odx, odt, ody, ograds = vc.port_vjp(name, x, t, y, dF, mask_ratio, noise)
    errs, med, worst = pc.grad_report(grads, ograds)
    ie = {"F": rel(F, oF), "dx": rel(dx, odx), "dt": rel(dt, odt), "dy": rel(dy, ody)}
    return ie, errs, med, worst


@pytest.mark.parametrize("name", CASES)
def test_cuda_vjp_matches_oracle(name):
    mask_ratio = max(vc.VJP_MASKS[name])
    amp = torch.load(os.path.join(pc.GOLDEN, f"vjp_{name}.pt"), weights_only=False)["cases"][mask_ratio]["ref_amp_bf16"]
    ie, errs, med, worst = _cuda_vs_port(name, mask_ratio)
    print(f"\n[{name} vjp mask {mask_ratio}] " + " ".join(f"{k} {v:.2e} (ref amp {amp[k]:.2e})" for k, v in ie.items())
          + f" | grads median {med:.2e} worst {worst:.2e} ({errs[0][1]}); ref amp {amp['grad_rel_median']:.2e} "
          f"{amp['grad_rel_max']:.2e}")
    for k, e in ie.items():
        assert e < 2 * amp[k] + 2e-2, (k, e)
    assert med < 1.5 * amp["grad_rel_median"] + 5e-3
    assert worst < 2 * amp["grad_rel_max"] + 2e-2, errs[:5]


@pytest.mark.parametrize("name", CASES)
def test_cuda_vjp_high_precision(name):
    ie, errs, med, worst = _cuda_vs_port(name, max(vc.VJP_MASKS[name]), ops_factory=_high_ops)
    print(f"\n[{name} vjp high] " + " ".join(f"{k} {v:.2e}" for k, v in ie.items()) +
          f" | grads median {med:.2e} worst {worst:.2e} ({errs[0][1]})")
    assert ie["dx"] < 1e-3 and ie["dt"] < 1e-3 and med < 1e-3, (ie, med)


def _zoo_vjp(arch, head_dim, input_size, in_channels, mask_ratio, scale=1.0, B=2, ops_factory=None):
    from micro_diffusion_b200.models import dit as zoo
    net = getattr(zoo, arch)(input_size=input_size, in_channels=in_channels, pos_interp_scale=scale,
                             ops_factory=ops_factory)
    net.load_state_dict(weights.synth_state_dict(net.state_dict(), seed=pc.WEIGHT_SEED))
    sd = {k: v.detach().clone() for k, v in net.state_dict().items()}
    net = net.to(DEV)
    g = torch.Generator().manual_seed(vc.VJP_SEED)
    x = torch.randn(B, in_channels, input_size, input_size, generator=g)
    t = 0.3 * torch.randn(B, generator=g)
    y = torch.randn(B, 1, 77, 1024, generator=g).half().float()
    dF = torch.randn(B, in_channels, input_size, input_size, generator=g)
    T = (input_size // 2) ** 2
    noise = vc.mask_noise(B, T, DEV).cpu() if mask_ratio > 0 else None
    F, dx, dt, dy, grads = vc.product_vjp(net, x.to(DEV), t.to(DEV), y.to(DEV), dF.to(DEV), mask_ratio)
    del net
    gc.collect()
    torch.cuda.empty_cache()
    P = {k: v.clone().requires_grad_(k not in ("pos_embed", "mask_token")) for k, v in sd.items()}
    cfg = port.PortConfig(patch_size=2, head_dim=head_dim, num_experts=8, expert_capacity=2.0)
    xo, to, yo = (v.clone().requires_grad_(True) for v in (x, t, y))
    oF = port.dit_forward(P, cfg, xo, to, yo, mask_ratio, noise)["sample"]
    (oF * dF).sum().backward()
    errs, med, worst = pc.grad_report(grads, {k: v.grad for k, v in P.items() if v.grad is not None})
    ie = {"F": rel(F, oF.detach()), "dx": rel(dx, xo.grad), "dt": rel(dt, to.grad), "dy": rel(dy, yo.grad)}
    return ie, errs, med, worst


@pytest.mark.parametrize("arch,head_dim,label,mask_ratio", [
    ("MicroDiT_Tiny_2", 32, "C2", 0.75), ("MicroDiT_Tiny_2", 32, "C3", 0.0),
    ("MicroDiT_XL_2", 64, "C2", 0.75), ("MicroDiT_XL_2", 64, "C3", 0.0),
])
def test_zoo_vjp_matches_oracle(arch, head_dim, label, mask_ratio):
    """The zoo models at the res-256 shapes of BASELINE.json (C2 mask 0.75, C3 mask 0), batch 2: CUDA VJP (bf16) vs the
    fp32 port's autograd.  The reference's own amp-bf16 VJP deviates by 1-4e-2 on the parity configs (tests/golden/
    vjp_*.pt): the bounds allow that class at 34 blocks.  The expert-choice router gates are bounded apart: a token near
    a top-k boundary changes expert under bf16, which moves that gate's gradient by O(1) relative and the norm3 gain
    feeding the same router by up to ~0.35 (MicroDiT_XL_2 at C2).  Correctness at the 1e-3 level is checked by the
    high-precision mode (test_tiny_zoo_vjp_high_precision, test_cuda_vjp_high_precision)."""
    ie, errs, med, worst = _zoo_vjp(arch, head_dim, 32, 4, mask_ratio)
    rest = [(e, k) for e, k in errs if not k.endswith("mlp.gate.weight")]
    gates = [(e, k) for e, k in errs if k.endswith("mlp.gate.weight")]
    print(f"\n[{arch} {label} vjp] " + " ".join(f"{k} {v:.2e}" for k, v in ie.items()) +
          f" | grads median {med:.2e} worst {rest[0][0]:.2e} ({rest[0][1]}), router gates worst {gates[0][0]:.2e}")
    assert max(ie.values()) < 6e-2, ie
    assert med < 6e-2 and rest[0][0] < 0.5 and gates[0][0] < 1.0, errs[:5]


def test_tiny_zoo_vjp_high_precision():
    ie, errs, med, worst = _zoo_vjp("MicroDiT_Tiny_2", 32, 32, 4, 0.75, ops_factory=_high_ops)
    print(f"\n[Tiny_2 vjp high] " + " ".join(f"{k} {v:.2e}" for k, v in ie.items()) +
          f" | grads median {med:.2e} worst {worst:.2e} ({errs[0][1]})")
    assert ie["dx"] < 1e-3 and ie["dt"] < 1e-3 and med < 1e-3, (ie, med)


# ------------------------------------------------------------------------------------------------ 3. self-consistency
def test_fused_loss_matches_the_loss_over_the_differentiable_wrapper():
    """MicroDiT_XL_2 at C2 (mask 0.75, batch 2): parameter gradients of the fused edm_loss_with_draws(...).backward()
    against the reference's loss formula (model.py:181-210) written in torch over model_forward_wrapper -> DiT.forward
    with the same draws.  Both run the same kernels in deterministic mode (no run-to-run atomics); they can differ only
    by fp32 reassociation in the loss gradient before its bf16 rounding, which the caption-stem cancellation of
    DESIGN.md 5.4 would amplify on a few parameters (measured on an H100: bit-identical)."""
    import torch.nn.functional as F
    from micro_diffusion_b200.models.dit import MicroDiT_XL_2
    from micro_diffusion_b200.models.model import LatentDiffusion, PrecomputedLatentStubs
    gc.collect()
    net = MicroDiT_XL_2(input_size=32, in_channels=4)
    net.load_state_dict(weights.synth_state_dict(net.state_dict(), seed=pc.WEIGHT_SEED))
    ld = LatentDiffusion(net.to(DEV), *PrecomputedLatentStubs.make(), train_mask_ratio=0.75, latent_res=32)
    ld.train()
    B, mask_ratio = 2, 0.75
    batch = weights.synth_batch(B, 4, 32, seed=pc.BATCH_SEED)
    rnd, eps, _ = weights.replay_draws(pc.DRAW_SEED, (B, 4, 32, 32), 256, 0.0)
    x = batch["image_latents"].float().to(DEV)
    y = batch["caption_latents"].to(DEV)
    noise = vc.mask_noise(B, 256, DEV)
    ops = ld.dit.engine.ops
    ops.set_deterministic(True)
    try:
        ld.dit.zero_grad(set_to_none=True)
        ld.edm_loss_with_draws(x, y, None, rnd.reshape(-1), eps, noise, mask_ratio).backward()
        g_fused = ld.dit.store.grad.clone()
        ld.dit.zero_grad(set_to_none=True)
        e = ld.edm_config
        sigma = (rnd.to(DEV) * e.P_std + e.P_mean).exp()
        weight = (sigma ** 2 + e.sigma_data ** 2) / (sigma * e.sigma_data) ** 2
        torch.manual_seed(vc.MASK_SEED)  # DiT.forward draws the same mask noise
        out = ld.model_forward_wrapper(x + eps.to(DEV) * sigma, sigma, y, ld.dit, mask_ratio=mask_ratio)
        loss = weight * (out["sample"] - x) ** 2
        loss = F.avg_pool2d(loss.mean(dim=1), 2).flatten(1)
        unmask = 1 - out["mask"]
        loss = ((loss * unmask).sum(dim=1) / unmask.sum(dim=1)).mean()
        loss.backward()
        g_vjp = ld.dit.store.grad.clone()
    finally:
        ops.set_deterministic(False)
    names = ld.dit._param_names
    errs = sorted((rel(g_vjp[s:s + n], g_fused[s:s + n]), k) for k, (s, n) in
                  ((k, (ld.dit.store.layout.slots[k][0], ld.dit.store.g[k].numel())) for k in names))
    med, worst = errs[len(errs) // 2][0], errs[-1]
    print(f"\n[XL_2 C2 fused loss vs wrapper loss] whole-gradient rel-L2 {rel(g_vjp, g_fused):.2e}; per-parameter median "
          f"{med:.2e} worst {worst[0]:.2e} ({worst[1]})")
    assert rel(g_vjp, g_fused) < 5e-3 and med < 1e-5 and worst[0] < 1e-2, errs[-5:]
    del ld, net
    gc.collect()
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------ 4. determinism
@pytest.mark.parametrize("name", ["P", "S"])
def test_deterministic_vjp_is_bit_reproducible_and_frozen_mode_agrees(name):
    net = vc.build_dit(name, device=DEV)
    ops = net.engine.ops
    x, t, y, dF = vc.vjp_inputs(name, device=DEV)
    mask_ratio = max(vc.VJP_MASKS[name])
    ops.set_deterministic(True)
    try:
        a = vc.product_vjp(net, x, t, y, dF, mask_ratio)
        b = vc.product_vjp(net, x, t, y, dF, mask_ratio)
        c = vc.product_vjp(net, x, t, y, dF, mask_ratio, frozen=True)
    finally:
        ops.set_deterministic(False)
    for i in range(4):
        assert torch.equal(a[i], b[i]) and torch.equal(a[i], c[i]), i
    assert set(a[4]) == set(b[4]) and all(torch.equal(a[4][k], b[4][k]) for k in a[4])
    assert not c[4]


# ------------------------------------------------------------------------------------------------ 5. memory
def test_backward_releases_the_saved_context():
    net = vc.build_dit("S", device=DEV)
    x, t, y, dF = vc.vjp_inputs("S", device=DEV)
    vc.product_vjp(net, x, t, y, dF, 0.5)   # weight copies, gradient buffer, workspaces
    gc.collect()  # objects of earlier tests may still sit in reference cycles: free them before the baseline
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    xr = x.clone().requires_grad_(True)
    torch.manual_seed(vc.MASK_SEED)
    out = net(xr, t, y, mask_ratio=0.5)["sample"]
    held = torch.cuda.memory_allocated() - before
    out.backward(dF)
    del out
    xr.grad = None
    torch.cuda.synchronize()
    after = torch.cuda.memory_allocated()
    print(f"\n[S vjp] saved context {held / 2 ** 20:.1f} MiB; after backward {after - before} bytes above the start")
    assert held > 1 << 20 and 0 <= after - before <= xr.numel() * 4
