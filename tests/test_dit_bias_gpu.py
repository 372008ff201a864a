"""use_bias=True end to end on the GPU: the bf16 CUDA path on the biased parity configs against the fixtures of the
unmodified reference (tests/golden/bias_*.pt) and the fp32 oracle, the high-precision mode, the unfused SwiGLU, the
deterministic mode, the VJP, and the reference DiT's default widths (dim 1152, mixer 4 x 512 with biased maps).
Bounds as tests/test_parity_gpu.py: relative to the reference's own recorded amp-bf16 deviation."""
import gc

import pytest
import torch

from oracle import port, weights
from tests import bias_common as bc
from tests import dit_vjp_common as vc
from tests import parity_common as pc

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
CASES = list(bc.BIAS_CONFIGS)
rel = pc.rel_l2


def _high_ops(device):
    from micro_diffusion_b200.ops import CudaOps
    return CudaOps(device, precision="high")


def _free():
    gc.collect()
    torch.cuda.empty_cache()


@pytest.mark.parametrize("name", CASES)
def test_cuda_path_matches_oracle_and_golden(name):
    fx = bc.golden(name)
    loss, grads, den, ld = bc.product_run(name, device=DEV)
    ops = ld.dit.engine.ops
    assert ops.launches > 100 and not ops.is_emulation and ld.dit.store.interleave
    del ld
    _free()
    oloss, ograds, oden = bc.oracle_run(name)
    errs, med, worst = pc.grad_report(grads, ograds)
    print(f"\n[{name}] loss cuda {loss:.6f} golden {fx['loss']:.6f} rel {abs(loss - fx['loss']) / fx['loss']:.2e} | "
          f"D_x relL2 {rel(den, fx['denoised_unmasked']):.2e} | grads median {med:.2e} worst {worst:.2e} ({errs[0][1]}) | "
          f"reference amp-bf16: loss {fx['ref_amp_bf16_loss_rel']:.2e} grads median {fx['ref_amp_bf16_grad_rel_median']:.2e}"
          f" worst {fx['ref_amp_bf16_grad_rel_max']:.2e}")
    assert abs(oloss - fx["loss"]) / fx["loss"] < 1e-5
    assert abs(loss - fx["loss"]) / fx["loss"] < 3e-3
    assert rel(den, fx["denoised_unmasked"]) < max(1e-2, fx["vjp"]["ref_amp_bf16"]["F"])
    assert med < 1.5 * fx["ref_amp_bf16_grad_rel_median"] + 5e-3
    assert worst < 2 * fx["ref_amp_bf16_grad_rel_max"] + 2e-2, errs[:5]
    for k, g in fx["grad_full"].items():
        assert rel(grads[k], g) < 2 * fx["ref_amp_bf16_grad_rel_max"] + 2e-2, k


@pytest.mark.parametrize("name", CASES)
def test_high_precision_mode_meets_1e3(name):
    fx = bc.golden(name)
    loss, grads, den, ld = bc.product_run(name, ops_factory=_high_ops, device=DEV)
    assert ld.dit.engine.ops.prec == 1
    del ld
    _free()
    lrel, drel = abs(loss - fx["loss"]) / fx["loss"], rel(den, fx["denoised_unmasked"])
    print(f"\n[{name} high] loss rel {lrel:.2e} D_x relL2 {drel:.2e}")
    assert lrel < 1e-3 and drel < 1e-3


def test_unfused_swiglu_agrees_with_the_fused_epilogue(monkeypatch):
    """MD_FUSE_SWIGLU=0 (read when the model is built): plain GEMM with the [b1 | b2] bias + md_swiglu_fwd, plain column
    sums of du -- the same function as the biased epilogue and md_colsum_interleaved, within bf16 noise."""
    l1, g1, d1, ld = bc.product_run("SB", device=DEV)
    assert ld.dit.store.interleave
    del ld
    monkeypatch.setenv("MD_FUSE_SWIGLU", "0")
    l0, g0, d0, ld = bc.product_run("SB", device=DEV)
    assert not ld.dit.store.interleave
    del ld
    _free()
    errs = sorted((rel(g1[k], g0[k]), k) for k in g0)
    print(f"\n[SB fused vs unfused] loss {abs(l1 - l0) / l0:.2e} D_x {rel(d1, d0):.2e} grads median "
          f"{errs[len(errs) // 2][0]:.2e} worst {errs[-1]}")
    assert abs(l1 - l0) / abs(l0) < 1e-3 and rel(d1, d0) < 1e-2
    assert errs[-1][0] < 5e-2 and errs[len(errs) // 2][0] < 1e-2, errs[-3:]
    b = [e for e, k in errs if k.endswith("mlp.w1.bias") or k.endswith("mlp.w2.bias")]
    assert b and max(b) < 2e-2


def test_deterministic_mode_reproduces_a_biased_step_bit_for_bit():
    from micro_diffusion_b200.train_step import FlatAdamW

    def one_step():
        _free()
        ld = bc.build_product("SB", device=DEV)
        ops = ld.dit.engine.ops
        ops.set_deterministic(True)
        try:
            opt = FlatAdamW(ld.dit, lr=1e-3, clip_norm=0.25)
            batch = {k: v.to(DEV) for k, v in weights.synth_batch(6, 4, 16, seed=5).items()}
            total = 0.0
            for i, s0 in enumerate(range(0, 6, 3)):
                torch.manual_seed(123 + i)
                loss = ld({k: v[s0:s0 + 3] for k, v in batch.items()})[0]
                (loss * 0.5).backward()
                total += float(loss.detach())
            g = ld.dit.store.grad.cpu()
            opt.step()
            torch.cuda.synchronize()
            return total, g, ld.dit.store.flat.cpu()
        finally:
            ops.set_deterministic(False)
            del ld

    l1, g1, w1 = one_step()
    l2, g2, w2 = one_step()
    assert l1 == l2 and torch.equal(g1, g2) and torch.equal(w1, w2)


@pytest.mark.parametrize("name", CASES)
def test_vjp_within_reference_amp_class(name):
    fx = bc.golden(name)["vjp"]
    amp = fx["ref_amp_bf16"]
    net = bc.build_dit(name, device=DEV)
    x, t, y, dF, mr, noise = bc.vjp_case(name)
    if mr > 0:  # get_mask draws from the CUDA generator here: the oracle replays that draw
        noise = vc.mask_noise(x.shape[0], noise.shape[1], DEV).cpu()
    F, dx, dt, dy, grads = vc.product_vjp(net, *(v.to(DEV) for v in (x, t, y, dF)), mr)
    del net
    _free()
    oF, odx, odt, ody, ograds = bc.port_vjp(name, x, t, y, dF, mr, noise)
    if mr == 0:
        assert rel(oF, fx["F"]) < 1e-5 and rel(odx, fx["dx"]) < 1e-5
    errs, med, worst = pc.grad_report(grads, ograds)
    ie = {"F": rel(F, oF), "dx": rel(dx, odx), "dt": rel(dt, odt), "dy": rel(dy, ody)}
    print(f"\n[{name} VJP] {ie} grads median {med:.2e} worst {worst:.2e} | reference amp-bf16 {amp}")
    for k, e in ie.items():
        assert e < 2 * amp[k] + 2e-2, (k, e, amp[k])
    assert med < 1.5 * amp["grad_rel_median"] + 5e-3 and worst < 2 * amp["grad_rel_max"] + 2e-2, errs[:5]


def test_frozen_vjp_input_gradients_are_bit_identical_in_deterministic_mode():
    net = bc.build_dit("SB", device=DEV)
    ops = net.engine.ops
    x, t, y, dF, mr, _ = bc.vjp_case("SB")
    ops.set_deterministic(True)
    try:
        flat0 = net.store.grad.clone()
        full = vc.product_vjp(net, *(v.to(DEV) for v in (x, t, y, dF)), mr)
        flat1 = net.store.grad.clone()
        frozen = vc.product_vjp(net, *(v.to(DEV) for v in (x, t, y, dF)), mr, frozen=True)
        assert torch.equal(net.store.grad, flat1) and not torch.equal(flat0, flat1)
    finally:
        ops.set_deterministic(False)
    for i in range(4):
        assert torch.equal(full[i], frozen[i]), i
    assert not frozen[4]
    del net
    _free()


def test_default_dit_widths_match_the_oracle():
    """DiT with every default but depth=4 (dim 1152, 18 heads of 64, mixer 4 x 512 with biased maps, expert capacity 1)
    at mask 0.75, batch 2: the generic (non-specialised) row kernels, against the fp32 port on the same seeded weights,
    with the zoo bounds of test_xl2_matches_oracle."""
    from micro_diffusion_b200.models.dit import DiT
    from micro_diffusion_b200.models.model import LatentDiffusion, PrecomputedLatentStubs
    mask_ratio, B, p_mean, p_std = 0.75, 2, -0.6, 1.2
    net = DiT(depth=4, input_size=32)
    assert net.cfg.use_bias and net.cfg.has_mixer_maps and net.cfg.dim == 1152
    net.load_state_dict(weights.synth_state_dict(net.state_dict(), seed=7))
    sd_cpu = {k: v.detach().clone() for k, v in net.state_dict().items()}
    ld = LatentDiffusion(net.to(DEV), *PrecomputedLatentStubs.make(), p_mean=p_mean, p_std=p_std,
                         train_mask_ratio=mask_ratio, latent_res=32)
    ld.train()
    batch = weights.synth_batch(B, 4, 32, seed=11)
    rnd, eps, noise = weights.replay_draws(123, (B, 4, 32, 32), 256, mask_ratio)
    loss = ld.edm_loss_with_draws(batch["image_latents"], batch["caption_latents"], batch["drop_caption_mask"],
                                  rnd.reshape(-1), eps, noise, mask_ratio)
    loss.backward()
    grads = {k: p.grad.detach().float().cpu() for k, p in net.named_parameters()}
    sigma = (rnd * p_std + p_mean).exp()
    x = batch["image_latents"].float()
    y = (batch["caption_latents"] * batch["drop_caption_mask"].view(-1, 1, 1, 1)).to(torch.float16)
    with torch.no_grad():
        net.eval()
        den = ld.model_forward_wrapper((x + eps * sigma).to(DEV), sigma.to(DEV), y.to(DEV), net, mask_ratio=0.0)["sample"]
    den, loss = den.float().cpu(), float(loss.detach())
    del ld, net
    _free()
    P = {k: v.clone().requires_grad_(k not in ("pos_embed", "mask_token")) for k, v in sd_cpu.items()}
    cfg = port.PortConfig(patch_size=2, head_dim=64, num_experts=8, expert_capacity=1.0, p_mean=p_mean, p_std=p_std)
    oloss, _ = port.latent_diffusion_forward(P, cfg, batch, rnd, eps, mask_ratio, noise)
    oloss.backward()
    ograds = {k: v.grad for k, v in P.items() if v.grad is not None}
    with torch.no_grad():
        oden = port.denoise({k: v.detach() for k, v in P.items()}, cfg, x + eps * sigma, sigma, y.float())["sample"]
    errs, med, worst = pc.grad_report(grads, ograds)
    lrel, drel = abs(loss - float(oloss)) / float(oloss), rel(den, oden)
    print(f"\n[DiT defaults, depth 4] loss rel {lrel:.2e} D_x relL2 {drel:.2e} grads median {med:.2e} worst {worst:.2e} "
          f"({errs[0][1]})")
    assert lrel < 5e-3 and drel < 2e-2
    assert med < 4e-2 and worst < 0.3, errs[:5]


def test_create_latent_diffusion_with_the_reference_dit_trains_and_samples():
    """dit_arch="DiT" (the Hydra _target_ path, every DiT default: 28 blocks of width 1152 with biases) with the
    precomputed-latent stubs: one training step, then a 2-step CFG sampler call with and without the prompt cache."""
    from micro_diffusion_b200.models.model import PrecomputedLatentStubs, create_latent_diffusion
    from micro_diffusion_b200.train_step import FlatAdamW
    _free()
    vae, te, tok = PrecomputedLatentStubs.make()
    ld = create_latent_diffusion(dit_arch="DiT", latent_res=32, train_mask_ratio=0.75, vae=vae, text_encoder=te,
                                 tokenizer=tok)
    assert ld.dit.cfg.use_bias and len(ld.dit.cfg.blocks) == 28
    ld.dit.to(DEV)
    ld.train()
    opt = FlatAdamW(ld.dit, lr=1e-4, clip_norm=0.25)
    batch = {k: v.to(DEV) for k, v in weights.synth_batch(2, 4, 32, seed=3).items()}
    torch.manual_seed(0)
    loss = ld(batch)[0]
    loss.backward()
    assert torch.isfinite(loss) and float(ld.dit.store.grad.abs().max()) > 0
    opt.step()
    ld.eval()
    g = torch.Generator(device=DEV).manual_seed(1)
    x = torch.randn(2, 4, 32, 32, device=DEV, generator=g)
    y = torch.randn(2, 1, 77, 1024, device=DEV, generator=g).half()
    ld.cache_prompt = True
    a = ld.edm_sampler_loop(x, y, steps=2, cfg=3.0)
    ld.cache_prompt = False
    b = ld.edm_sampler_loop(x, y, steps=2, cfg=3.0)
    print(f"\n[create_latent_diffusion DiT] loss {float(loss.detach()):.4f} sampler cached vs uncached {rel(a, b):.2e}")
    assert torch.isfinite(a).all() and torch.isfinite(b).all()
    assert rel(a, b) < 1e-2
    del ld, opt
    _free()
