"""Shared pieces of the head_dim=128 tests: the two parity configs with 128-wide attention heads, and the seeded loss /
VJP cases of the oracle and of the product on them (built like tests/bias_common.py, with the seeds of
tests/parity_common.py and tests/dit_vjp_common.py)."""
import os

import torch

from oracle import port, weights
from tests import bias_common as bc
from tests import dit_vjp_common as vc
from tests import parity_common as pc

#   H   dim 256 (two backbone heads), a one-head mixer (patch_mixer_dim 128: mixer maps), mask 0.75, no biases
#   HS  dim 384, per-block qkv ratios -> 2 / 3 / 6 / 3 heads, 2 mixer heads (patch_mixer_dim 256: mixer maps), 3
#       cross-attention heads, MoE in the backbone, use_bias=True, mask 0
HD128_CONFIGS = {
    "H": dict(ctor=dict(input_size=32, patch_size=2, in_channels=4, dim=256, depth=2, head_dim=128,
                        patch_mixer_depth=2, patch_mixer_dim=128, use_bias=False, expert_capacity=2.0),
              batch=4, mask_ratio=0.75, p_mean=-0.6, p_std=1.2),
    "HS": dict(ctor=dict(input_size=16, patch_size=2, in_channels=4, dim=384, depth=4, head_dim=128,
                         multiple_of=64, qkv_multipliers=[0.5, 1.0, 1.5, 1.0], ffn_multipliers=[0.5, 1.5, 2.5, 4.0],
                         patch_mixer_depth=2, patch_mixer_dim=256, patch_mixer_qkv_ratio=1.0,
                         patch_mixer_mlp_ratio=2.0, use_bias=True, num_experts=8, expert_capacity=2.0,
                         pos_interp_scale=2.0),
               batch=3, mask_ratio=0.0, p_mean=0.0, p_std=0.6),
}
VJP_MASKS = {"H": (0.0, 0.75), "HS": (0.0,)}  # the VJP cases stored in tests/golden/hd128_<cfg>.pt

# biased configs need the bias contracts of the fused SwiGLU; they are the stock contracts everywhere else
Emu = bc.BiasEmuOps


def golden(name):
    return torch.load(os.path.join(pc.GOLDEN, f"hd128_{name}.pt"), weights_only=False)


def case_inputs(name):
    """(config, ctor, batch, rnd, eps, mask noise) of the seeded loss case."""
    c = HD128_CONFIGS[name]
    ct = c["ctor"]
    batch = weights.synth_batch(c["batch"], ct["in_channels"], ct["input_size"], seed=pc.BATCH_SEED)
    g = ct["input_size"] // ct["patch_size"]
    rnd, eps, noise = weights.replay_draws(pc.DRAW_SEED, (c["batch"], ct["in_channels"], ct["input_size"],
                                                          ct["input_size"]), g * g, c["mask_ratio"])
    return c, ct, batch, rnd, eps, noise


def template(name):
    """Reference state_dict shapes (and the pos_embed buffer) of a config, without building a module."""
    from micro_diffusion_b200.arch import DiTConfig
    ct = HD128_CONFIGS[name]["ctor"]
    cfg = DiTConfig(**ct)
    sd = {k: torch.zeros(s) for k, s in cfg.buffer_specs() + cfg.param_specs()}
    g = ct["input_size"] // ct["patch_size"]
    sd["pos_embed"] = port.sincos_pos_embed(ct["dim"], g, ct.get("pos_interp_scale", 1.0), g).unsqueeze(0)
    return sd


def oracle_run(name):
    """fp32 oracle on the seeded weights: loss, parameter grads, unmasked D_x."""
    c, ct, batch, rnd, eps, noise = case_inputs(name)
    sd = weights.synth_state_dict(template(name), seed=pc.WEIGHT_SEED)
    P = {k: v.clone().requires_grad_(k not in ("pos_embed", "mask_token")) for k, v in sd.items()}
    cfg = pc.port_config(c, ct)
    loss, _ = port.latent_diffusion_forward(P, cfg, batch, rnd, eps, c["mask_ratio"], noise)
    loss.backward()
    grads = {k: v.grad for k, v in P.items() if v.grad is not None}
    with torch.no_grad():
        sigma = (rnd * c["p_std"] + c["p_mean"]).exp()
        x = batch["image_latents"].float()
        y = (batch["caption_latents"] * batch["drop_caption_mask"].view(-1, 1, 1, 1)).to(torch.float16).float()
        den = port.denoise({k: v.detach() for k, v in P.items()}, cfg, x + eps * sigma, sigma, y)["sample"]
    return float(loss.detach()), grads, den


def build_dit(name, ops_factory=None, device="cpu"):
    from micro_diffusion_b200.models.dit import DiT
    net = DiT(**HD128_CONFIGS[name]["ctor"], ops_factory=ops_factory)
    net.load_state_dict(weights.synth_state_dict(net.state_dict(), seed=pc.WEIGHT_SEED))
    return net.to(device) if device != "cpu" else net


def build_product(name, ops_factory=None, device="cpu"):
    from micro_diffusion_b200.models.model import LatentDiffusion, PrecomputedLatentStubs
    c = HD128_CONFIGS[name]
    net = build_dit(name, ops_factory, device)
    ld = LatentDiffusion(net, *PrecomputedLatentStubs.make(), p_mean=c["p_mean"], p_std=c["p_std"],
                         train_mask_ratio=c["mask_ratio"], latent_res=c["ctor"]["input_size"])
    ld.train()
    return ld


def product_run(name, ops_factory=None, device="cpu", ld=None):
    """The fused EDM loss step (forward + backward) and the unmasked D_x of the product on the seeded case."""
    c, ct, batch, rnd, eps, noise = case_inputs(name)
    ld = ld or build_product(name, ops_factory, device)
    loss = ld.edm_loss_with_draws(batch["image_latents"], batch["caption_latents"], batch["drop_caption_mask"],
                                  rnd.reshape(-1), eps, noise, c["mask_ratio"])
    loss.backward()
    grads = {k: p.grad.detach().float().cpu() for k, p in ld.dit.named_parameters()}
    with torch.no_grad():
        sigma = (rnd * c["p_std"] + c["p_mean"]).exp()
        x = batch["image_latents"].float()
        y = (batch["caption_latents"] * batch["drop_caption_mask"].view(-1, 1, 1, 1)).to(torch.float16)
        dev = ld.dit.store.device
        ld.dit.eval()
        den = ld.model_forward_wrapper((x + eps * sigma).to(dev), sigma.to(dev), y.to(dev), ld.dit, mask_ratio=0.0)["sample"]
        ld.dit.train()
    return float(loss.detach()), grads, den.float().cpu(), ld


def vjp_inputs(name):
    """x, t, y, dF of the VJP case: the draws of dit_vjp_common.vjp_inputs at this config's shapes."""
    c = HD128_CONFIGS[name]
    ct = c["ctor"]
    B = c["batch"]
    g = torch.Generator().manual_seed(vc.VJP_SEED)
    x = torch.randn(B, ct["in_channels"], ct["input_size"], ct["input_size"], generator=g)
    t = 0.3 * torch.randn(B, generator=g)
    y = torch.randn(B, 1, 77, ct.get("caption_channels", 1024), generator=g).half().float()
    dF = torch.randn(B, ct["in_channels"], ct["input_size"], ct["input_size"], generator=g)
    return x, t, y, dF


def vjp_case(name, mask_ratio):
    """(x, t, y, dF, mask noise) of a stored VJP case."""
    x, t, y, dF = vjp_inputs(name)
    ct = HD128_CONFIGS[name]["ctor"]
    noise = vc.mask_noise(x.shape[0], (ct["input_size"] // ct["patch_size"]) ** 2) if mask_ratio > 0 else None
    return x, t, y, dF, noise


def port_vjp(name, x, t, y, dF, mask_ratio=0.0, noise=None):
    """fp32 oracle: F = DiT.forward and the autograd gradients of <F, dF> wrt x, t, y and every parameter."""
    c = HD128_CONFIGS[name]
    cfg = pc.port_config(c, c["ctor"])
    sd = weights.synth_state_dict(template(name), seed=pc.WEIGHT_SEED)
    P = {k: v.clone().requires_grad_(k not in ("pos_embed", "mask_token")) for k, v in sd.items()}
    x, t, y = (v.detach().float().cpu().clone().requires_grad_(True) for v in (x, t, y))
    F = port.dit_forward(P, cfg, x, t, y, mask_ratio, noise)["sample"]
    (F * dF.float().cpu()).sum().backward()
    return F.detach(), x.grad, t.grad, y.grad, {k: v.grad for k, v in P.items() if v.grad is not None}
