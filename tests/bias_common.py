"""Shared pieces of the use_bias=True tests: the biased parity configs, the CPU contracts of the biased fused SwiGLU and
of the interleaved column sum, and the seeded loss / VJP cases of the oracle and of the product on those configs."""
import copy
import os

import torch

from oracle import port, weights
from oracle.configs import PARITY_CONFIGS
from oracle.emu_ops import EPI_SWIGLU, interleave_perm
from tests import dit_vjp_common as vc
from tests import parity_common as pc

# every parity config again with the reference's default use_bias=True:
#   PB   P  (mixer width = backbone width: identity maps; head_dim 32, mask 0.75, interleaved SwiGLU)
#   SB   S  (mixer maps with biases, MoE, per-block ratios, mask 0.5)
#   S16B S16 (head_dim 64, 16 latent channels, mask 0)
BASE = {"PB": "P", "SB": "S", "S16B": "S16"}
BIAS_CONFIGS = {}
for _b, _p in BASE.items():
    BIAS_CONFIGS[_b] = copy.deepcopy(PARITY_CONFIGS[_p])
    BIAS_CONFIGS[_b]["ctor"]["use_bias"] = True
VJP_MASK = {"PB": 0.75, "SB": 0.0, "S16B": 0.0}  # the VJP case stored in tests/golden/bias_<cfg>.pt
DEFAULT_KEYS = os.path.join(pc.GOLDEN, "bias_default_dit_keys.json")


def golden(name):
    return torch.load(os.path.join(pc.GOLDEN, f"bias_{name}.pt"), weights_only=False)


class BiasEmuOps(vc.VJPEmuOps):
    """VJPEmuOps plus the CPU contracts of the bias of MD_EPI_SWIGLU (natural-order [b1 | b2], mapped onto the interleaved
    columns) and of md_colsum_interleaved.  Every other op is the stock contract."""

    def gemm(self, A, B, Cm, *, epi=0, bias=None, **kw):
        if epi == EPI_SWIGLU and bias is not None:
            bias = bias.index_select(-1, interleave_perm(bias.shape[-1] // 2))
        return super().gemm(A, B, Cm, epi=epi, bias=bias, **kw)

    def colsum_interleaved(self, x, out, half):
        self.launches += 1
        out.index_add_(0, interleave_perm(half), x.float().sum(0))


# ------------------------------------------------------------------------------------------------ seeded cases
def case_inputs(name):
    """(config, ctor, batch, rnd, eps, mask noise): the parity case of the base config (the draws do not depend on
    use_bias)."""
    _, _, batch, rnd, eps, noise = pc.case_inputs(BASE[name])
    c = BIAS_CONFIGS[name]
    return c, c["ctor"], batch, rnd, eps, noise


def template(name):
    """Reference state_dict shapes (and the pos_embed buffer) of a bias config, without building a module."""
    from micro_diffusion_b200.arch import DiTConfig
    ct = BIAS_CONFIGS[name]["ctor"]
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
    net = DiT(**BIAS_CONFIGS[name]["ctor"], ops_factory=ops_factory)
    net.load_state_dict(weights.synth_state_dict(net.state_dict(), seed=pc.WEIGHT_SEED))
    return net.to(device) if device != "cpu" else net


def build_product(name, ops_factory=None, device="cpu"):
    from micro_diffusion_b200.models.model import LatentDiffusion, PrecomputedLatentStubs
    c = BIAS_CONFIGS[name]
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


def vjp_case(name):
    """(x, t, y, dF, mask_ratio, mask noise) of the stored VJP case."""
    x, t, y, dF = vc.vjp_inputs(BASE[name])
    mr = VJP_MASK[name]
    ct = BIAS_CONFIGS[name]["ctor"]
    noise = vc.mask_noise(x.shape[0], (ct["input_size"] // ct["patch_size"]) ** 2) if mr > 0 else None
    return x, t, y, dF, mr, noise


def port_vjp(name, x, t, y, dF, mask_ratio=0.0, noise=None):
    """fp32 oracle: F = DiT.forward and the autograd gradients of <F, dF> wrt x, t, y and every parameter."""
    c = BIAS_CONFIGS[name]
    cfg = pc.port_config(c, c["ctor"])
    sd = weights.synth_state_dict(template(name), seed=pc.WEIGHT_SEED)
    P = {k: v.clone().requires_grad_(k not in ("pos_embed", "mask_token")) for k, v in sd.items()}
    x, t, y = (v.detach().float().cpu().clone().requires_grad_(True) for v in (x, t, y))
    F = port.dit_forward(P, cfg, x, t, y, mask_ratio, noise)["sample"]
    (F * dF.float().cpu()).sum().backward()
    return F.detach(), x.grad, t.grad, y.grad, {k: v.grad for k, v in P.items() if v.grad is not None}
