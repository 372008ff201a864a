"""Shared pieces of the DiT autograd (VJP) tests: the CPU contracts of the three adjoint kernels, the seeded VJP cases,
the oracle's autograd VJP and the product's, and the op-sequence recorder that pins the fused loss path."""
import math

import torch

from oracle import configs, port, weights
from oracle.emu_ops import EmuOps
from tests import parity_common as pc

VJP_SEED, MASK_SEED = 41, 43
VJP_MASKS = {"P": (0.0, 0.75), "S": (0.0,), "S16": (0.0,)}  # the cases stored in tests/golden/vjp_<cfg>.pt
REF_SAMPLES = 32


class VJPEmuOps(EmuOps):
    """EmuOps plus the CPU contracts of md_unpatchify_bwd / md_patchify_bwd / md_timestep_embed_bwd, and a count of the
    GEMM launches."""

    def __init__(self, device="cpu", exact=False):
        super().__init__(device, exact)
        self.gemm_launches = 0

    def gemm(self, *args, **kwargs):
        self.gemm_launches += 1
        return super().gemm(*args, **kwargs)

    def unpatchify_bwd(self, dF, keep_rows, dftok, p, Tk):
        """Adjoint of edm_output's un-mask + unpatchify: dF [B,C,H,W] -> dftok [B*Tk, p*p*C] (column (i*p+j)*C+c)."""
        self.launches += 1
        B, Cc, H, W = dF.shape
        T = (H // p) * (W // p)
        tok = dF.float().reshape(B, Cc, H // p, p, W // p, p).permute(0, 2, 4, 3, 5, 1).reshape(B * T, p * p * Cc)
        if keep_rows is not None:
            tok = tok[keep_rows.long()]
        dftok.copy_(tok.reshape(B * Tk, p * p * Cc))

    def patchify_bwd(self, dpatches, scale, dx, p):
        """Adjoint of patchify (col2im, column (c*p+i)*p+j): dpatches [B*T, C*p*p] -> dx [B,C,H,W]."""
        self.launches += 1
        B, Cc, H, W = dx.shape
        v = dpatches.float().reshape(B, H // p, W // p, Cc, p, p).permute(0, 3, 1, 4, 2, 5).reshape(B, Cc, H, W)
        dx.copy_(v * scale.view(B, 1, 1, 1) if scale is not None else v)

    def timestep_embed_bwd(self, dfreq, t, dt):
        """Adjoint of timestep_embed: dt[b] = sum_i f_i (dfreq[b, half+i] cos(t f_i) - dfreq[b, i] sin(t f_i))."""
        self.launches += 1
        half = dfreq.shape[1] // 2
        freqs = torch.exp(-math.log(10000.0) * torch.arange(half, dtype=torch.float32) / half)
        a = t.float()[:, None] * freqs[None]
        d = dfreq.float()
        dt.copy_((freqs[None] * (d[:, half:2 * half] * torch.cos(a) - d[:, :half] * torch.sin(a))).sum(1))


# ------------------------------------------------------------------------------------------------ seeded cases
def template(name):
    """Reference state_dict shapes (and the pos_embed buffer) of a parity config, without building a module."""
    from micro_diffusion_b200.arch import DiTConfig
    ct = configs.PARITY_CONFIGS[name]["ctor"]
    cfg = DiTConfig(**ct)
    sd = {k: torch.zeros(s) for k, s in cfg.buffer_specs() + cfg.param_specs()}
    g = ct["input_size"] // ct["patch_size"]
    sd["pos_embed"] = port.sincos_pos_embed(ct["dim"], g, ct.get("pos_interp_scale", 1.0), g).unsqueeze(0)
    return sd


def vjp_inputs(name, batch=None, device="cpu"):
    """x (the preconditioned input), t [B] (ln(sigma)/4 scale), y [B,1,77,Dc] (fp16-exact values) and the output
    cotangent dF: pure functions of VJP_SEED."""
    c = configs.PARITY_CONFIGS[name]
    ct = c["ctor"]
    B = batch or c["batch"]
    g = torch.Generator().manual_seed(VJP_SEED)
    x = torch.randn(B, ct["in_channels"], ct["input_size"], ct["input_size"], generator=g)
    t = 0.3 * torch.randn(B, generator=g)
    y = torch.randn(B, 1, 77, ct.get("caption_channels", 1024), generator=g).half().float()
    dF = torch.randn(B, ct["in_channels"], ct["input_size"], ct["input_size"], generator=g)
    return x.to(device), t.to(device), y.to(device), dF.to(device)


def mask_noise(rows, tokens, device="cpu"):
    """The uniform draw of get_mask (utils.py:390) that the default generator of `device` makes right after
    torch.manual_seed(MASK_SEED)."""
    return torch.rand(rows, tokens, device=device, generator=torch.Generator(device).manual_seed(MASK_SEED))


def port_vjp(name, x, t, y, dF, mask_ratio=0.0, noise=None, guidance=1.0):
    """fp32 oracle: F = DiT.forward (with_cfg when guidance != 1) and the autograd gradients of <F, dF> wrt x, t, y and
    every parameter."""
    c = configs.PARITY_CONFIGS[name]
    cfg = pc.port_config(c, c["ctor"])
    sd = weights.synth_state_dict(template(name), seed=pc.WEIGHT_SEED)
    P = {k: v.clone().requires_grad_(k not in ("pos_embed", "mask_token")) for k, v in sd.items()}
    x, t, y = (v.detach().float().cpu().clone().requires_grad_(True) for v in (x, t, y))
    if guidance == 1.0:
        F = port.dit_forward(P, cfg, x, t, y, mask_ratio, noise)["sample"]
    else:
        tt = t if len(t) == 1 else torch.cat([t, t], 0)
        out = port.dit_forward(P, cfg, torch.cat([x, x], 0), tt, torch.cat([y, torch.zeros_like(y)], 0), mask_ratio, noise)
        cond, unc = torch.split(out["sample"], x.shape[0], dim=0)
        F = unc + guidance * (cond - unc)
    (F * dF.float().cpu()).sum().backward()
    grads = {k: v.grad for k, v in P.items() if v.grad is not None}
    return F.detach(), x.grad, t.grad, y.grad, grads


def build_dit(name, ops_factory=None, device="cpu"):
    from micro_diffusion_b200.models.dit import DiT
    net = DiT(**configs.PARITY_CONFIGS[name]["ctor"], ops_factory=ops_factory)
    net.load_state_dict(weights.synth_state_dict(net.state_dict(), seed=pc.WEIGHT_SEED))
    return net.to(device) if device != "cpu" else net


def product_vjp(net, x, t, y, dF, mask_ratio=0.0, guidance=1.0, frozen=False):
    """F = net(x, t, y, cfg=guidance, mask_ratio=...) under autograd and the gradients of <F, dF> (on the host)."""
    net.requires_grad_(not frozen)
    net.zero_grad(set_to_none=True)
    x, t, y = (v.detach().clone().requires_grad_(True) for v in (x, t, y))
    torch.manual_seed(MASK_SEED)
    out = net(x, t, y, cfg=guidance, mask_ratio=mask_ratio)
    (out["sample"] * dF).sum().backward()
    grads = {k: p.grad.detach().float().cpu().clone() for k, p in net.named_parameters() if p.grad is not None}
    return out["sample"].detach().cpu(), x.grad.cpu(), t.grad.cpu(), y.grad.cpu(), grads


# ------------------------------------------------------------------------------------------------ fingerprints
def sample_index(name, numel):
    g = torch.Generator().manual_seed(sum(name.encode()) * 7919 + numel + 1)
    return torch.randint(0, numel, (min(REF_SAMPLES, numel),), generator=g)


def fingerprint(name, g):
    """Norm, dot with the seeded probe weights.synth_tensor("probe:" + name) and REF_SAMPLES seeded elements."""
    g = g.detach().float()
    pr = weights.synth_tensor("probe:" + name, g.shape, 99)
    flat = g.reshape(-1)
    idx = sample_index(name, flat.numel())
    return {"norm": float(g.norm()), "dot": float((g * pr).sum()), "index": idx, "values": flat[idx].clone()}


def fingerprint_error(name, g, fp):
    """Largest of the norm / dot / sampled-element deviations, relative to the stored norm."""
    g = g.detach().float()
    norm = fp["norm"] + 1e-30
    pr = weights.synth_tensor("probe:" + name, g.shape, 99)
    flat = g.reshape(-1)
    assert torch.equal(fp["index"], sample_index(name, flat.numel())), name
    return max(abs(float(g.norm()) - fp["norm"]) / norm,
               abs(float((g * pr).sum()) - fp["dot"]) / (norm * float(pr.norm())),
               float((flat[fp["index"]] - fp["values"]).abs().max()) / norm)


# ------------------------------------------------------------------------------------------------ loss-path pin
def _sig(v):
    if torch.is_tensor(v):
        return f"T{tuple(v.shape)}:{str(v.dtype).replace('torch.', '')}"
    if isinstance(v, float):
        return repr(round(v, 9))
    if v is None or isinstance(v, (bool, int, str)):
        return repr(v)
    return type(v).__name__


class RecordingEmuOps(EmuOps):
    """EmuOps (exact) that records every op call -- name, tensor shapes / dtypes and scalar arguments -- in order."""

    def __init__(self, device="cpu"):
        super().__init__(device, exact=True)
        self.calls = []

    def __getattribute__(self, attr):
        v = object.__getattribute__(self, attr)
        if attr.startswith("_") or not callable(v) or attr in ("set_deterministic",):
            return v
        calls = object.__getattribute__(self, "calls")

        def rec(*args, **kwargs):
            calls.append(attr + "(" + ",".join([_sig(a) for a in args] +
                                               [f"{k}={_sig(kwargs[k])}" for k in sorted(kwargs)]) + ")")
            return v(*args, **kwargs)
        return rec


def record_loss_path(name):
    """Op sequence of one fused training forward + backward (edm_loss_with_draws(...).backward())."""
    c, ct, batch, rnd, eps, noise = pc.case_inputs(name)
    ld = pc.build_product(name, ops_factory=lambda d: RecordingEmuOps(d))
    ops = ld.dit.engine.ops
    ops.calls.clear()
    loss = ld.edm_loss_with_draws(batch["image_latents"], batch["caption_latents"], batch["drop_caption_mask"],
                                  rnd.reshape(-1), eps, noise, c["mask_ratio"])
    n_fwd = len(ops.calls)
    loss.backward()
    return {"forward": ops.calls[:n_fwd], "backward": ops.calls[n_fwd:]}
