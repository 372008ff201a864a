"""Generate tests/golden/hd128_<cfg>.pt from the UNMODIFIED reference (needs $MICRODIT_REFERENCE_ROOT).

    python tools/make_hd128_golden.py

For the head_dim=128 configs H / HS (tests/hd128_common.HD128_CONFIGS), the reference DiT with synthetic weights
(oracle.weights, seed 7) in fp32 on CPU:
  * one training forward + backward of LatentDiffusion on the seeded case (the draws replayed from
    torch.manual_seed(123)): the loss, fingerprints (norm, dot with a seeded probe, seeded elements) of every parameter
    gradient, and the unmasked D_x on the same draws;
  * DiT.forward_without_cfg with x, t, y requiring grad and the gradient of <F, dF> for the seeded cotangent, at each
    mask ratio of hd128_common.VJP_MASKS: F, full dx and dt, fingerprints of dy and of every parameter gradient;
  * both again under amp-bf16 autocast: the reference's own bf16 deviation from its fp32 result, the bound the bf16 kernel
    path is held to;
  * the state_dict key / shape list.
hd128_H.pt also holds the key / shape list of DiT(head_dim=128) with every other argument at its default (built on the
meta device).
"""
from __future__ import annotations

import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import ref_import, weights  # noqa: E402
from tests import dit_vjp_common as vc  # noqa: E402
from tests import hd128_common as hc  # noqa: E402
from tests import parity_common as pc  # noqa: E402


def _dev(a, b):
    return sorted(pc.rel_l2(a[k], b[k]) for k in b)


def loss_case(ref_dit, name):
    c, ct, batch, rnd, eps, noise = hc.case_inputs(name)
    net = ref_dit.DiT(**ct)
    net.load_state_dict(weights.synth_state_dict(net.state_dict(), seed=pc.WEIGHT_SEED))
    ld = ref_import.build_reference_latent_diffusion(net, c["p_mean"], c["p_std"], c["mask_ratio"], ct["input_size"])
    ld.train()
    res = {}
    for mode in ("fp32", "bf16"):
        net.zero_grad(set_to_none=True)
        torch.manual_seed(pc.DRAW_SEED)
        with torch.autocast("cpu", dtype=torch.bfloat16, enabled=mode == "bf16"):
            loss, _, _ = ld({k: v.clone() for k, v in batch.items()})
        loss.backward()
        res[mode] = (float(loss), {k: p.grad.detach().clone() for k, p in net.named_parameters()})
    (l32, g32), (l16, g16) = res["fp32"], res["bf16"]
    dev = _dev(g16, g32)
    sigma = (rnd * c["p_std"] + c["p_mean"]).exp()
    x = batch["image_latents"].float()
    y = (batch["caption_latents"] * batch["drop_caption_mask"].view(-1, 1, 1, 1)).to(torch.float16).float()
    with torch.no_grad():
        net.eval()
        den = ld.model_forward_wrapper(x + eps * sigma, sigma, y, net, mask_ratio=0.0)["sample"]
    return net, {"loss": l32, "ref_amp_bf16_loss_rel": abs(l16 - l32) / l32,
                 "ref_amp_bf16_grad_rel_median": dev[len(dev) // 2], "ref_amp_bf16_grad_rel_max": dev[-1],
                 "denoised_unmasked": den.clone(), "grads": {k: vc.fingerprint(k, g) for k, g in g32.items()}}


def vjp_case(net, name, mask_ratio):
    net.train()
    x0, t0, y0, dF, _ = hc.vjp_case(name, mask_ratio)
    res = {}
    for mode in ("fp32", "bf16"):
        x, t, y = (v.clone().requires_grad_(True) for v in (x0, t0, y0))
        net.zero_grad(set_to_none=True)
        torch.manual_seed(vc.MASK_SEED)  # get_mask's torch.rand is the forward's only draw
        with torch.autocast("cpu", dtype=torch.bfloat16, enabled=mode == "bf16"):
            out = net.forward_without_cfg(x, t, y, mask_ratio=mask_ratio)
        (out["sample"].float() * dF).sum().backward()
        res[mode] = (out["sample"].detach().float(), x.grad, t.grad, y.grad,
                     {k: p.grad.detach().clone() for k, p in net.named_parameters()})
    (F, dx, dt, dy, grads), (bF, bdx, bdt, bdy, bgrads) = res["fp32"], res["bf16"]
    dev = _dev(bgrads, grads)
    return {"mask_ratio": mask_ratio, "F": F.clone(), "dx": dx.clone(), "dt": dt.clone(), "dy": vc.fingerprint("dy", dy),
            "grads": {k: vc.fingerprint(k, g) for k, g in grads.items()},
            "ref_amp_bf16": {"F": pc.rel_l2(bF, F), "dx": pc.rel_l2(bdx, dx), "dt": pc.rel_l2(bdt, dt),
                             "dy": pc.rel_l2(bdy, dy), "grad_rel_median": dev[len(dev) // 2], "grad_rel_max": dev[-1]}}


def main():
    ref_dit, _, _ = ref_import.load_reference()
    for name in hc.HD128_CONFIGS:
        net, fx = loss_case(ref_dit, name)
        fx.update({"config": name, "seeds": (pc.WEIGHT_SEED, pc.BATCH_SEED, pc.DRAW_SEED, vc.VJP_SEED, vc.MASK_SEED),
                   "keys": [(k, tuple(v.shape)) for k, v in net.state_dict().items()], "torch_version": torch.__version__})
        fx["vjp"] = {mr: vjp_case(net, name, mr) for mr in hc.VJP_MASKS[name]}
        if name == "H":
            with torch.device("meta"):
                dnet = ref_dit.DiT(head_dim=128)
            fx["default_dit_keys"] = [(k, tuple(v.shape)) for k, v in dnet.state_dict().items()]
        path = os.path.join(ROOT, "tests", "golden", f"hd128_{name}.pt")
        torch.save(fx, path)
        print(name, fx["loss"], fx["ref_amp_bf16_loss_rel"], {mr: v["ref_amp_bf16"] for mr, v in fx["vjp"].items()},
              f"-> {path} ({os.path.getsize(path) / 1024:.0f} KiB)")


if __name__ == "__main__":
    main()
