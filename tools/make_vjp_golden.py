"""Generate tests/golden/vjp_<cfg>.pt from the UNMODIFIED reference (needs $MICRODIT_REFERENCE_ROOT).

    python tools/make_vjp_golden.py

For P / S / S16: the reference DiT (synthetic weights, oracle.weights seed 7) in fp32 on CPU, DiT.forward_without_cfg
(dit.py:455-519) with x, t and y requiring grad, and the gradient of <F, dF> for a seeded cotangent dF
(tests/dit_vjp_common.vjp_inputs).  Every config at mask 0, P also at mask 0.75 with get_mask's torch.rand replayed
from torch.manual_seed(MASK_SEED).  Stored per case: F, full dx and dt, and fingerprints (norm, dot with a seeded probe,
seeded elements) of dy and of every parameter gradient.  Also the reference's own amp-bf16 deviation from its fp32 VJP
(relative L2 of F, dx, dt, dy; median and max over the parameter gradients): the yardstick the bf16 kernel path is held
to.  Inputs and weights are pure functions of the seeds.
"""
from __future__ import annotations

import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import configs, ref_import, weights  # noqa: E402
from tests import dit_vjp_common as vc  # noqa: E402
from tests import parity_common as pc  # noqa: E402


def main():
    ref_dit, _, _ = ref_import.load_reference()
    for name, masks in vc.VJP_MASKS.items():
        ct = configs.PARITY_CONFIGS[name]["ctor"]
        net = ref_dit.DiT(**ct)
        net.load_state_dict(weights.synth_state_dict(net.state_dict(), seed=pc.WEIGHT_SEED))
        net.train()
        fx = {"config": name, "seeds": (pc.WEIGHT_SEED, vc.VJP_SEED, vc.MASK_SEED), "cases": {},
              "torch_version": torch.__version__}
        for mask_ratio in masks:
            res = {}
            for mode in ("fp32", "bf16"):
                x, t, y, dF = (v.clone() for v in vc.vjp_inputs(name))
                for v in (x, t, y):
                    v.requires_grad_(True)
                net.zero_grad(set_to_none=True)
                torch.manual_seed(vc.MASK_SEED)  # get_mask's torch.rand is the forward's only draw
                with torch.autocast("cpu", dtype=torch.bfloat16, enabled=mode == "bf16"):
                    out = net.forward_without_cfg(x, t, y, mask_ratio=mask_ratio)
                (out["sample"].float() * dF).sum().backward()
                res[mode] = (out, x.grad, t.grad, y.grad, {k: p.grad.detach().clone() for k, p in net.named_parameters()})
            out, dx, dt, dy, grads = res["fp32"]
            b_out, b_dx, b_dt, b_dy, b_grads = res["bf16"]
            dev = sorted(pc.rel_l2(b_grads[k], grads[k]) for k in grads)
            case = {"F": out["sample"].detach().clone(), "dx": dx.clone(), "dt": dt.clone(),
                    "dy": vc.fingerprint("dy", dy), "grads": {k: vc.fingerprint(k, g) for k, g in grads.items()},
                    "ref_amp_bf16": {"F": pc.rel_l2(b_out["sample"].detach(), out["sample"].detach()),
                                     "dx": pc.rel_l2(b_dx, dx), "dt": pc.rel_l2(b_dt, dt), "dy": pc.rel_l2(b_dy, dy),
                                     "grad_rel_median": dev[len(dev) // 2], "grad_rel_max": dev[-1]}}
            if mask_ratio > 0:
                case["mask"] = out["mask"].detach().clone()
                g = ct["input_size"] // ct["patch_size"]
                assert torch.equal(vc.mask_noise(dx.shape[0], g * g).argsort(1).argsort(1) >= int(g * g * (1 - mask_ratio)),
                                   case["mask"].bool()), "get_mask replay does not match the global RNG stream"
            fx["cases"][mask_ratio] = case
            print(name, mask_ratio, float(out["sample"].detach().norm()), float(dx.norm()), case["ref_amp_bf16"])
        path = os.path.join(ROOT, "tests", "golden", f"vjp_{name}.pt")
        torch.save(fx, path)
        print(f"-> {path} ({os.path.getsize(path) / 1024:.0f} KiB)")


if __name__ == "__main__":
    main()
