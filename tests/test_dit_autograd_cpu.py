"""Autograd through DiT.forward and model_forward_wrapper on CPU, with the kernels replaced by their CPU contracts
(oracle.emu_ops + the adjoint contracts of tests/dit_vjp_common.py): the oracle is pinned to the reference's autograd
(tests/golden/vjp_*.pt), the adjoint contracts to torch.autograd of the ops they invert, the engine's VJP to the
oracle, and the fused loss path to the op sequence it issued before the VJP existed (tests/golden/loss_path_ops.json)."""
import json
import os
from functools import partial

import pytest
import torch

from oracle import configs, port
from oracle.emu_ops import EmuOps
from tests import dit_vjp_common as vc
from tests import parity_common as pc

CASES = list(configs.PARITY_CONFIGS)
rel = pc.rel_l2


def _grid(name):
    ct = configs.PARITY_CONFIGS[name]["ctor"]
    return ct["input_size"] // ct["patch_size"]


# ------------------------------------------------------------------------------------------------ 1. oracle vs reference
@pytest.mark.parametrize("name", CASES)
def test_port_vjp_matches_reference_fixture(name):
    fx = torch.load(os.path.join(pc.GOLDEN, f"vjp_{name}.pt"), weights_only=False)
    assert set(fx["cases"]) == set(vc.VJP_MASKS[name])
    for mask_ratio, ref in fx["cases"].items():
        x, t, y, dF = vc.vjp_inputs(name)
        noise = vc.mask_noise(x.shape[0], _grid(name) ** 2) if mask_ratio > 0 else None
        F, dx, dt, dy, grads = vc.port_vjp(name, x, t, y, dF, mask_ratio, noise)
        assert rel(F, ref["F"]) < 1e-5 and rel(dx, ref["dx"]) < 1e-5 and rel(dt, ref["dt"]) < 1e-5, mask_ratio
        assert vc.fingerprint_error("dy", dy, ref["dy"]) < 1e-5
        assert set(grads) == set(ref["grads"])
        errs = sorted((vc.fingerprint_error(k, grads[k], fp), k) for k, fp in ref["grads"].items())
        assert errs[-1][0] < 1e-5, errs[-3:]


# ------------------------------------------------------------------------------------------------ 2. adjoint contracts
def _vjp(f, x, cot):
    x = x.detach().clone().requires_grad_(True)
    (f(x) * cot).sum().backward()
    return x.grad


@pytest.mark.parametrize("C,p,masked", [(4, 2, False), (4, 2, True), (16, 2, True), (4, 4, False)])
def test_unpatchify_bwd_is_the_adjoint_of_edm_output(C, p, masked):
    o = vc.VJPEmuOps(exact=True)
    B, H = 3, 16
    T = (H // p) ** 2
    g = torch.Generator().manual_seed(1)
    Tk = T // 4 if masked else T
    restore = keep = None
    if masked:
        ids_restore = torch.empty(B, T, dtype=torch.int32)
        keep = torch.empty(B * Tk, dtype=torch.int32)
        o.mask_sort(torch.rand(B, T, generator=g), None, ids_restore, torch.empty(B, T), keep, Tk)
        restore = ids_restore
    mt = torch.randn(p * p * C, generator=g)
    dF = torch.randn(B, C, H, H, generator=g)

    def fwd(ftok):
        fx = torch.empty(B, C, H, H)
        with torch.enable_grad():
            # edm_output as a differentiable torch expression: the same gather / reshape the contract performs
            Nf = p * p * C
            f = ftok.reshape(B, Tk, Nf)
            if restore is not None:
                full = torch.cat([f, mt.reshape(1, 1, Nf).expand(B, T - Tk, Nf)], 1)
                f = torch.gather(full, 1, restore.long()[..., None].expand(B, T, Nf))
            img = f.reshape(B, H // p, H // p, p, p, C).permute(0, 5, 1, 3, 2, 4).reshape(B, C, H, H)
        o.edm_output(ftok.detach(), restore, mt, None, None, fx, None, p, Tk)
        assert torch.equal(fx, img.detach())
        return img

    ref = _vjp(fwd, torch.randn(B * Tk, p * p * C, generator=g), dF)
    out = torch.empty(B * Tk, p * p * C)
    o.unpatchify_bwd(dF, keep, out, p, Tk)
    assert torch.allclose(out, ref, atol=1e-6)


@pytest.mark.parametrize("C,p,scaled", [(4, 2, False), (4, 2, True), (16, 2, True), (4, 4, False)])
def test_patchify_bwd_is_the_adjoint_of_patchify(C, p, scaled):
    o = vc.VJPEmuOps(exact=True)
    B, H = 2, 16
    g = torch.Generator().manual_seed(2)
    scale = torch.rand(B, generator=g) + 0.5 if scaled else None
    cot = torch.randn(B * (H // p) ** 2, C * p * p, generator=g)

    def fwd(x):
        out = torch.empty(cot.shape)
        o.patchify(x.detach(), scale, out, p)
        v = x * (scale.view(B, 1, 1, 1) if scaled else 1.0)
        t = v.reshape(B, C, H // p, p, H // p, p).permute(0, 2, 4, 1, 3, 5).reshape(cot.shape)
        assert torch.equal(out, t.detach())
        return t

    ref = _vjp(fwd, torch.randn(B, C, H, H, generator=g), cot)
    dx = torch.empty(B, C, H, H)
    o.patchify_bwd(cot, scale, dx, p)
    assert torch.allclose(dx, ref, atol=1e-6)


@pytest.mark.parametrize("dim", [256, 512])
def test_timestep_embed_bwd_is_the_adjoint_of_timestep_embed(dim):
    o = vc.VJPEmuOps(exact=True)
    g = torch.Generator().manual_seed(3)
    t = 2 * torch.randn(5, generator=g)
    cot = torch.randn(5, dim, generator=g)
    out = torch.empty(5, dim)
    o.timestep_embed(t, out)
    assert torch.allclose(out, port.timestep_embedding(t, dim), atol=1e-6)
    ref = _vjp(lambda v: port.timestep_embedding(v, dim), t, cot)
    dt = torch.empty(5)
    o.timestep_embed_bwd(cot, t, dt)
    assert torch.allclose(dt, ref, rtol=1e-4, atol=1e-4)


# ------------------------------------------------------------------------------------------------ 3. engine vs oracle
VJP_VARIANTS = [(0.0, False, 1.0), (0.75, False, 1.0), (0.0, True, 3.0), (0.75, True, 1.0)]


def _compare(name, mask_ratio, t_one, guidance, exact):
    net = vc.build_dit(name, ops_factory=lambda d: vc.VJPEmuOps(d, exact=exact))
    x, t, y, dF = vc.vjp_inputs(name)
    if t_one:
        t = t[:1]
    rows = x.shape[0] * (2 if guidance != 1.0 else 1)
    noise = vc.mask_noise(rows, _grid(name) ** 2) if mask_ratio > 0 else None
    F, dx, dt, dy, grads = vc.product_vjp(net, x, t, y, dF, mask_ratio, guidance)
    oF, odx, odt, ody, ograds = vc.port_vjp(name, x, t, y, dF, mask_ratio, noise, guidance)
    assert dt.shape == t.shape and dy.shape == y.shape and dx.shape == x.shape
    assert set(grads) == set(ograds)
    errs, med, worst = pc.grad_report(grads, ograds)
    return rel(F, oF), {"dx": rel(dx, odx), "dt": rel(dt, odt), "dy": rel(dy, ody)}, errs, med, worst


@pytest.mark.parametrize("mask_ratio,t_one,guidance", VJP_VARIANTS)
@pytest.mark.parametrize("name", CASES)
def test_engine_vjp_exact_matches_oracle(name, mask_ratio, t_one, guidance):
    fe, ie, errs, med, worst = _compare(name, mask_ratio, t_one, guidance, exact=True)
    assert fe < 1e-5
    assert max(ie.values()) < 1e-4, ie
    assert worst < 1e-4, errs[:5]


@pytest.mark.parametrize("name", CASES)
def test_engine_vjp_bf16_rounding_within_reference_amp_class(name):
    """bf16 rounding points of the kernels vs the fp32 oracle, against the reference's own amp-bf16 deviation from its
    fp32 VJP on the same case (stored with the fixture)."""
    mask_ratio = max(vc.VJP_MASKS[name])
    amp = torch.load(os.path.join(pc.GOLDEN, f"vjp_{name}.pt"), weights_only=False)["cases"][mask_ratio]["ref_amp_bf16"]
    fe, ie, errs, med, worst = _compare(name, mask_ratio, False, 1.0, exact=False)
    assert fe < 2 * amp["F"] + 2e-2
    for k, e in ie.items():
        assert e < 2 * amp[k] + 2e-2, (k, e, amp[k])
    assert med < 1.5 * amp["grad_rel_median"] + 5e-3, (med, amp["grad_rel_median"])
    assert worst < 2 * amp["grad_rel_max"] + 2e-2, errs[:5]


# ------------------------------------------------------------------------------------------------ 4. model_forward_wrapper
def _ld(name, exact=True):
    from micro_diffusion_b200.models.model import LatentDiffusion, PrecomputedLatentStubs
    c = configs.PARITY_CONFIGS[name]
    net = vc.build_dit(name, ops_factory=lambda d: vc.VJPEmuOps(d, exact=exact))
    return LatentDiffusion(net, *PrecomputedLatentStubs.make(), p_mean=c["p_mean"], p_std=c["p_std"],
                           latent_res=c["ctor"]["input_size"])


@pytest.mark.parametrize("name,guidance", [("P", 1.0), ("S", 1.0), ("P", 3.0)])
def test_model_forward_wrapper_is_differentiable(name, guidance):
    ld = _ld(name)
    x, t, y, dF = vc.vjp_inputs(name)
    sigma = (4 * t).exp()
    xs, sg, yy = (v.clone().requires_grad_(True) for v in (2 * x, sigma, y))
    fn = partial(ld.dit.forward, cfg=guidance) if guidance != 1.0 else ld.dit
    out = ld.model_forward_wrapper(xs, sg, yy, fn, mask_ratio=0.0)["sample"]
    (out * dF).sum().backward()
    grads = {k: p.grad.detach().clone() for k, p in ld.dit.named_parameters()}
    # oracle: port.denoise (model.py:144-179) under autograd
    c = configs.PARITY_CONFIGS[name]
    sd = port_sd = vc.weights.synth_state_dict(vc.template(name), seed=pc.WEIGHT_SEED)
    P = {k: v.clone().requires_grad_(k not in ("pos_embed", "mask_token")) for k, v in sd.items()}
    ox, osg, oy = (v.clone().requires_grad_(True) for v in (2 * x, sigma, y))
    pcfg = pc.port_config(c, c["ctor"])
    if guidance == 1.0:
        ref = port.denoise(P, pcfg, ox, osg, oy)["sample"]
    else:
        c_skip, c_out, c_in, c_noise = port.edm_precondition(pcfg, osg.view(-1, 1, 1, 1))
        xin = c_in * ox
        o2 = port.dit_forward(P, pcfg, torch.cat([xin, xin]), torch.cat([c_noise.flatten()] * 2),
                              torch.cat([oy, torch.zeros_like(oy)]))["sample"]
        cond, unc = torch.split(o2, x.shape[0])
        ref = c_skip * ox + c_out * (unc + guidance * (cond - unc))
    (ref * dF).sum().backward()
    assert rel(out.detach(), ref.detach()) < 1e-5
    assert rel(xs.grad, ox.grad) < 1e-4 and rel(sg.grad, osg.grad) < 1e-4 and rel(yy.grad, oy.grad) < 1e-4
    errs, med, worst = pc.grad_report(grads, {k: v.grad for k, v in P.items() if v.grad is not None})
    assert worst < 1e-4, errs[:5]
    del port_sd


def test_model_forward_wrapper_without_grad_takes_the_fused_path():
    ld = _ld("P")
    x, t, y, _ = vc.vjp_inputs("P")
    eng = ld.dit.engine
    calls = []
    orig = eng.denoise
    eng.denoise = lambda *a, **k: (calls.append(k), orig(*a, **k))[1]
    with torch.no_grad():
        out = ld.model_forward_wrapper(x.requires_grad_(True), (4 * t).exp(), y, ld.dit, mask_ratio=0.0)
    assert out["sample"].grad_fn is None and not out["sample"].requires_grad and len(calls) == 1
    # with grad mode on but nothing requiring grad, the fused path is kept too
    ld.dit.requires_grad_(False)
    out = ld.model_forward_wrapper(x.detach(), (4 * t).exp(), y, ld.dit, mask_ratio=0.0)
    assert out["sample"].grad_fn is None and len(calls) == 2


# ------------------------------------------------------------------------------------------------ 5. semantics
def test_gradients_accumulate_across_live_forwards_and_zero_grad():
    net = vc.build_dit("P", ops_factory=lambda d: vc.VJPEmuOps(d, exact=True))
    x, t, y, dF = vc.vjp_inputs("P")
    _, dx1, _, _, g1 = vc.product_vjp(net, x, t, y, dF)
    net.zero_grad(set_to_none=True)
    xr = x.clone().requires_grad_(True)
    outs = [net(xr, t, y)["sample"] for _ in range(2)]  # two live contexts before any backward
    for o in outs:
        (o * dF).sum().backward()
    for k, p in net.named_parameters():
        assert torch.allclose(p.grad, 2 * g1[k], rtol=1e-5, atol=1e-7), k
        assert p.grad.data_ptr() == net.store.g[k].data_ptr()
    assert torch.allclose(xr.grad, 2 * dx1, rtol=1e-5, atol=1e-7)
    net.zero_grad(set_to_none=True)
    assert all(p.grad is None for p in net.parameters())
    (net(x, t, y)["sample"] * dF).sum().backward()  # re-attached and zeroed, not stale
    for k, p in net.named_parameters():
        assert torch.allclose(p.grad, g1[k], rtol=1e-5, atol=1e-7), k


def test_second_backward_raises():
    net = vc.build_dit("P", ops_factory=lambda d: vc.VJPEmuOps(d, exact=True))
    x, t, y, dF = vc.vjp_inputs("P")
    loss = (net(x.requires_grad_(True), t, y)["sample"] * dF).sum()
    loss.backward(retain_graph=True)
    with pytest.raises(RuntimeError, match="backward called twice"):
        loss.backward()


def test_mixed_freezing_raises():
    net = vc.build_dit("P", ops_factory=lambda d: vc.VJPEmuOps(d, exact=True))
    x, t, y, _ = vc.vjp_inputs("P")
    net.blocks[0].requires_grad_(False)
    with pytest.raises(NotImplementedError, match="all of them, or on none"):
        net(x, t, y)
    with torch.no_grad():  # inference does not care
        net(x, t, y)


@pytest.mark.parametrize("mask_ratio", [0.0, 0.75])
def test_all_frozen_gives_the_same_input_gradients_with_fewer_gemms(mask_ratio):
    net = vc.build_dit("S", ops_factory=lambda d: vc.VJPEmuOps(d, exact=False))
    x, t, y, dF = vc.vjp_inputs("S")
    ops = net.engine.ops
    net(x, t, y)  # warm the weight copies
    runs = {}
    for frozen in (False, True):
        g0, l0 = ops.gemm_launches, ops.launches
        flat0 = net.store.grad.clone()
        F, dx, dt, dy, grads = vc.product_vjp(net, x, t, y, dF, mask_ratio, frozen=frozen)
        runs[frozen] = (F, dx, dt, dy, ops.gemm_launches - g0, ops.launches - l0)
        if frozen:
            assert not grads and all(p.grad is None for p in net.parameters())
            assert torch.equal(net.store.grad, flat0)  # the flat gradient buffer is not written
    for i in range(4):
        assert torch.equal(runs[False][i], runs[True][i]), i
    assert runs[True][4] < runs[False][4] and runs[True][5] < runs[False][5], (runs[True][4:], runs[False][4:])
    # input gradients of x only: the conditioning stem's backward is skipped altogether
    net.requires_grad_(False)
    g0 = ops.gemm_launches
    xr = x.clone().requires_grad_(True)
    torch.manual_seed(vc.MASK_SEED)
    (net(xr, t, y, mask_ratio=mask_ratio)["sample"] * dF).sum().backward()
    assert torch.equal(xr.grad, runs[True][1]) and ops.gemm_launches - g0 < runs[True][4]


def test_forward_without_grad_saves_nothing():
    net = vc.build_dit("P", ops_factory=lambda d: vc.VJPEmuOps(d, exact=True))
    x, t, y, _ = vc.vjp_inputs("P")
    seen = []
    orig = net.engine.forward_raw
    net.engine.forward_raw = lambda *a, **k: (seen.append(k.get("keep", False)), orig(*a, **k))[1]
    with torch.no_grad():
        out = net(x.requires_grad_(True), t, y)
    assert out["sample"].grad_fn is None and seen == [False]


# ------------------------------------------------------------------------------------------------ 6. loss path unchanged
@pytest.mark.parametrize("name", ["P", "S"])
def test_fused_loss_path_issues_the_same_op_sequence(name):
    ref = json.load(open(os.path.join(pc.GOLDEN, "loss_path_ops.json")))[name]
    got = vc.record_loss_path(name)
    for part in ("forward", "backward"):
        a, b = got[part], ref[part]
        first = next((i for i, (u, v) in enumerate(zip(a, b)) if u != v), min(len(a), len(b)))
        assert a == b, (part, len(a), len(b), first, a[first:first + 2], b[first:first + 2])


def test_emu_ops_used_here_are_the_stock_contracts():
    """The adjoint contracts extend EmuOps without changing any of its ops."""
    for k, v in vars(EmuOps).items():
        if callable(v) and not k.startswith("_") and k != "gemm":
            assert getattr(vc.VJPEmuOps, k) is v, k
