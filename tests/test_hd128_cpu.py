"""head_dim=128 on CPU, with the kernels replaced by their CPU contracts (oracle.emu_ops): the oracle against the unmodified
reference (tests/golden/hd128_*.pt), the engine's loss path, VJP and frozen VJP against the oracle, and the state_dict of
DiT(head_dim=128) at the reference's default widths."""
import pytest
import torch

from micro_diffusion_b200.arch import DiTConfig
from tests import dit_vjp_common as vc
from tests import hd128_common as hc
from tests import parity_common as pc

CASES = list(hc.HD128_CONFIGS)
VJP_CASES = [(n, mr) for n in CASES for mr in hc.VJP_MASKS[n]]
rel = pc.rel_l2


def _exact(d):
    return hc.Emu(d, exact=True)


def _bf16(d):
    return hc.Emu(d, exact=False)


@pytest.mark.parametrize("name", CASES)
def test_configs_have_128_wide_heads_and_several_head_counts(name):
    cfg = DiTConfig(**hc.HD128_CONFIGS[name]["ctor"])
    blocks = cfg.all_blocks()
    assert all(b.attn_dim == 128 * b.heads and b.dim == 128 * b.xheads for b in blocks)
    if name == "HS":
        assert len({b.heads for b in blocks}) >= 3


@pytest.mark.parametrize("name", CASES)
def test_state_dict_matches_reference(name):
    fx = hc.golden(name)
    net = hc.build_dit(name, ops_factory=_exact)
    assert [(k, tuple(v.shape)) for k, v in net.state_dict().items()] == [(k, tuple(s)) for k, s in fx["keys"]]


def test_default_dit_with_128_wide_heads_has_the_reference_state_dict():
    """DiT(head_dim=128) with every other argument at its default -- from the architecture arithmetic alone."""
    keys = hc.golden("H")["default_dit_keys"]
    cfg = DiTConfig(head_dim=128)
    got = [(k, tuple(s)) for k, s in cfg.buffer_specs() + cfg.param_specs()]
    assert sorted(got) == sorted((k, tuple(s)) for k, s in keys)
    assert len(keys) == 671
    assert {b.heads for b in cfg.blocks} == {9} and {b.heads for b in cfg.mixer_blocks} == {4}


@pytest.mark.parametrize("name", CASES)
def test_port_matches_reference_fixture(name):
    fx = hc.golden(name)
    loss, grads, den = hc.oracle_run(name)
    assert abs(loss - fx["loss"]) / fx["loss"] < 1e-6
    assert rel(den, fx["denoised_unmasked"]) < 1e-5
    assert set(grads) == set(fx["grads"])
    errs = sorted((vc.fingerprint_error(k, grads[k], fp), k) for k, fp in fx["grads"].items())
    assert errs[-1][0] < 1e-4, errs[-3:]
    for mr, v in fx["vjp"].items():
        x, t, y, dF, noise = hc.vjp_case(name, mr)
        F, dx, dt, dy, vgrads = hc.port_vjp(name, x, t, y, dF, mr, noise)
        assert rel(F, v["F"]) < 1e-5 and rel(dx, v["dx"]) < 1e-5 and rel(dt, v["dt"]) < 1e-5, mr
        assert vc.fingerprint_error("dy", dy, v["dy"]) < 1e-5
        errs = sorted((vc.fingerprint_error(k, vgrads[k], fp), k) for k, fp in v["grads"].items())
        assert errs[-1][0] < 1e-5, (mr, errs[-3:])


@pytest.mark.parametrize("name", CASES)
def test_engine_exact_matches_oracle(name):
    loss, grads, den, _ = hc.product_run(name, ops_factory=_exact)
    oloss, ograds, oden = hc.oracle_run(name)
    assert abs(loss - oloss) / oloss < 1e-6
    assert rel(den, oden) < 1e-5
    assert set(grads) == set(ograds)
    errs, med, worst = pc.grad_report(grads, ograds)
    assert med < 2e-6 and worst < 5e-5, errs[:5]


@pytest.mark.parametrize("name", CASES)
def test_engine_bf16_rounding_within_reference_amp_class(name):
    fx = hc.golden(name)
    loss, grads, den, _ = hc.product_run(name, ops_factory=_bf16)
    oloss, ograds, oden = hc.oracle_run(name)
    assert abs(loss - oloss) / oloss < 3e-3
    assert rel(den, oden) < max(1e-2, max(v["ref_amp_bf16"]["F"] for v in fx["vjp"].values()))
    errs, med, worst = pc.grad_report(grads, ograds)
    assert med < 1.5 * fx["ref_amp_bf16_grad_rel_median"] + 5e-3, (med, fx["ref_amp_bf16_grad_rel_median"])
    assert worst < 2 * fx["ref_amp_bf16_grad_rel_max"] + 2e-2, errs[:5]


@pytest.mark.parametrize("name,mr", VJP_CASES)
def test_engine_vjp_exact_matches_oracle(name, mr):
    net = hc.build_dit(name, ops_factory=_exact)
    x, t, y, dF, noise = hc.vjp_case(name, mr)
    F, dx, dt, dy, grads = vc.product_vjp(net, x, t, y, dF, mr)
    oF, odx, odt, ody, ograds = hc.port_vjp(name, x, t, y, dF, mr, noise)
    assert rel(F, oF) < 1e-5
    assert rel(dx, odx) < 1e-4 and rel(dt, odt) < 1e-4 and rel(dy, ody) < 1e-4
    assert set(grads) == set(ograds)
    errs, med, worst = pc.grad_report(grads, ograds)
    assert worst < 1e-4, errs[:5]


@pytest.mark.parametrize("name", CASES)
def test_frozen_vjp_gives_the_same_input_gradients_and_leaves_the_buffer_alone(name):
    net = hc.build_dit(name, ops_factory=_bf16)
    mr = hc.VJP_MASKS[name][-1]
    x, t, y, dF, _ = hc.vjp_case(name, mr)
    ops = net.engine.ops
    runs = {}
    for frozen in (False, True):
        flat0 = net.store.grad.clone()
        l0 = ops.launches
        F, dx, dt, dy, grads = vc.product_vjp(net, x, t, y, dF, mr, frozen=frozen)
        runs[frozen] = (F, dx, dt, dy, ops.launches - l0)
        if frozen:
            assert not grads and torch.equal(net.store.grad, flat0)
    for i in range(4):
        assert torch.equal(runs[False][i], runs[True][i]), i
    assert runs[True][4] < runs[False][4]
