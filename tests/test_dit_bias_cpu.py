"""use_bias=True (the reference DiT's default) on CPU, with the kernels replaced by their CPU contracts (oracle.emu_ops plus
the bias contracts of tests/bias_common.py): state_dict and parameter layout, init, the engine's loss path and VJP against
the oracle, the oracle against the unmodified reference (tests/golden/bias_*.pt), and the two-rank gradient exchange."""
import hashlib
import json
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from micro_diffusion_b200.arch import DiTConfig, micro_dit_tiny_2_kwargs, micro_dit_xl_2_kwargs
from micro_diffusion_b200.params import ParamLayout, ParamStore
from oracle import weights
from oracle.configs import PARITY_CONFIGS
from oracle.emu_ops import EPI_SWIGLU, EmuOps, interleave_perm
from tests import bias_common as bc
from tests import dit_vjp_common as vc
from tests import parity_common as pc

CASES = list(bc.BIAS_CONFIGS)
rel = pc.rel_l2


def _exact(d):
    return bc.BiasEmuOps(d, exact=True)


def _bf16(d):
    return bc.BiasEmuOps(d, exact=False)


def _bias_names(ct):
    """Parameters use_bias=True adds to a config."""
    off = DiTConfig(**{**ct, "use_bias": False}).param_specs()
    return [n for n, _ in DiTConfig(**{**ct, "use_bias": True}).param_specs() if n not in dict(off)]


# ------------------------------------------------------------------------------------------------ 1. state dict
@pytest.mark.parametrize("name", CASES)
def test_state_dict_matches_reference(name):
    fx = bc.golden(name)
    net = bc.build_dit(name, ops_factory=_exact)
    sd = net.state_dict()
    assert [(k, tuple(v.shape)) for k, v in sd.items()] == [(k, tuple(s)) for k, s in fx["keys"]]
    ref = weights.synth_state_dict(sd, seed=3)
    ordered = {k: ref[k] for k, _ in fx["keys"]}  # the reference's own order
    net.load_state_dict(ordered)
    for k, v in net.state_dict().items():
        assert torch.equal(v, ordered[k]), k


def test_default_dit_state_dict_matches_reference():
    """DiT() with every default argument (dim 1152, depth 28, mixer 4 x 512 with biased maps) -- from the architecture
    arithmetic alone: the full-size model is not built here."""
    keys = json.load(open(bc.DEFAULT_KEYS))
    cfg = DiTConfig()
    assert cfg.use_bias
    assert [[k, list(s)] for k, s in cfg.buffer_specs() + cfg.param_specs()] == keys
    lay = ParamLayout(cfg)
    assert set(lay.slots) == {k for k, _ in keys[2:]}


# ------------------------------------------------------------------------------------------------ 2. layout
# (total, back_start, kv_back, sha256 of the sorted slots) of the bias-free layouts, from the rules before biases existed
BIAS_FREE_LAYOUTS = {
    "P": (2503680, 1910784, (495616, 561152), "828e0943e9b2233c"),
    "S": (10303488, 6361088, (2450432, 2974720), "abc2b267a95b9b88"),
    "S16": (1555456, 1153024, (347136, 412672), "960e9ca077e4edf6"),
    "Tiny_2": (200693760, 92365824, (34141184, 42529792), "6acc57c676a244dd"),
    "XL_2": (1165444096, 442240000, (213849088, 272569344), "a9c08510d0a8355b"),
}


def _bias_free_ctor(name):
    if name == "Tiny_2":
        return micro_dit_tiny_2_kwargs()
    if name == "XL_2":
        return micro_dit_xl_2_kwargs()
    return PARITY_CONFIGS[name]["ctor"]


@pytest.mark.parametrize("name", list(BIAS_FREE_LAYOUTS))
def test_bias_free_layout_is_unchanged(name):
    lay = ParamLayout(DiTConfig(**_bias_free_ctor(name)))
    digest = hashlib.sha256(repr(sorted(lay.slots.items())).encode()).hexdigest()[:16]
    assert (lay.total, lay.back_start, lay.kv_back, digest) == BIAS_FREE_LAYOUTS[name]
    assert not lay.bias
    g = lay.groups["kv.blocks"]  # the early exchange range is exactly the stacked backbone K/V weight, as before
    assert lay.kv_back == (g.offset, g.offset + g.numel)


def _reducer(lay):
    from micro_diffusion_b200.train_step import GradReducer
    return GradReducer(ParamStore(lay, "cpu", torch.float32), shard=False)


@pytest.mark.parametrize("name", CASES + ["DiT()"])
def test_bias_layout_keeps_the_stacks_and_the_exchange_ranges(name):
    cfg = DiTConfig() if name == "DiT()" else DiTConfig(**bc.BIAS_CONFIGS[name]["ctor"])
    lay = ParamLayout(cfg)
    ra = lay.RANGE_ALIGN
    assert lay.total % ra == 0 and lay.back_start % ra == 0 and lay.kv_back[0] % ra == 0 and lay.kv_back[1] % ra == 0
    # w1 | w2 weight stack and [b1 | b2] bias stack of every SwiGLU
    for b in [*cfg.all_blocks(), None]:
        pre = "y_emb_preprocess.mlp." if b is None else b.name + ".mlp."
        if b is not None and b.moe:
            continue
        f = lay.slots[pre + "w1.bias"][1][0]
        assert lay.slots[pre + "w2.weight"][0] == lay.slots[pre + "w1.weight"][0] + f * lay.slots[pre + "w1.weight"][1][1]
        assert lay.bias[pre + "w12"] == (lay.slots[pre + "w1.bias"][0], 2 * f)
        assert lay.slots[pre + "w2.bias"][0] == lay.slots[pre + "w1.bias"][0] + f
    # stage-wide K/V bias stacks: every block's [2D] kv_linear bias in block order, contiguous
    for stage, blocks in (("kv.patch_mixer", cfg.mixer_blocks), ("kv.blocks", cfg.blocks)):
        o, n = lay.bias[stage]
        assert n == sum(2 * b.dim for b in blocks)
        for b in blocks:
            assert lay.slots[b.name + ".cross_attn.kv_linear.bias"][0] == o
            o += 2 * b.dim
    # the backbone K/V bias stack belongs to the "back" range, the mixer's does not
    o, n = lay.bias["kv.blocks"]
    assert lay.kv_back[0] <= o and o + n <= lay.kv_back[1]
    st = ParamStore(lay, "cpu", torch.float32)
    assert st.is_back(o) and not st.is_back(lay.bias["kv.patch_mixer"][0])
    if name == "DiT()":
        return
    red = _reducer(lay)
    assert any(a <= o and o + n <= b for a, b in red.early)
    assert all(a % ra == 0 and b % ra == 0 for a, b in red.early + red.late)
    # every early range is final once the backbone backward is done: no stem / mixer tensor inside
    for nm, (off, shape) in lay.slots.items():
        inside = any(a <= off < b for a, b in red.early)
        assert inside == (st.is_back(off)), nm


# ------------------------------------------------------------------------------------------------ 3. init
def test_init_zeroes_every_bias_and_the_output():
    ct = bc.BIAS_CONFIGS["SB"]["ctor"]
    from micro_diffusion_b200.models.dit import DiT
    net = DiT(**ct, ops_factory=_exact)
    P = dict(net.named_parameters())
    names = _bias_names(ct)
    assert len(names) > 0
    for n in names:
        assert torch.count_nonzero(P[n]) == 0, n
    x, t, y, _ = vc.vjp_inputs("S")
    with torch.no_grad():
        out = net(x, t, y)["sample"]
    assert torch.count_nonzero(out) == 0


# ------------------------------------------------------------------------------------------------ 4. CPU contracts
def test_swiglu_bias_contract_maps_the_natural_order_onto_the_interleaved_columns():
    o = bc.BiasEmuOps(exact=True)
    g = torch.Generator().manual_seed(4)
    M, K, f = 5, 16, 96
    x, w, b = torch.randn(M, K, generator=g), torch.randn(2 * f, K, generator=g), torch.randn(2 * f, generator=g)
    perm = interleave_perm(f)
    u, h = torch.empty(M, 2 * f), torch.empty(M, f)
    o.gemm(x, w[perm], u, epi=EPI_SWIGLU, C2=h, bias=b)
    un = x @ w.t() + b  # natural order
    assert torch.allclose(u, un[:, perm], atol=1e-5)
    assert torch.allclose(h, torch.nn.functional.silu(un[:, :f]) * un[:, f:], atol=1e-5)
    out = torch.full((2 * f,), 0.5)
    o.colsum_interleaved(u, out, f)
    assert torch.allclose(out, 0.5 + un.sum(0), atol=1e-4)


def test_bias_contracts_extend_the_stock_ones():
    for k, v in vars(EmuOps).items():
        if callable(v) and not k.startswith("_") and k != "gemm":
            assert getattr(bc.BiasEmuOps, k) is v, k


# ------------------------------------------------------------------------------------------------ 5. oracle vs reference
@pytest.mark.parametrize("name", CASES)
def test_port_matches_reference_fixture(name):
    fx = bc.golden(name)
    loss, grads, den = bc.oracle_run(name)
    assert abs(loss - fx["loss"]) / fx["loss"] < 1e-6
    assert rel(den, fx["denoised_unmasked"]) < 1e-5
    assert set(grads) == set(fx["grads"])
    errs = sorted((vc.fingerprint_error(k, grads[k], fp), k) for k, fp in fx["grads"].items())
    assert errs[-1][0] < 1e-4, errs[-3:]
    for k, g in fx["grad_full"].items():
        assert rel(grads[k], g) < 1e-4, k
    v = fx["vjp"]
    x, t, y, dF, mr, noise = bc.vjp_case(name)
    F, dx, dt, dy, vgrads = bc.port_vjp(name, x, t, y, dF, mr, noise)
    assert rel(F, v["F"]) < 1e-5 and rel(dx, v["dx"]) < 1e-5 and rel(dt, v["dt"]) < 1e-5
    assert vc.fingerprint_error("dy", dy, v["dy"]) < 1e-5
    errs = sorted((vc.fingerprint_error(k, vgrads[k], fp), k) for k, fp in v["grads"].items())
    assert errs[-1][0] < 1e-5, errs[-3:]


# ------------------------------------------------------------------------------------------------ 6. engine vs oracle
@pytest.mark.parametrize("name", CASES)
def test_engine_exact_matches_oracle(name):
    loss, grads, den, ld = bc.product_run(name, ops_factory=_exact)
    oloss, ograds, oden = bc.oracle_run(name)
    assert abs(loss - oloss) / oloss < 1e-6
    assert rel(den, oden) < 1e-5
    assert set(grads) == set(ograds)
    errs, med, worst = pc.grad_report(grads, ograds)
    # fp32 reassociation: the cross-attention query path (norm2, q_linear weight and bias) of S16 sits at ~1e-5 with or
    # without biases (the bias-free S16 shows 7e-6 there); everything else is at 1e-6
    assert med < 2e-6 and worst < 5e-5, errs[:5]


@pytest.mark.parametrize("name", CASES)
def test_engine_bf16_rounding_within_reference_amp_class(name):
    """bf16 rounding points and the interleaved w1 | w2 stacks of the fused SwiGLU (biased epilogue, interleaved bias
    column sums) against the fp32 oracle, within the reference's own amp-bf16 deviation on the same case."""
    fx = bc.golden(name)
    loss, grads, den, ld = bc.product_run(name, ops_factory=_bf16)
    assert ld.dit.store.interleave
    oloss, ograds, oden = bc.oracle_run(name)
    assert abs(loss - oloss) / oloss < 3e-3
    # D_x: SB lands at 1.1e-2 (identical with MD_FUSE_SWIGLU=0); the reference's own amp-bf16 output deviates 1.5e-2
    assert rel(den, oden) < max(1e-2, fx["vjp"]["ref_amp_bf16"]["F"])
    errs, med, worst = pc.grad_report(grads, ograds)
    assert med < 1.5 * fx["ref_amp_bf16_grad_rel_median"] + 5e-3, (med, fx["ref_amp_bf16_grad_rel_median"])
    assert worst < 2 * fx["ref_amp_bf16_grad_rel_max"] + 2e-2, errs[:5]


def test_prompt_cache_applies_the_kv_bias_before_the_row_norm():
    ld = bc.build_product("SB", ops_factory=_exact)
    ld.eval()
    eng = ld.dit.engine
    cap = torch.randn(2, 1, 77, 1024).half()
    x, sg = torch.randn(2, 4, 16, 16), torch.full((2,), 1.5)
    d0, _, _ = eng.denoise(x, sg, cap, edm=ld._edm_scalars(), prompt=eng.prompt_cache(cap))
    d1, _, _ = eng.denoise(x, sg, cap, edm=ld._edm_scalars())
    assert rel(d0, d1) < 1e-6


# ------------------------------------------------------------------------------------------------ 7. VJP
@pytest.mark.parametrize("name", CASES)
def test_engine_vjp_exact_matches_oracle(name):
    net = bc.build_dit(name, ops_factory=_exact)
    x, t, y, dF, mr, noise = bc.vjp_case(name)
    F, dx, dt, dy, grads = vc.product_vjp(net, x, t, y, dF, mr)
    oF, odx, odt, ody, ograds = bc.port_vjp(name, x, t, y, dF, mr, noise)
    assert rel(F, oF) < 1e-5
    assert rel(dx, odx) < 1e-4 and rel(dt, odt) < 1e-4 and rel(dy, ody) < 1e-4
    assert set(grads) == set(ograds)
    errs, med, worst = pc.grad_report(grads, ograds)
    assert worst < 1e-4, errs[:5]


def test_all_frozen_vjp_gives_the_same_input_gradients_and_leaves_the_buffer_alone():
    net = bc.build_dit("SB", ops_factory=_bf16)
    x, t, y, dF, mr, _ = bc.vjp_case("SB")
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


# ------------------------------------------------------------------------------------------------ 8. two ranks
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, out_path, shard):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.set_num_threads(2)
    from micro_diffusion_b200.train_step import FlatAdamW, GradReducer
    ld = bc.build_product("PB", ops_factory=_exact)
    opt = FlatAdamW(ld.dit, lr=1e-3, clip_norm=0.25, eps=1e-2)
    red = GradReducer(ld.dit.store, buckets=3, shard=shard)
    assert red.shard == shard
    full = weights.synth_batch(4, 4, 32, seed=5)
    mine = {k: v[rank * 2:(rank + 1) * 2].clone() for k, v in full.items()}
    torch.manual_seed(100 + rank)
    eng = ld.dit.engine
    loss = ld(mine)[0]
    eng.on_backbone_grads_ready = red.reduce_early
    loss.backward()
    eng.on_backbone_grads_ready = None
    red.reduce()
    g = ld.dit.store.grad.clone()
    opt.step(None, red)
    ld.dit.store.refresh_copies(eng.ops, None, force=True)
    opt.gather_state()
    torch.save({"grad": g, "flat": ld.dit.store.flat.clone(), "owned": red.owned}, out_path + f".{rank}")
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("shard", [False, True])
def test_two_rank_step_matches_single_process(tmp_path, shard):
    out = str(tmp_path / "rank.pt")
    mp.start_processes(_worker, args=(2, _free_port(), out, shard), nprocs=2, join=True, start_method="spawn")
    got, got1 = torch.load(out + ".0"), torch.load(out + ".1")
    if shard:
        cover = torch.zeros_like(got["grad"], dtype=torch.int32)
        merged = torch.zeros_like(got["grad"])
        for r in (got, got1):
            for a, b in r["owned"]:
                cover[a:b] += 1
                merged[a:b] = r["grad"][a:b]
        assert int(cover.min()) == 1 and int(cover.max()) == 1
        got["grad"] = merged
    assert torch.equal(got["flat"], got1["flat"])
    from micro_diffusion_b200.train_step import FlatAdamW
    ld = bc.build_product("PB", ops_factory=_exact)
    opt = FlatAdamW(ld.dit, lr=1e-3, clip_norm=0.25, eps=1e-2)
    full = weights.synth_batch(4, 4, 32, seed=5)
    for r in range(2):
        torch.manual_seed(100 + r)
        (0.5 * ld({k: v[r * 2:(r + 1) * 2].clone() for k, v in full.items()})[0]).backward()
    g = ld.dit.store.grad.clone()
    opt.step()
    kv = ld.dit.store.layout.bias["kv.blocks"]
    assert float(g[kv[0]:kv[0] + kv[1]].abs().max()) > 0  # the backbone K/V bias stack is trained and exchanged
    assert torch.allclose(got["grad"], g, rtol=1e-4, atol=1e-7)
    assert torch.allclose(got["flat"], ld.dit.store.flat, rtol=1e-5, atol=1e-6)
