"""The CUDA-graph Heun sampler (engine.SamplerGraph) on the GPU: bit-identical to the eager loop (final latents and the D
of every denoiser call), the same random numbers, the eager loop wherever the graph path is not eligible, reuse and
invalidation of the captured graphs, no host sync while replaying, and the two new kernels against the torch expressions
they replace."""
import contextlib
import os

import pytest
import torch

from micro_diffusion_b200 import engine as engine_mod
from micro_diffusion_b200._lib import MicroditLibraryError
from micro_diffusion_b200.models.model import LatentDiffusion, PrecomputedLatentStubs
from tests import hd128_common as hc
from tests import parity_common as pc

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
CHURN = dict(S_churn=40, S_min=0.1, S_max=10)  # 5 steps (t ~ 80, 17.5, 2.5, 0.17, 0.002): gamma off, off, on, on, off


def _same(a, b):
    """Bit-identical, NaN where the other is NaN (one Heun step divides 0 by 0 in the schedule, in both paths)."""
    if a.shape != b.shape or a.dtype != b.dtype or not torch.equal(a.isnan(), b.isnan()):
        return False
    return torch.equal(torch.where(a.isnan(), 0, a), torch.where(b.isnan(), 0, b))


def _runs(ld):
    return sum(g.runs for g in ld.dit.engine._sampler_graphs.values())


def _sample(ld, x, y, steps, cfg, graph, seed=1234):
    """(latents, [D of every call]) of one seeded edm_sampler_loop, on the graph path or the eager loop."""
    calls = []
    ld.sampler_graph, ld.sampler_debug = graph, (lambda k, j, d: calls.append((k, j, d.detach().clone())))
    try:
        torch.manual_seed(seed)
        out = ld.edm_sampler_loop(x, y, steps=steps, cfg=cfg)
    finally:
        ld.sampler_graph, ld.sampler_debug = True, None
    return out, calls


def _check_identical(ld, x, y, steps, cfg):
    before = _runs(ld)
    g_out, g_calls = _sample(ld, x, y, steps, cfg, True)
    assert _runs(ld) == before + 1, "the graph path did not run"
    e_out, e_calls = _sample(ld, x, y, steps, cfg, False)
    assert _runs(ld) == before + 1
    assert [c[:2] for c in g_calls] == [c[:2] for c in e_calls] and len(e_calls) == 2 * steps - 1
    for (k, j, a), (_, _, b) in zip(g_calls, e_calls):
        assert _same(a, b), f"D of step {k} call {j} differs"
    assert _same(g_out, e_out)
    return g_out


def _inputs(ld, B, seed=0):
    net = ld.dit
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(B, net.in_channels, net.input_size, net.input_size, device=DEV, generator=g)
    y = torch.randn(B, 1, 77, net.cfg.caption_channels, device=DEV, generator=g).half()
    return x, y


def _small(name, ops_factory=None):
    ld = hc.build_product(name, ops_factory, device=DEV) if name == "H" else pc.build_product(name, ops_factory, device=DEV)
    ld.eval()
    return ld


def _xl2(latent, scale):
    from micro_diffusion_b200.models.dit import MicroDiT_XL_2
    from oracle import weights
    net = MicroDiT_XL_2(input_size=latent, in_channels=4, pos_interp_scale=scale)
    net.load_state_dict(weights.synth_state_dict(net.state_dict(), seed=7))
    vae, te, tok = PrecomputedLatentStubs.make()
    ld = LatentDiffusion(net.to(DEV), vae, te, tok, latent_res=latent)
    ld.eval()
    return ld


@pytest.fixture(scope="module")
def small_models():
    models = {}
    yield lambda name: models.setdefault(name, _small(name))
    models.clear()


@pytest.mark.parametrize("steps,churn", [(1, False), (2, False), (5, False), (5, True)])
@pytest.mark.parametrize("cfg", [1.0, 5.0])
@pytest.mark.parametrize("name", ["P", "S", "S16", "H"])
def test_graph_sampler_is_bit_identical(small_models, name, cfg, steps, churn):
    ld = small_models(name)
    ld.edm_config.update(S_churn=0, S_min=0, S_max=float("inf"))
    if churn:
        ld.edm_config.update(CHURN)
    x, y = _inputs(ld, 3)
    _check_identical(ld, x, y, steps, cfg)


@pytest.mark.parametrize("latent,scale,B", [(32, 1.0, 2), (64, 2.0, 1)])
def test_graph_sampler_is_bit_identical_xl2(latent, scale, B):
    ld = _xl2(latent, scale)
    ld.edm_config.update(CHURN)
    x, y = _inputs(ld, B)
    _check_identical(ld, x, y, 3, 5.0)
    _check_identical(ld, x, y, 2, 1.0)


@pytest.mark.parametrize("mode", ["high", "deterministic"])
def test_graph_sampler_is_bit_identical_in_other_modes(mode):
    from micro_diffusion_b200.ops import CudaOps
    if mode == "high":
        ld = _small("S", ops_factory=lambda d: CudaOps(d, precision="high"))
        assert ld.dit.engine.ops.prec == 1
    else:
        ld = _small("S")
    ld.edm_config.update(CHURN)
    x, y = _inputs(ld, 2)
    ops = ld.dit.engine.ops
    try:
        if mode == "deterministic":
            ops.set_deterministic(True)
        for cfg in (1.0, 5.0):
            _check_identical(ld, x, y, 5, cfg)
    finally:
        if mode == "deterministic":
            ops.set_deterministic(False)


@pytest.mark.parametrize("name", ["P", "S"])
def test_graph_sampler_matches_reference_fixture(name):
    """The graph path against the unmodified reference's fp32 sampler (tests/golden/sampler_*.pt), with the bounds of
    test_parity_gpu.py::test_sampler_matches_reference_fixture."""
    from oracle.make_golden import SAMPLER_STEPS, sampler_inputs
    fx = torch.load(os.path.join(pc.GOLDEN, f"sampler_{name}.pt"), weights_only=False)
    ld = _small(name)
    x, y = sampler_inputs(name)
    for g in (1.0, 3.0):
        before = _runs(ld)
        a = ld.edm_sampler_loop(x.to(DEV), y.half().to(DEV), steps=SAMPLER_STEPS, cfg=g)
        assert _runs(ld) == before + 1
        err = pc.rel_l2(a.cpu(), fx[f"out_cfg{g}"])
        print(f"\n[{name}] graph sampler cfg={g}: rel-L2 vs reference {err:.2e}")
        assert err < 3e-2


class _Text:
    """Text-encoder stand-in for generate(): a fixed function of the token ids."""

    def __init__(self, channels):
        self.channels = channels

    def requires_grad_(self, flag):
        return self

    def encode(self, ids, attention_mask=None):
        g = torch.Generator(device=ids.device).manual_seed(int(ids.sum()))
        return (torch.randn(ids.shape[0], 1, 77, self.channels, device=ids.device, generator=g).half(),)


def test_generate_consumes_the_rng_like_the_eager_loop():
    ld = _small("P")
    ld.text_encoder = _Text(ld.dit.cfg.caption_channels)
    ld.vae.to(DEV)
    ids = torch.arange(3 * 77).reshape(3, 77)
    res = {}
    for graph in (True, False):
        ld.sampler_graph = graph
        calls = []
        ld.randn_like = lambda t: calls.append(1) or torch.randn_like(t)
        torch.manual_seed(77)
        before = _runs(ld)
        lat = ld.generate(tokenized_prompts=ids, guidance_scale=5.0, num_inference_steps=6, seed=3,
                          return_only_latents=True)
        res[graph] = (lat, torch.cuda.get_rng_state(), len(calls), _runs(ld) - before)
    ld.sampler_graph = True
    assert res[True][3] == 1 and res[False][3] == 0
    assert _same(res[True][0], res[False][0])
    assert torch.equal(res[True][1], res[False][1])
    assert res[True][2] == res[False][2] == 6


def test_ineligible_calls_take_the_eager_loop():
    from micro_diffusion_b200.models.dit import DiT
    ld = _small("P")
    x, y = _inputs(ld, 2)

    class Sub(LatentDiffusion):
        def model_forward_wrapper(self, *a, **k):
            return super().model_forward_wrapper(*a, **k)

    @contextlib.contextmanager
    def no_cache():
        ld.cache_prompt = False
        yield
        ld.cache_prompt = True

    @contextlib.contextmanager
    def custom_forward():
        ld.dit.forward = lambda *a, **k: DiT.forward(ld.dit, *a, **k)
        yield
        del ld.dit.forward

    @contextlib.contextmanager
    def subclass():
        ld.__class__ = Sub
        yield
        ld.__class__ = LatentDiffusion

    @contextlib.contextmanager
    def grad_inputs():
        with torch.enable_grad():
            yield

    for case in (no_cache, custom_forward, subclass, grad_inputs):
        for cfg in (1.0, 5.0):
            xin = x.clone().requires_grad_() if case is grad_inputs else x
            before = _runs(ld)
            with case():
                torch.manual_seed(9)
                a = ld.edm_sampler_loop(xin, y, steps=3, cfg=cfg)
                assert _runs(ld) == before, case.__name__
                b, _ = _sample(ld, xin, y, 3, cfg, False, seed=9)
            assert _same(a, b), case.__name__
    before = _runs(ld)
    _sample(ld, x, y, 3, 5.0, False)
    assert _runs(ld) == before


def test_graphs_are_reused_and_follow_the_weights():
    from micro_diffusion_b200.ema import FlatEMA
    from micro_diffusion_b200.train_step import FlatAdamW
    from oracle import weights
    ld = _small("S")
    x, y = _inputs(ld, 2)
    for cfg in (1.0, 5.0):
        _check_identical(ld, x, y, 4, cfg)
    graphs = dict(ld.dit.engine._sampler_graphs)
    assert len(graphs) == 2 and all(g.captures == 1 for g in graphs.values())
    _check_identical(ld, x, y, 4, 5.0)
    _check_identical(ld, x, y, 3, 5.0)  # fewer steps: the same graphs
    assert all(g.captures == 1 for g in graphs.values()) and ld.dit.engine._sampler_graphs == graphs
    # weight updates: FlatAdamW steps (with an EMA), then sampling with the EMA weights swapped in
    opt = FlatAdamW(ld.dit, lr=1e-3)
    ema = FlatEMA(ld.dit, smoothing=0.5, ema_start="1ba")
    ld.train()
    for s in range(2):
        batch = {k: v.to(DEV) for k, v in weights.synth_batch(4, 4, 16, seed=40 + s).items()}
        ld(batch)[0].backward()
        opt.step(None, None, ema)
        opt.zero_grad()
    ld.eval()
    moved = _check_identical(ld, x, y, 4, 5.0)
    with ema.applied():
        in_ema = _check_identical(ld, x, y, 4, 5.0)
    assert not _same(moved, in_ema)
    assert _same(_check_identical(ld, x, y, 4, 5.0), moved)
    assert all(g.captures == 1 for g in graphs.values())
    # .to() rebinds the storage: the graphs are dropped with the old engine and captured anew
    ld.dit.to(DEV)
    assert ld.dit.engine._sampler_graphs == {}
    _check_identical(ld, x, y, 4, 5.0)
    ld.dit.engine.release_sampler_graphs()
    assert ld.dit.engine._sampler_graphs == {}


def test_replay_does_not_sync_with_the_host(monkeypatch):
    ld = _small("P")
    x, y = _inputs(ld, 2)
    orig = engine_mod.SamplerGraph._replay
    replays = []

    def strict(self, n, debug):
        torch.cuda.set_sync_debug_mode("error")
        try:
            orig(self, n, debug)
        finally:
            torch.cuda.set_sync_debug_mode(0)
        replays.append(n)

    monkeypatch.setattr(engine_mod.SamplerGraph, "_replay", strict)
    for cfg in (1.0, 5.0):
        a = ld.edm_sampler_loop(x, y, steps=4, cfg=cfg)
        assert torch.isfinite(a).all()
    assert replays == [4, 4]


# ------------------------------------------------------------------------------------------------ kernels
def _heun_ref(stage, x, x_hat, d_cur, den, noise, table, k, m, s_noise):
    """The torch fp64 expressions of _heun the stages replace, with 0-dim device tensors like the eager loop."""
    tc, tn, th = table[k], table[k + 1], table[m + 1 + k]
    if stage == 0:
        x_hat = x + (th ** 2 - tc ** 2).sqrt() * s_noise * noise[k]
        return x, x_hat, d_cur, x_hat.to(torch.float32), th.to(torch.float32)
    if stage == 1:
        d_cur = (x_hat - den.to(torch.float64)) / th
        x = x_hat + (tn - th) * d_cur
        return x, x_hat, d_cur, x.to(torch.float32), tn.to(torch.float32)
    d_prime = (x - den.to(torch.float64)) / tn
    return x_hat + (tn - th) * (0.5 * d_cur + 0.5 * d_prime), x_hat, d_cur, None, None


@pytest.mark.parametrize("copies", [1, 2])
def test_heun_stage_kernels_match_torch(copies):
    from micro_diffusion_b200.ops import CudaOps
    o = CudaOps(DEV)
    g = torch.Generator(device=DEV).manual_seed(11)
    B, shape, m = 3, (4, 8, 8), 6
    f64 = torch.float64
    # a schedule reaching sigma_min, with t_hat > t_cur on some steps
    t = torch.tensor([80.0, 17.5, 2.52, 0.17, 0.0021, 0.002, 0.0], dtype=f64, device=DEV)
    th = t[:m] * torch.tensor([1.0, 1.3, 1.41, 1.0, 1.2, 1.0], dtype=f64, device=DEV)
    table = torch.cat([t, th])
    noise = torch.randn((m, B, *shape), dtype=f64, device=DEV, generator=g)
    for k in range(m):
        for stage in (0, 1, 2):
            x = torch.randn((B, *shape), dtype=f64, device=DEV, generator=g) * t[k]
            x_hat = x + torch.randn(x.shape, dtype=f64, device=DEV, generator=g) * 1e-3
            d_cur = torch.randn(x.shape, dtype=f64, device=DEV, generator=g)
            den = torch.randn(x.shape, device=DEV, generator=g)
            want = _heun_ref(stage, x, x_hat, d_cur, den, noise, table, k, m, 1.003)
            xin = torch.full((copies * B, *shape), float("nan"), device=DEV)
            sigma = torch.full((copies * B,), float("nan"), device=DEV)
            step = torch.tensor([k], dtype=torch.int32, device=DEV)
            o.edm_heun(stage, x, x_hat, d_cur, den, noise, xin if stage < 2 else None, sigma, table, step, 1.003)
            assert torch.equal(x, want[0]) and torch.equal(x_hat, want[1]) and torch.equal(d_cur, want[2]), (k, stage)
            if stage < 2:
                for c in range(copies):
                    assert torch.equal(xin[c * B:(c + 1) * B], want[3]), (k, stage)
                assert torch.equal(sigma, want[4].expand(copies * B)), (k, stage)
    o.edm_heun(o.HEUN_NEXT, None, None, None, None, None, None, None, None, step, 1.0)
    assert int(step) == m
    with pytest.raises(MicroditLibraryError):
        o._call("md_edm_heun", 5, *([None] * 8), step.data_ptr(), m, B, 1, 1, 1.0)
    with pytest.raises(MicroditLibraryError):
        o._call("md_edm_heun", 1, x.data_ptr(), x.data_ptr(), None, None, None, None, None, table.data_ptr(),
                step.data_ptr(), m, B, 1, 1, 1.0)


def test_heun_stage_poisons_out_of_range_steps():
    from micro_diffusion_b200.ops import CudaOps
    o = CudaOps(DEV)
    f64 = torch.float64
    table = torch.tensor([1.0, 0.5, 0.0, 1.0, 0.5], dtype=f64, device=DEV)
    x = torch.ones((2, 4), dtype=f64, device=DEV)
    noise = torch.ones((2, 2, 4), dtype=f64, device=DEV)
    for k in (-1, 2, 1000):
        x_hat = torch.zeros_like(x)
        xin, sigma = torch.zeros((2, 4), device=DEV), torch.zeros(2, device=DEV)
        o.edm_heun(0, x, x_hat, None, None, noise, xin, sigma, table, torch.tensor([k], dtype=torch.int32, device=DEV),
                   1.0)
        assert x_hat.isnan().all() and xin.isnan().all() and sigma.isnan().all()


def test_guided_output_kernel_matches_torch():
    from micro_diffusion_b200.ops import CudaOps
    o = CudaOps(DEV)
    g = torch.Generator(device=DEV).manual_seed(12)
    B, C, H, W, p, sd = 3, 4, 16, 16, 2, 0.9
    T, Nf = (H // p) * (W // p), p * p * C
    ftok = torch.randn(2 * B * T, Nf, device=DEV, generator=g)
    x = torch.randn(B, C, H, W, device=DEV, generator=g)
    sigma_b = torch.tensor([0.002, 0.00201, 14.5], device=DEV)
    for cfg in (5.0, 3.0, 1.5):
        dx = torch.full_like(x, float("nan"))
        o.edm_output_cfg(ftok, x, sigma_b, torch.tensor([cfg], device=DEV), dx, sd, p)
        # the token layout of md_edm_output (unpatchify), then model.py:197-201 as written
        fx = ftok.reshape(2 * B, H // p, W // p, p, p, C).permute(0, 5, 1, 3, 2, 4).reshape(2 * B, C, H, W)
        cond, unc = torch.split(fx, B, dim=0)
        f = unc + cfg * (cond - unc)
        sg = sigma_b.view(-1, 1, 1, 1)
        want = (sd ** 2 / (sg ** 2 + sd ** 2)) * x + (sg * sd / (sg ** 2 + sd ** 2).sqrt()) * f
        assert torch.equal(dx, want), cfg
    with pytest.raises(MicroditLibraryError):
        o._call("md_edm_output_cfg", ftok.data_ptr(), x.data_ptr(), sigma_b.data_ptr(), None, dx.data_ptr(), 0.9, 0.81,
                B, C, H, W, p)
    with pytest.raises(AssertionError):
        o.edm_output_cfg(ftok[:-1], x, sigma_b, torch.tensor([5.0], device=DEV), dx, sd, p)
