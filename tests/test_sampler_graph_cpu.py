"""Host side of the CUDA-graph Heun sampler (engine.SamplerGraph), without a GPU: the eligibility rule, the schedule table,
the pre-drawn noise, and a pure-torch restatement of the three md_edm_heun stages in the kernels' association order, which
must reproduce LatentDiffusion._heun bit for bit (it pins the order the CUDA code follows)."""
import ctypes
from functools import partial

import numpy as np
import pytest
import torch

from micro_diffusion_b200 import ops as ops_mod
from micro_diffusion_b200.engine import SamplerGraph
from micro_diffusion_b200.models.model import LatentDiffusion
from oracle.emu_ops import EmuOps
from tests import parity_common as pc


def _ld():
    return pc.build_product("P", ops_factory=lambda d: EmuOps(d))


class _FakeDenoiser(LatentDiffusion):
    """_heun over a cheap deterministic fp32 denoiser: the sampler arithmetic is what is under test."""

    def model_forward_wrapper(self, x, sigma, y, model_forward_fxn, mask_ratio=0.0, **kwargs):
        return {"sample": torch.tanh(x) * 0.7 + sigma.reshape(-1, 1, 1, 1) * 0.01}


def _fake_ld(churn):
    ld = _ld()
    ld.__class__ = _FakeDenoiser
    if churn:  # gamma switches on and off mid-run (5 steps: t ~ 80, 17.5, 2.5, 0.17, 0.002)
        ld.edm_config.update(S_churn=40, S_min=0.1, S_max=10)
    return ld


def _t_steps(ld, n):
    e = ld.edm_config
    i = torch.arange(n, dtype=torch.float64)
    t = (e.sigma_max ** (1 / e.rho) + i / (n - 1) * (e.sigma_min ** (1 / e.rho) - e.sigma_max ** (1 / e.rho))) ** e.rho
    return torch.cat([t, torch.zeros_like(t[:1])])


def test_eligibility_rule(monkeypatch):
    ld = _ld()
    x, y = torch.zeros(2, 4, 32, 32), torch.zeros(2, 1, 77, 1024)
    fwd, fwd_cfg = ld.dit.forward, partial(ld.dit.forward, cfg=5.0)
    assert not ld._sampler_graph_eligible(fwd, x, y, {})  # EmuOps: the eager loop
    monkeypatch.setattr(ops_mod, "CudaOps", EmuOps)     # from here on the ops count as the CUDA ops
    assert ld._sampler_graph_eligible(fwd, x, y, {}) and ld._sampler_graph_eligible(fwd_cfg, x, y, {})
    assert not ld._sampler_graph_eligible(fwd, x, y, {"extra": 1})
    assert not ld._sampler_graph_eligible(lambda *a, **k: None, x, y, {})
    with torch.enable_grad():
        assert ld._sampler_graph_eligible(fwd, x, y, {})  # grad mode alone: the sampler computes no gradient anyway
        assert not ld._sampler_graph_eligible(fwd, x.clone().requires_grad_(), y, {})
        assert not ld._sampler_graph_eligible(fwd, x, y.clone().requires_grad_(), {})
    with torch.no_grad():
        assert ld._sampler_graph_eligible(fwd, x.clone().requires_grad_(), y, {})
    ld.cache_prompt = False
    assert not ld._sampler_graph_eligible(fwd, x, y, {})
    ld.cache_prompt, ld.sampler_graph = True, False
    assert not ld._sampler_graph_eligible(fwd, x, y, {})
    ld.sampler_graph = True
    ld.__class__ = _FakeDenoiser  # overrides model_forward_wrapper
    assert not ld._sampler_graph_eligible(fwd, x, y, {})


@pytest.mark.parametrize("churn", [False, True])
@pytest.mark.parametrize("n", [1, 2, 5, 30])
def test_schedule_table_matches_heun(n, churn):
    ld = _fake_ld(churn)
    e = ld.edm_config
    t_steps = _t_steps(ld, n)
    t_cpu, t_hat = ld._heun_schedule(t_steps, n)
    want = []
    for t_cur in t_steps[:-1]:  # _heun's own expressions
        gamma = min(e.S_churn / n, np.sqrt(2) - 1) if e.S_min <= t_cur <= e.S_max else 0
        want.append(torch.as_tensor(t_cur + gamma * t_cur))
    tab = SamplerGraph.schedule_table(t_cpu, t_hat, n + 3)
    m = n + 3
    same = lambda a, b: torch.equal(torch.nan_to_num(a, 7.0), torch.nan_to_num(b, 7.0))
    assert same(tab[:n + 1], t_steps) and same(tab[m + 1:m + 1 + n], torch.stack(want))
    assert not tab[n + 1:m + 1].any() and not tab[m + 1 + n:].any()
    if churn and n == 5:
        assert [bool(a != b) for a, b in zip(t_hat, t_steps[:-1])] == [False, False, True, True, False]


def test_predrawn_noise_leaves_the_generator_where_the_eager_loop_does():
    n = 4
    x = torch.randn(2, 4, 32, 32, generator=torch.Generator().manual_seed(0))
    y = torch.zeros(2, 1, 77, 1024)
    runs = {}
    for mode in ("eager", "predraw"):
        ld = _fake_ld(False)
        g = torch.Generator().manual_seed(123)
        drawn = []
        ld.randn_like = lambda t: drawn.append(torch.randn(t.shape, dtype=t.dtype, generator=g)) or drawn[-1]
        if mode == "eager":
            ld.edm_sampler_loop(x, y, steps=n)
        else:
            ld._predraw_noise(x.to(torch.float64), n)
        runs[mode] = (drawn, g.get_state())
    (a, sa), (b, sb) = runs["eager"], runs["predraw"]
    assert len(a) == len(b) == n and all(torch.equal(u, v) for u, v in zip(a, b))
    assert all(u.dtype == torch.float64 for u in b)
    assert torch.equal(sa, sb)


def _stage_in(x, noise, t_cur, t_hat, s_noise):
    return x + (torch.sqrt(t_hat * t_hat - t_cur * t_cur) * s_noise) * noise


def _stage_euler(x_hat, den, t_hat, t_next):
    d_cur = (x_hat - den.to(torch.float64)) / t_hat
    return d_cur, x_hat + (t_next - t_hat) * d_cur


def _stage_correct(x, x_hat, d_cur, den, t_hat, t_next):
    d_prime = (x - den.to(torch.float64)) / t_next
    return x_hat + (t_next - t_hat) * (0.5 * d_cur + 0.5 * d_prime)


@pytest.mark.parametrize("churn", [False, True])
@pytest.mark.parametrize("n", [2, 5])
def test_stage_restatement_reproduces_heun(n, churn):
    """md_edm_heun's stages as torch ops on 0-dim fp64 tensors read from the schedule table, fed with the fp32 casts the
    kernels write (x_hat / x_next and t_hat / t_next .to(float32)), equal _heun bit for bit."""
    ld = _fake_ld(churn)
    ld.edm_config.S_noise = 1.003
    x = torch.randn(2, 4, 32, 32, generator=torch.Generator().manual_seed(1))
    y = torch.zeros(2, 1, 77, 1024)
    torch.manual_seed(5)
    want = ld.edm_sampler_loop(x, y, steps=n)
    t_steps = _t_steps(ld, n)
    t_cpu, t_hat = ld._heun_schedule(t_steps, n)
    torch.manual_seed(5)
    noise = ld._predraw_noise(x.to(torch.float64), n)
    tab = SamplerGraph.schedule_table(t_cpu, t_hat, n)
    den = lambda v, s: ld.model_forward_wrapper(v.to(torch.float32), s.to(torch.float32), y, None)["sample"]
    xs = x.to(torch.float64) * t_steps[0]
    for k in range(n):
        tc, tn, th = tab[k], tab[k + 1], tab[n + 1 + k]
        x_hat = _stage_in(xs, noise[k], tc, th, ld.edm_config.S_noise)
        d_cur, xs = _stage_euler(x_hat, den(x_hat, th), th, tn)
        if k < n - 1:
            xs = _stage_correct(xs, x_hat, d_cur, den(xs, tn), th, tn)
    assert torch.equal(xs.to(torch.float32), want)


def test_guided_output_restatement_matches_model_forward_wrapper():
    """md_edm_output_cfg's rounding: c_skip = reciprocal(sg*sg + sd2) * sd2, c_out = (sg*sd) / sqrt(sg*sg + sd2), every
    fp32 product and sum on its own -- the torch expression of the guided branch (model.py:197-201)."""
    g = torch.Generator().manual_seed(3)
    B, sd, cfg = 3, 0.9, 5.0
    x, cond, unc = (torch.randn(B, 4, 8, 8, generator=g) for _ in range(3))
    sigma = torch.tensor([0.002, 0.0021, 37.0])
    f = unc + cfg * (cond - unc)
    sg = sigma.view(-1, 1, 1, 1)
    want = (sd ** 2 / (sg ** 2 + sd ** 2)) * x + (sg * sd / (sg ** 2 + sd ** 2).sqrt()) * f
    sd_f, sd2_f = torch.tensor(sd, dtype=torch.float32), torch.tensor(sd ** 2, dtype=torch.float32)
    den = sg * sg + sd2_f
    got = (den.reciprocal() * sd2_f) * x + ((sg * sd_f) / den.sqrt()) * (unc + torch.tensor(cfg, dtype=torch.float32) * (cond - unc))
    assert torch.equal(got, want)


def test_sampler_entry_points_refuse_malformed_arguments():
    """Argument checks happen before any launch, so they run without a GPU."""
    from micro_diffusion_b200 import _lib
    lib = _lib.load()
    lib.md_last_error.restype = ctypes.c_char_p
    heun = lib.md_edm_heun
    heun.restype, heun.argtypes = ctypes.c_int, ops_mod._PROTOS["md_edm_heun"]
    p = ctypes.c_void_p(16)  # never dereferenced: every call below is refused first

    def call(stage, x=p, x_hat=p, d_cur=p, den=p, noise=p, xin=p, sigma=p, table=p, step=p, max_steps=4, B=2, n=64,
             copies=1):
        return heun(stage, x, x_hat, d_cur, den, noise, xin, sigma, table, step, max_steps, B, n, copies, 1.0, None)

    for bad in (dict(stage=4), dict(stage=-1), dict(stage=0, step=None), dict(stage=3, step=None),
                dict(stage=0, noise=None), dict(stage=0, xin=None), dict(stage=0, sigma=None), dict(stage=0, table=None),
                dict(stage=1, den=None), dict(stage=1, d_cur=None), dict(stage=2, x_hat=None), dict(stage=2, den=None),
                dict(stage=0, max_steps=0), dict(stage=1, B=0), dict(stage=1, n=0), dict(stage=0, copies=3)):
        assert call(**bad) == -1, bad
        assert lib.md_last_error().startswith(b"md_edm_heun")
    cfg = lib.md_edm_output_cfg
    cfg.restype, cfg.argtypes = ctypes.c_int, ops_mod._PROTOS["md_edm_output_cfg"]
    for args in ((None, p, p, p, p, 0.9, 0.81, 2, 4, 8, 8, 2, None), (p, p, p, None, p, 0.9, 0.81, 2, 4, 8, 8, 2, None),
                 (p, p, p, p, None, 0.9, 0.81, 2, 4, 8, 8, 2, None), (p, p, p, p, p, 0.9, 0.81, 2, 4, 8, 7, 2, None),
                 (p, p, p, p, p, 0.9, 0.81, 2, 4, 8, 8, 0, None)):
        assert cfg(*args) == -1, args
        assert lib.md_last_error().startswith(b"md_edm_output_cfg")
