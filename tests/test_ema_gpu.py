"""Weight EMA on the H100: md_adamw_ema / md_swap_f32 against md_adamw and torch, the Trainer with and without EMA on
MicroDiT_Tiny_2 / MicroDiT_XL_2 (C2 shapes), sampling from the EMA, and the sharded swap over two GPUs (skipped on a
one-GPU machine)."""
import gc
import os
import socket

import pytest
import torch

from tests import ema_common as ec

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _ops():
    from micro_diffusion_b200.ops import CudaOps
    return CudaOps(DEV)


@pytest.fixture
def deterministic():
    """Deterministic mode for the test (the fast path's atomics are not bit-reproducible from run to run)."""
    ops = _ops()
    ops.set_deterministic(True)
    yield
    ops.set_deterministic(False)


def _f32(x):
    return float(torch.tensor(x, dtype=torch.float32))


def test_adamw_ema_kernel_matches_adamw_and_torch():
    ops = _ops()
    g = torch.Generator(device=DEV).manual_seed(5)
    n = 3 * 1024 * 1024 + 3  # float4 body + a 3-element tail
    p0 = torch.randn(n, device=DEV, generator=g)
    gr = torch.randn(n, device=DEV, generator=g) * 1e-2
    m0 = torch.randn(n, device=DEV, generator=g) * 1e-3
    v0 = torch.rand(n, device=DEV, generator=g) * 1e-4
    e0 = p0 + 1e-2 * torch.randn(n, device=DEV, generator=g)
    sumsq = torch.zeros(1, device=DEV)
    ops.sumsq(gr, sumsq)
    for s in (_f32(0.9975), _f32(0.5), 0.0, 1.0):
        args = (sumsq, 0.25, 2.4e-4, 0.9, 0.999, 1e-8, 0.1, 7)
        pa, ma, va = p0.clone(), m0.clone(), v0.clone()
        ops.adamw(pa, gr, ma, va, *args)
        pb, mb, vb, eb = p0.clone(), m0.clone(), v0.clone(), e0.clone()
        flag = torch.zeros(1, dtype=torch.int32, device=DEV)
        ops.adamw_ema(pb, gr, mb, vb, *args, eb, s, nonfinite=flag)
        torch.cuda.synchronize()
        assert torch.equal(pa, pb) and torch.equal(ma, mb) and torch.equal(va, vb) and int(flag) == 0
        want = ec.ema_update(e0, pa, s)
        assert bool(((eb - want).abs() <= ec.ulp_bound(e0, pa, s)).all()), s
    # a non-finite gradient norm: nothing is written, the flag is raised
    bad = torch.full((1,), float("inf"), device=DEV)
    pb, mb, vb, eb = p0.clone(), m0.clone(), v0.clone(), e0.clone()
    flag = torch.zeros(1, dtype=torch.int32, device=DEV)
    ops.adamw_ema(pb, gr, mb, vb, bad, 0.25, 2.4e-4, 0.9, 0.999, 1e-8, 0.1, 7, eb, 0.99, nonfinite=flag)
    torch.cuda.synchronize()
    assert int(flag) == 1
    assert torch.equal(pb, p0) and torch.equal(mb, m0) and torch.equal(vb, v0) and torch.equal(eb, e0)


def test_swap_kernel_exchanges_and_rejects_aliasing():
    from micro_diffusion_b200.ops import MicroditLibraryError
    ops = _ops()
    buf = torch.randn(2 * 100003 + 8, device=DEV)
    for off in (0, 1):  # 16-byte aligned (float4 body) and misaligned (scalar) ranges
        a, b = buf[off:off + 100003], buf[100003 + 5:2 * 100003 + 5]
        a0, b0 = a.clone(), b.clone()
        ops.swap(a, b)
        torch.cuda.synchronize()
        assert torch.equal(a, b0) and torch.equal(b, a0)
    with pytest.raises(MicroditLibraryError):
        ops.swap(buf[:1000], buf[:1000])
    with pytest.raises(MicroditLibraryError):
        ops.swap(buf[:1000], buf[4:1004])


def _loader(n, B, dev=DEV):
    from oracle import weights
    return [{k: v.to(dev) for k, v in weights.synth_batch(B, 4, 32, seed=300 + i).items()} for i in range(n)]


def _model(arch):
    from micro_diffusion_b200.models.model import create_latent_diffusion, PrecomputedLatentStubs
    torch.manual_seed(0)
    return create_latent_diffusion(dit_arch=arch, latent_res=32, in_channels=4, train_mask_ratio=0.75,
                                   vae=PrecomputedLatentStubs._VAE(), text_encoder=PrecomputedLatentStubs._Text(),
                                   tokenizer=PrecomputedLatentStubs._Tok()).to(DEV)


KW = dict(lr=1e-4, t_warmup="0ba", device_train_microbatch_size=2, log_every=1, log_fn=lambda s: None)


@pytest.mark.parametrize("arch", ["MicroDiT_Tiny_2", "MicroDiT_XL_2"])
def test_trainer_with_ema_keeps_training_bit_identical(arch, deterministic):
    """A few steps at C2 shapes (res 256 latents, mask 0.75, batch 2) with and without EMA (start 1, every batch):
    bit-identical weights; the start is an exact copy and every fused update matches torch per element."""
    from micro_diffusion_b200.trainer import Trainer
    steps = 3
    ld = _model(arch)
    torch.manual_seed(3)
    Trainer(ld, _loader(steps, 2), max_duration=f"{steps}ba", **KW).fit()
    plain = ld.dit.store.flat.cpu()
    del ld
    gc.collect()
    torch.cuda.empty_cache()
    ld = _model(arch)
    torch.manual_seed(3)
    tr = Trainer(ld, _loader(steps, 2), max_duration=f"{steps}ba", ema_smoothing=0.75, ema_start="1ba", **KW)
    ema, flat, checked = tr.ema, ld.dit.store.flat, []
    step = tr.optimizer.step

    def checking(*a, **k):
        prev = ema.ema.clone() if ema.started else None
        step(*a, **k)
        if prev is None:
            assert torch.equal(ema.ema, flat)  # the start: a plain copy
        else:
            err = (ema.ema - ec.ema_update(prev, flat, ema.smoothing)).abs()
            assert bool((err <= ec.ulp_bound(prev, flat, ema.smoothing)).all())
        checked.append(prev is not None)
    tr.optimizer.step = checking
    tr.fit()
    assert checked == [False, True, True]
    assert torch.equal(flat.cpu(), plain)


class _Encoder:
    """A text encoder stand-in: fixed caption embeddings per token row ([B, 1, 77, 1024] fp16)."""

    def encode(self, tokens, attention_mask=None):
        g = torch.Generator(device=tokens.device).manual_seed(int(tokens.sum()))
        return (torch.randn(tokens.shape[0], 1, 77, 1024, device=tokens.device, generator=g).half(),)


def test_generate_under_applied_equals_a_model_loaded_from_ema_state_dict(tmp_path, deterministic):
    from micro_diffusion_b200.trainer import Trainer, ema_state_dict
    ld = _model("MicroDiT_Tiny_2")
    tr = Trainer(ld, _loader(3, 2), max_duration="3ba", ema_smoothing=0.5, ema_start="1ba",
                 save_folder=str(tmp_path), save_interval="3ba", **KW)
    tr.fit()
    toks = torch.arange(2 * 77, device=DEV).reshape(2, 77)
    ld.text_encoder, ld.vae.device = _Encoder(), torch.device(DEV)
    flat = ld.dit.store.flat.clone()
    with tr.ema.applied():
        a = ld.generate(tokenized_prompts=toks, num_inference_steps=3, guidance_scale=3.0, seed=7,
                        return_only_latents=True)
    assert torch.equal(ld.dit.store.flat, flat)
    b_model = _model("MicroDiT_Tiny_2")
    b_model.text_encoder, b_model.vae.device = _Encoder(), torch.device(DEV)
    b_model.dit.load_state_dict(ema_state_dict(os.path.join(str(tmp_path), "ba3.pt")))
    b = b_model.generate(tokenized_prompts=toks, num_inference_steps=3, guidance_scale=3.0, seed=7,
                         return_only_latents=True)
    assert torch.equal(a, b)
    c = ld.generate(tokenized_prompts=toks, num_inference_steps=3, guidance_scale=3.0, seed=7, return_only_latents=True)
    assert not torch.equal(a, c)  # the training weights sample something else (the prompt cache was invalidated)


# ------------------------------------------------------------------------------------------------ two GPUs
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, out, shard):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    from micro_diffusion_b200.ema import FlatEMA
    from micro_diffusion_b200.train_step import FlatAdamW, GradReducer
    from oracle import weights
    from tests import parity_common as pc
    ld = pc.build_product("S", device=dev)
    opt = FlatAdamW(ld.dit, lr=1e-3, clip_norm=0.25, eps=1e-2)
    red = GradReducer(ld.dit.store, ops=ld.dit.engine.ops, shard=shard)
    assert red.shard == shard
    ema = FlatEMA(ld.dit, smoothing=0.5, ema_start="1ba")
    st = ld.dit.store
    for s in range(3):
        full = {k: v.to(dev) for k, v in weights.synth_batch(6, 4, 16, seed=80 + s).items()}
        torch.manual_seed(100 + 10 * s + rank)
        loss = ld({k: v[rank * 3:(rank + 1) * 3].clone() for k, v in full.items()})[0]
        ld.dit.engine.on_backbone_grads_ready = red.reduce_early
        loss.backward()
        ld.dit.engine.on_backbone_grads_ready = None
        red.reduce()
        opt.step(None, red, ema)
        opt.zero_grad()
    st.refresh_copies(ld.dit.engine.ops, None, force=True)
    torch.cuda.synchronize()
    flat = st.flat.cpu()
    with ema.applied():
        torch.cuda.synchronize()
        applied = st.flat.cpu()
    st.refresh_copies(ld.dit.engine.ops, None, force=True)
    torch.cuda.synchronize()
    restored = st.flat.cpu()
    ema.gather_state()
    torch.cuda.synchronize()
    torch.save({"flat": flat, "applied": applied, "restored": restored, "ema": ema.ema.cpu()}, f"{out}.{rank}")
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("shard", [True, False])
def test_two_gpu_ema_swap_and_gather(tmp_path, shard):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    import torch.multiprocessing as mp
    out = str(tmp_path / "rank.pt")
    mp.start_processes(_worker, args=(2, _free_port(), out, shard), nprocs=2, join=True, start_method="spawn")
    got = [torch.load(f"{out}.{r}") for r in range(2)]
    for r in got:
        assert torch.equal(r["restored"], r["flat"]) and torch.equal(r["applied"], r["ema"])
    assert torch.equal(got[0]["ema"], got[1]["ema"]) and torch.equal(got[0]["flat"], got[1]["flat"])
