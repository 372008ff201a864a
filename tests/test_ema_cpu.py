"""Weight EMA (ema.FlatEMA) on CPU: the kernels are the CPU contracts (tests/ema_common.EMAEmuOps, exact fp32)."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from tests import ema_common as ec
from tests import parity_common as pc
from tests.test_train_config_cpu import REF_CONFIGS

KW = dict(lr=1e-3, eps=1e-2, t_warmup="2ba", alpha_f=0.33, device_train_microbatch_size=2, log_every=1)


def _build(name="P"):
    return pc.build_product(name, ops_factory=lambda d: ec.EMAEmuOps(d, exact=True))


def _loader(n, B=4, seed0=50):
    from oracle import weights
    return [weights.synth_batch(B, 4, 32, seed=seed0 + i) for i in range(n)]


def _run(n=4, record=False, **ema):
    """A Trainer over n batches from seed 3: (trainer, logged losses, flat weights after every step if `record`)."""
    from micro_diffusion_b200.trainer import Trainer
    model = _build()
    logs, snaps = [], []
    torch.manual_seed(3)
    tr = Trainer(model, _loader(n), max_duration=f"{n}ba", log_fn=logs.append, **KW, **ema)
    if record:
        step = tr.optimizer.step

        def recording(*a, **k):
            step(*a, **k)
            snaps.append(model.dit.store.flat.clone())
        tr.optimizer.step = recording
    tr.fit()
    return tr, [s.split(" lr ")[0] for s in logs], snaps


def test_ema_leaves_training_bit_identical():
    plain, lp, _ = _run()
    withe, le, _ = _run(ema_smoothing=0.9, ema_start="1ba", ema_update_interval="1ba")
    assert plain.ema is None and withe.ema is not None and withe.ema.started
    assert torch.equal(plain.model.dit.store.flat, withe.model.dit.store.flat)
    assert torch.equal(plain.optimizer.m, withe.optimizer.m) and torch.equal(plain.optimizer.v, withe.optimizer.v)
    assert lp == le and len(lp) == 4


@pytest.mark.parametrize("ema", [
    dict(ema_smoothing=0.9, ema_start="1ba"),
    dict(ema_half_life="3ba", ema_start="1ba"),
    dict(ema_smoothing=0.8, ema_start="2ba"),
    dict(ema_smoothing=0.75, ema_start="1ba", ema_update_interval="2ba"),
])
def test_ema_matches_the_torch_restatement_of_the_schedule(ema):
    tr, _, snaps = _run(record=True, **ema)
    e = tr.ema
    if "ema_half_life" in ema:
        assert e.smoothing == 2.0 ** (-1 / 3)
    assert len(snaps) == 4
    want = ec.ema_reference(snaps, e.smoothing, e.ema_start, e.update_interval)
    assert torch.equal(e.ema, want)
    assert not torch.equal(e.ema, tr.model.dit.store.flat)


def test_flat_ema_arguments():
    from micro_diffusion_b200.ema import FlatEMA
    dit = _build().dit
    with pytest.raises(ValueError):
        FlatEMA(dit)
    with pytest.raises(ValueError):
        FlatEMA(dit, smoothing=0.9, half_life="10ba")
    with pytest.raises(ValueError):
        FlatEMA(dit, smoothing=0.9, ema_start="1ep")
    with pytest.raises(ValueError):
        FlatEMA(dit, half_life="2dur")
    assert FlatEMA(dit, half_life="8ba", update_interval="2ba").smoothing == 2.0 ** (-2 / 8)
    e = FlatEMA(dit, smoothing=0.5, ema_start="5ba")
    before = dit.store.flat.clone()
    with e.applied():  # not started: nothing happens
        assert torch.equal(dit.store.flat, before)


def test_evaluate_runs_on_the_ema_weights(tmp_path):
    from micro_diffusion_b200.trainer import Trainer, ema_state_dict
    tr, _, _ = _run(ema_smoothing=0.5, ema_start="1ba")
    tr.eval_loader = _loader(2, seed0=900)
    ck = str(tmp_path / "ema.pt")
    from micro_diffusion_b200.trainer import save_checkpoint
    save_checkpoint(ck, tr.model, tr.optimizer, tr.batch, ema=tr.ema)
    flat = tr.model.dit.store.flat.clone()
    torch.manual_seed(11)
    got = tr.evaluate()
    assert torch.equal(tr.model.dit.store.flat, flat)  # training weights restored bit for bit
    other = _build()
    other.dit.load_state_dict(ema_state_dict(ck))
    assert torch.equal(other.dit.store.flat, tr.ema.ema)
    torch.manual_seed(11)
    want = Trainer(other, [], max_duration="1ba", log_fn=lambda s: None, eval_dataloader=tr.eval_loader,
                   **KW).evaluate()
    assert got == want
    # and the training weights give another loss
    torch.manual_seed(11)
    assert tr._evaluate() != got


def test_checkpoint_resume_and_ignore_keys(tmp_path):
    from micro_diffusion_b200.trainer import Trainer
    ema = dict(ema_smoothing=0.6, ema_start="1ba")
    a, _, _ = _run(**ema)
    b = _build()
    torch.manual_seed(3)
    tb = Trainer(b, _loader(2), max_duration="4ba", save_folder=str(tmp_path), save_interval="2ba",
                 log_fn=lambda s: None, **KW, **ema)
    tb.fit(until=2)
    rng = torch.get_rng_state()
    ck = os.path.join(str(tmp_path), "ba2.pt")
    raw = torch.load(ck, weights_only=False)
    entry = raw["state"]["algorithms"]["EMA"]
    assert entry["started"] and entry["smoothing"] == 0.6 and entry["update_interval"] == 1 and entry["ema_start"] == 1
    assert set(entry["ema_weights"]) == {f"dit.{k}" for k, _ in b.dit.named_parameters()}
    flat2 = b.dit.store.flat.clone()
    c = _build()
    tc = Trainer(c, _loader(4)[2:], max_duration="4ba", load_path=ck, log_fn=lambda s: None, **KW, **ema)
    assert tc.batch == 2 and tc.ema.started and torch.equal(tc.ema.ema, tb.ema.ema)
    torch.set_rng_state(rng)
    tc.fit()
    assert torch.equal(c.dit.store.flat, a.model.dit.store.flat)
    assert torch.equal(tc.ema.ema, a.ema.ema)
    # weights only: the training weights, no EMA
    d = _build()
    td = Trainer(d, [], max_duration="4ba", load_path=ck, load_weights_only=True, log_fn=lambda s: None, **KW, **ema)
    assert td.batch == 0 and not td.ema.started and torch.equal(d.dit.store.flat, flat2)
    # the EMA entry dropped, whole or in part: the EMA starts again on its schedule
    for pat in ("state/algorithms/EMA*", "state/algorithms/EMA/ema_weights/dit.blocks.0.*"):
        e = _build()
        te = Trainer(e, [], max_duration="4ba", load_path=ck, load_ignore_keys=[pat], log_fn=lambda s: None, **KW,
                     **ema)
        assert te.batch == 2 and not te.ema.started and torch.equal(e.dit.store.flat, flat2)
    with pytest.raises(ValueError):
        from micro_diffusion_b200.trainer import ema_state_dict, save_checkpoint
        plain = str(tmp_path / "plain.pt")
        save_checkpoint(plain, a.model, a.optimizer, 4)
        ema_state_dict(plain)


def test_nonfinite_step_leaves_the_ema_untouched():
    from micro_diffusion_b200.ema import FlatEMA
    from micro_diffusion_b200.train_step import FlatAdamW
    ld = _build()
    st = ld.dit.store
    opt = FlatAdamW(ld.dit, lr=1e-3)
    ema = FlatEMA(ld.dit, smoothing=0.5)
    st.grad.normal_()
    opt.step(None, None, ema)  # batch 1: the EMA starts (copy)
    st.grad.normal_()
    opt.step(None, None, ema)  # batch 2: fused update
    assert ema.started and int(opt.nonfinite) == 0
    e, p, m = ema.ema.clone(), st.flat.clone(), opt.m.clone()
    st.grad.normal_()
    st.grad[7] = float("nan")
    opt.step(None, None, ema)
    assert int(opt.nonfinite) == 1
    assert torch.equal(ema.ema, e) and torch.equal(st.flat, p) and torch.equal(opt.m, m)


def test_reference_yaml_ema_sections():
    from micro_diffusion_b200 import train
    want = {"res_512_pretrain": (0.99975, "25000ba"), "res_512_finetune": (0.9975, "1000ba")}
    for name, (s, start) in want.items():
        cfg = train.load_config(os.path.join(REF_CONFIGS, name + ".yaml"))
        kw = train.trainer_kwargs(cfg)
        assert (kw["ema_smoothing"], kw["ema_start"], kw["ema_update_interval"], kw["ema_half_life"]) == \
            (s, start, "1ba", None)
        assert "ema" not in " ".join(train.ignored_sections(cfg))
        off = train.trainer_kwargs(train.load_config(os.path.join(REF_CONFIGS, name + ".yaml"), ["algorithms.ema=null"]))
        assert not any(k.startswith("ema_") for k in off)
    for name in ("res_256_pretrain", "res_256_finetune"):
        kw = train.trainer_kwargs(train.load_config(os.path.join(REF_CONFIGS, name + ".yaml")))
        assert not any(k.startswith("ema_") for k in kw)
    base = {"_target_": "diffusion.algorithms.ema.EMA", "half_life": None, "smoothing": 0.99, "update_interval": "1ba",
            "ema_start": "0ba"}
    assert train.ema_kwargs({"algorithms": {"ema": base}})["ema_smoothing"] == 0.99
    assert train.ema_kwargs({"algorithms": {"ema": {**base, "smoothing": None, "half_life": "100ba"}}})[
        "ema_half_life"] == "100ba"
    for bad in ({"half_life": "100ba"}, {"smoothing": None}, {"ema_start": "1ep"}, {"update_interval": "2ep"},
                {"_target_": "composer.algorithms.SWA"}, {"beta": 1}):
        with pytest.raises(ValueError):
            train.ema_kwargs({"algorithms": {"ema": {**base, **bad}}})


# ------------------------------------------------------------------------------------------------ two gloo ranks
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


STEPS, SMOOTH = 3, 0.5


def _halves(step):
    from oracle import weights
    return weights.synth_batch(4, 4, 32, seed=70 + step)


def _worker(rank, world, port, out_path, shard):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.set_num_threads(2)
    from micro_diffusion_b200.ema import FlatEMA
    from micro_diffusion_b200.train_step import FlatAdamW, GradReducer
    ld = _build()
    opt = FlatAdamW(ld.dit, lr=1e-3, clip_norm=None, eps=1e-2)
    red = GradReducer(ld.dit.store, buckets=3, shard=shard)
    assert red.shard == shard
    ema = FlatEMA(ld.dit, smoothing=SMOOTH, ema_start="1ba")
    st = ld.dit.store
    for s in range(STEPS):
        full = _halves(s)
        mine = {k: v[rank * 2:(rank + 1) * 2].clone() for k, v in full.items()}
        torch.manual_seed(100 + 10 * s + rank)
        loss = ld(mine)[0]
        ld.dit.engine.on_backbone_grads_ready = red.reduce_early  # the owned shares are those of the early / late split
        loss.backward()
        ld.dit.engine.on_backbone_grads_ready = None
        red.reduce()
        opt.step(None, red, ema)
        opt.zero_grad()
    st.refresh_copies(ld.dit.engine.ops, None, force=True)
    flat = st.flat.clone()
    with ema.applied():
        applied = st.flat.clone()
    restored = st.flat.clone()
    ema.gather_state()
    torch.save({"flat": flat, "applied": applied, "restored": restored, "ema": ema.ema.clone()}, out_path + f".{rank}")
    dist.barrier()
    dist.destroy_process_group()


def test_two_rank_ema_sharded_equals_replicated_and_one_process(tmp_path):
    """Sharded (owned shares, swap + all-gather in applied()) and replicated (full buffers) EMAs over two gloo ranks:
    bit-identical to each other, equal to the one-process EMA over the concatenated batch, and applied() gives every
    rank the full EMA weights and restores the training weights bit for bit."""
    got = {}
    for shard in (False, True):
        out = str(tmp_path / f"rank{int(shard)}.pt")
        mp.start_processes(_worker, args=(2, _free_port(), out, shard), nprocs=2, join=True, start_method="spawn")
        got[shard] = [torch.load(f"{out}.{r}") for r in range(2)]
    for shard, ranks in got.items():
        for r in ranks:
            assert torch.equal(r["restored"], r["flat"])
            assert torch.equal(r["applied"], r["ema"])
        assert torch.equal(ranks[0]["ema"], ranks[1]["ema"]) and torch.equal(ranks[0]["flat"], ranks[1]["flat"])
    assert torch.equal(got[True][0]["ema"], got[False][0]["ema"])
    assert torch.equal(got[True][0]["flat"], got[False][0]["flat"])
    # one process over the concatenated batch
    from micro_diffusion_b200.ema import FlatEMA
    from micro_diffusion_b200.train_step import FlatAdamW
    ld = _build()
    opt = FlatAdamW(ld.dit, lr=1e-3, clip_norm=None, eps=1e-2)
    ema = FlatEMA(ld.dit, smoothing=SMOOTH, ema_start="1ba")
    for s in range(STEPS):
        full = _halves(s)
        for r in range(2):
            torch.manual_seed(100 + 10 * s + r)
            (0.5 * ld({k: v[r * 2:(r + 1) * 2].clone() for k, v in full.items()})[0]).backward()
        opt.step(None, None, ema)
        opt.zero_grad()
    assert torch.allclose(got[True][0]["flat"], ld.dit.store.flat, rtol=1e-5, atol=1e-6)
    assert torch.allclose(got[True][0]["ema"], ema.ema, rtol=1e-5, atol=1e-6)
