"""Run the reference's YAML configs without Hydra / Composer (SURVEY.md §8 f-2):

    torchrun --nproc-per-node 8 -m micro_diffusion_b200.train --config-path configs --config-name res_256_pretrain.yaml \
        trainer.device_train_microbatch_size=512 dataset.train.datadir=[/data/mds_latents]

The file format and the keys are the reference's (configs/res_*.yaml; consumed by train.py:14-126): `model` (the
`create_latent_diffusion` kwargs), `dataset` (+ `dataset.train`: the latents dataloader kwargs), `optimizer`
(torch.optim.AdamW kwargs), `scheduler` (Composer's CosineAnnealingWithWarmup / Constant / ConstantWithWarmup), `algorithms.gradient_clipping`,
`algorithms.ema` (an EMA of the weights, ema.FlatEMA; the override `algorithms.ema=null` turns it off), `trainer` (max_duration, save/load options, device_train_microbatch_size), `seed`.  `${key}` / `${a.b}` interpolation
and `a.b=value` command-line overrides follow OmegaConf's surface for the subset the configs use.  What the hot path
does not cover is accepted and ignored with a note: loggers, the image-monitor callback,
`misc.compile`, `fsdp_config` (weights are replicated, gradients all-reduced -- train_step.GradReducer), and
`algorithms.low_precision_layernorm` (LayerNorm statistics are fp32 inside md_ln_fwd already).
"""
from __future__ import annotations

import argparse
import os
import re
from typing import Any, Dict, List, Optional

import torch
import yaml

_INTERP = re.compile(r"\$\{([^}]+)\}")


def _lookup(root: dict, dotted: str):
    node: Any = root
    for part in dotted.split("."):
        node = node[part]
    return node


def _resolve(node, root):
    if isinstance(node, dict):
        return {k: _resolve(v, root) for k, v in node.items()}
    if isinstance(node, list):
        return [_resolve(v, root) for v in node]
    if isinstance(node, str):
        m = _INTERP.fullmatch(node)
        if m:  # whole-value interpolation keeps the referenced type (seed: ${seed} stays an int)
            return _resolve(_lookup(root, m.group(1)), root)
        return _INTERP.sub(lambda mm: str(_resolve(_lookup(root, mm.group(1)), root)), node)
    return node


def apply_overrides(cfg: dict, overrides: List[str]) -> dict:
    for ov in overrides:
        if "=" not in ov:
            raise ValueError(f"override {ov!r} is not of the form a.b=value")
        key, val = ov.split("=", 1)
        node = cfg
        parts = key.split(".")
        for p in parts[:-1]:
            node = node.setdefault(p, {})
        node[parts[-1]] = yaml.safe_load(val)
    return cfg


def load_config(path: str, overrides: Optional[List[str]] = None) -> dict:
    with open(path) as f:
        cfg = yaml.safe_load(f)
    cfg = apply_overrides(cfg, overrides or [])
    return _resolve(cfg, cfg)


def ignored_sections(cfg: dict) -> List[str]:
    """Config entries that exist for Composer / Hydra machinery outside the hot path."""
    notes = []
    if cfg.get("logger"):
        notes.append("logger.* (Composer loggers)")
    for name, cb in (cfg.get("callbacks") or {}).items():
        if not str((cb or {}).get("_target_", "")).endswith("NaNCatcher"):
            notes.append(f"callbacks.{name}")
    if (cfg.get("algorithms") or {}).get("low_precision_layernorm"):
        notes.append("algorithms.low_precision_layernorm (already fp32 statistics in md_ln_fwd)")
    if (cfg.get("misc") or {}).get("compile"):
        notes.append("misc.compile (nothing to trace: the path is a fixed kernel sequence)")
    tr = cfg.get("trainer") or {}
    if tr.get("fsdp_config"):
        notes.append("trainer.fsdp_config (replicated weights + all-reduce of the flat gradient)")
    return notes


def trainer_kwargs(cfg: dict) -> Dict[str, Any]:
    """The Trainer arguments a config implies (pure function of the config: unit-testable without a GPU)."""
    opt = dict(cfg.get("optimizer") or {})
    target = str(opt.pop("_target_", "torch.optim.AdamW"))
    if not target.endswith("AdamW"):
        raise ValueError(f"only AdamW is implemented on the fused optimizer path, config asks for {target}")
    from .trainer import SCHEDULERS
    sched = dict(cfg.get("scheduler") or {})
    st = str(sched.pop("_target_", "composer.optim.CosineAnnealingWithWarmupScheduler")).split(".")[-1]
    if st not in SCHEDULERS:
        raise ValueError(f"unsupported scheduler {st} (known: {sorted(SCHEDULERS)})")
    clip = ((cfg.get("algorithms") or {}).get("gradient_clipping") or {})
    if clip and clip.get("clipping_type", "norm") != "norm":
        raise ValueError("only clipping_type: norm is implemented")
    tr = cfg.get("trainer") or {}
    betas = tuple(opt.get("betas", (0.9, 0.999)))
    return dict(
        max_duration=tr.get("max_duration", "1ba"), lr=float(opt.get("lr", 1e-3)), betas=(float(betas[0]), float(betas[1])),
        eps=float(opt.get("eps", 1e-8)), weight_decay=float(opt.get("weight_decay", 1e-2)),
        clip_norm=float(clip["clip_norm"]) if clip else None,
        scheduler=SCHEDULERS[st], t_warmup=sched.get("t_warmup", "0ba"), alpha_f=float(sched.get("alpha_f", 0.0)),
        alpha=float(sched.get("alpha", 1.0)),
        device_train_microbatch_size=int(tr.get("device_train_microbatch_size", 256)),
        save_folder=tr.get("save_folder"), save_interval=tr.get("save_interval", "1000000000ba"),
        load_path=tr.get("load_path"), load_weights_only=bool(tr.get("load_weights_only", False)),
        load_strict_model_weights=bool(tr.get("load_strict_model_weights", True)),
        load_ignore_keys=tuple(tr.get("load_ignore_keys") or ()),
        save_num_checkpoints_to_keep=tr.get("save_num_checkpoints_to_keep"),
        **ema_kwargs(cfg),
    )


_EMA_FIELDS = ("_target_", "half_life", "smoothing", "update_interval", "ema_start")


def ema_kwargs(cfg: dict) -> Dict[str, Any]:
    """`algorithms.ema` (configs/res_512_pretrain.yaml:3-9, any `_target_` ending in `.EMA`) as Trainer arguments;
    {} when the section is absent or null (`algorithms.ema=null` turns a config's EMA off).  What the trainer cannot
    honour raises: both or neither of half_life / smoothing, units other than batches, unknown fields."""
    ema = (cfg.get("algorithms") or {}).get("ema")
    if not ema:
        return {}
    target = str(ema.get("_target_", ""))
    if not target.endswith(".EMA"):
        raise ValueError(f"algorithms.ema: expected an EMA algorithm (_target_ ending in .EMA), got {target!r}")
    unknown = sorted(set(ema) - set(_EMA_FIELDS))
    if unknown:
        raise ValueError(f"algorithms.ema: unsupported fields {unknown}")
    hl, sm = ema.get("half_life"), ema.get("smoothing")
    if (hl is None) == (sm is None):
        raise ValueError("algorithms.ema: set exactly one of half_life and smoothing")
    from .trainer import parse_batches
    interval, start = ema.get("update_interval") or "1ba", ema.get("ema_start") or "0ba"
    for name, val in (("half_life", hl), ("update_interval", interval), ("ema_start", start)):
        if val is not None:
            try:
                parse_batches(val)
            except ValueError as e:
                raise ValueError(f"algorithms.ema.{name}: {e}") from None
    return dict(ema_smoothing=None if sm is None else float(sm), ema_half_life=hl, ema_update_interval=interval,
                ema_start=start)


def build(cfg: dict, device, rank: int = 0, world: int = 1, model=None):
    """(model, loader, Trainer) for a resolved config.  `model` may be injected (tests)."""
    from .data import DeviceBatchLoader, LatentsDataset
    from .models.model import create_latent_diffusion
    from .models.utils import text_encoder_embedding_format
    from .trainer import Trainer
    torch.manual_seed(int(cfg.get("seed", 0)))  # reproducibility.seed_all (train.py:23)
    mcfg = dict(cfg["model"])
    mcfg.pop("_target_", None)
    assert mcfg.get("precomputed_latents", True), \
        "For microbudget training, we assume that latents are already precomputed for all datasets"  # train.py:25
    if model is None:
        model = create_latent_diffusion(**mcfg).to(device)
    # Composer seeds every process with seed + global rank AFTER the identically-seeded model construction, so the ranks
    # draw different sigma / noise / patch masks (the replicas have no parameter broadcast and rely on the shared init)
    torch.manual_seed(int(cfg.get("seed", 0)) + int(rank))
    ds_cfg = cfg["dataset"]
    tr_cfg = dict(ds_cfg["train"])
    seq, dim = text_encoder_embedding_format(mcfg.get("text_encoder_name", "openclip:hf-hub:apple/DFN5B-CLIP-ViT-H-14-378"))
    ds = LatentsDataset(tr_cfg["datadir"], image_size=ds_cfg["image_size"], cap_seq_size=seq, cap_emb_dim=dim,
                        cap_drop_prob=ds_cfg.get("cap_drop_prob", 0.0))
    per_rank = int(ds_cfg["train_batch_size"]) // world  # train.py:50
    loader = DeviceBatchLoader(ds, per_rank, device, rank=rank, world=world, shuffle=bool(tr_cfg.get("shuffle", True)),
                               drop_last=bool(tr_cfg.get("drop_last", True)), seed=int(cfg.get("seed", 0)))
    kw = trainer_kwargs(cfg)
    ev_cfg = ds_cfg.get("eval")
    interval = (cfg.get("trainer") or {}).get("eval_interval", 0)
    if (cfg.get("misc") or {}).get("compile"):
        interval = 0  # train.py:99-101 disables online evals when misc.compile is set
    if ev_cfg and interval not in (None, 0, "0ba"):
        eds = LatentsDataset(ev_cfg["datadir"], image_size=ds_cfg["image_size"], cap_seq_size=seq, cap_emb_dim=dim)
        kw["eval_dataloader"] = DeviceBatchLoader(eds, int(ds_cfg.get("eval_batch_size", per_rank * world)) // world, device,
                                                  rank=rank, world=world, shuffle=False, drop_last=False,
                                                  seed=int(cfg.get("seed", 0)))
        kw["eval_interval"] = interval
    trainer = Trainer(model, loader, **kw)
    return model, loader, trainer


def main(argv: Optional[List[str]] = None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--config-path", default=".")
    ap.add_argument("--config-name", required=True)
    ap.add_argument("overrides", nargs="*", help="a.b=value (YAML-typed)")
    args = ap.parse_args(argv)
    name = args.config_name if args.config_name.endswith((".yaml", ".yml")) else args.config_name + ".yaml"
    cfg = load_config(os.path.join(args.config_path, name), args.overrides)
    import torch.distributed as dist
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    device = torch.device("cuda", local)
    torch.cuda.set_device(device)
    if world > 1:
        dist.init_process_group("nccl", device_id=device)
    if rank == 0:
        for note in ignored_sections(cfg):
            print(f"[micro_diffusion_b200.train] ignoring {note}")
    _, _, trainer = build(cfg, device, rank, world)
    if rank == 0 and trainer.ema is not None:
        e = trainer.ema
        print(f"[micro_diffusion_b200.train] EMA of the weights (smoothing {e.smoothing:.6g} every {e.update_interval} "
              f"batches) starts after batch {e.ema_start}")
    loss = trainer.fit()
    if world > 1:
        dist.destroy_process_group()
    return loss


if __name__ == "__main__":
    main()
