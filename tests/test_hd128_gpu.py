"""head_dim=128 on the GPU: every attention entry point at 128-wide heads against the CPU contract (oracle.emu_ops, as
tests/test_attn_tc_gpu.py), and DiT(head_dim=128) end to end -- the bf16 path and the high-precision mode against the
fixtures of the unmodified reference (tests/golden/hd128_*.pt), deterministic mode, the VJP, the CFG sampler against the
oracle sampler, and one training step plus sampling at the reference's default and MicroDiT_XL_2 widths."""
import gc

import pytest
import torch

from oracle import port, weights
from tests import dit_vjp_common as vc
from tests import hd128_common as hc
from tests import parity_common as pc

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
BF16 = torch.bfloat16
HD = 128
CASES = list(hc.HD128_CONFIGS)
rel = pc.rel_l2

# (B, H, Tq, Tk): key counts 64 / 77 / 120 / 256 / 1024, query counts 64 / 256 / 1024, ragged counts, grids of more
# than 132 CTAs, up to 16 heads (H * hd <= 2048: the generic backward's limit)
SHAPES = [(2, 2, 64, 64), (2, 3, 64, 77), (2, 2, 64, 120), (2, 2, 256, 256), (1, 2, 1024, 1024), (2, 3, 256, 77),
          (1, 2, 1024, 77), (2, 2, 256, 120), (2, 2, 1024, 256), (3, 2, 130, 33), (3, 2, 50, 200), (2, 3, 100, 1000),
          (40, 8, 64, 77), (64, 16, 64, 64), (4, 16, 256, 256), (1, 1, 64, 1024)]
FWD_ENTRIES = {"md_attn_fwd": None, "md_attn_fwd_mma": False, "md_attn_fwd_tc": True}
BWD_ENTRIES = {"md_attn_bwd": None, "md_attn_bwd_mma": False}


def _free():
    gc.collect()
    torch.cuda.empty_cache()


def _operands(B, H, Tq, Tk, seed, dtype=BF16):
    hsz = H * HD
    g = torch.Generator().manual_seed(seed)
    qkv = torch.randn(B * Tq, 3 * hsz + 64, generator=g).to(dtype)  # q a column slice of a wider buffer
    kv = torch.randn(B * Tk, 2 * hsz, generator=g).to(dtype)
    do = torch.randn(B * Tq, hsz, generator=g).to(dtype)
    return qkv, kv, do


def _ops(attn_tc=None, precision="bf16"):
    from micro_diffusion_b200.ops import CudaOps
    ops = CudaOps(torch.device(DEV), precision=precision)
    ops.attn_tc = attn_tc
    return ops


def _calls(ops):
    """Names of the C entry points an ops object calls."""
    names = []
    orig = ops._call

    def rec(name, *a, **k):
        names.append(name)
        return orig(name, *a, **k)
    ops._call = rec
    return names


# ------------------------------------------------------------------------------------------------ 1. kernels
@pytest.mark.parametrize("entry", list(FWD_ENTRIES))
@pytest.mark.parametrize("B,H,Tq,Tk", SHAPES)
def test_attn_fwd_matches_contract(entry, B, H, Tq, Tk):
    from oracle.emu_ops import EmuOps
    hsz = H * HD
    qkv, kv, _ = _operands(B, H, Tq, Tk, 1)
    o_ref = torch.zeros(B * Tq, hsz, dtype=BF16); lse_ref = torch.zeros(B, H, Tq)
    EmuOps("cpu").attn_fwd(qkv[:, :hsz], kv[:, :hsz], kv[:, hsz:], o_ref, lse_ref, B, H, Tq, Tk, HD)
    ops = _ops(FWD_ENTRIES[entry])
    names = _calls(ops)
    qd, kd = qkv.to(DEV), kv.to(DEV)
    o = torch.zeros(B * Tq, hsz, dtype=BF16, device=DEV); lse = torch.zeros(B, H, Tq, device=DEV)
    ops.attn_fwd(qd[:, :hsz], kd[:, :hsz], kd[:, hsz:], o, lse, B, H, Tq, Tk, HD)
    torch.cuda.synchronize()
    assert names == [entry]
    err = rel(o.cpu(), o_ref)
    print(f"\n[{entry} B={B} H={H} Tq={Tq} Tk={Tk}] o rel {err:.3e} lse maxabs {float((lse.cpu() - lse_ref).abs().max()):.3e}")
    assert err < 2e-2, err
    assert torch.allclose(lse.cpu(), lse_ref, atol=2e-3, rtol=1e-3)


@pytest.mark.parametrize("entry", list(BWD_ENTRIES))
@pytest.mark.parametrize("B,H,Tq,Tk", SHAPES)
def test_attn_bwd_matches_contract(entry, B, H, Tq, Tk):
    from oracle.emu_ops import EmuOps
    hsz = H * HD
    qkv, kv, do = _operands(B, H, Tq, Tk, 2)
    emu = EmuOps("cpu")
    o_ref = torch.zeros(B * Tq, hsz, dtype=BF16); lse_ref = torch.zeros(B, H, Tq)
    emu.attn_fwd(qkv[:, :hsz], kv[:, :hsz], kv[:, hsz:], o_ref, lse_ref, B, H, Tq, Tk, HD)
    dq_ref = torch.zeros(B * Tq, hsz, dtype=BF16); dkv_ref = torch.zeros(B * Tk, 2 * hsz, dtype=BF16)
    emu.attn_bwd(do, qkv[:, :hsz], kv[:, :hsz], kv[:, hsz:], o_ref, lse_ref, torch.zeros(B, H, Tq), dq_ref,
                 dkv_ref[:, :hsz], dkv_ref[:, hsz:], B, H, Tq, Tk, HD)
    ops = _ops(BWD_ENTRIES[entry])
    names = _calls(ops)
    qd, kd, dod, od, lsed = qkv.to(DEV), kv.to(DEV), do.to(DEV), o_ref.to(DEV), lse_ref.to(DEV)
    dq = torch.zeros(B * Tq, hsz, dtype=BF16, device=DEV); dkv = torch.zeros(B * Tk, 2 * hsz, dtype=BF16, device=DEV)
    ops.attn_bwd(dod, qd[:, :hsz], kd[:, :hsz], kd[:, hsz:], od, lsed, None, dq, dkv[:, :hsz], dkv[:, hsz:], B, H, Tq, Tk, HD)
    torch.cuda.synchronize()
    assert names == [entry]
    e = (rel(dq.cpu(), dq_ref), rel(dkv[:, :hsz].cpu(), dkv_ref[:, :hsz]), rel(dkv[:, hsz:].cpu(), dkv_ref[:, hsz:]))
    print(f"\n[{entry} B={B} H={H} Tq={Tq} Tk={Tk}] dq {e[0]:.3e} dk {e[1]:.3e} dv {e[2]:.3e}")
    assert max(e) < 2e-2, e


def test_wgmma_switch_keeps_its_meaning_at_128():
    """attn_tc = True: the wgmma forward (any Tk at hd 128) and, with no wgmma backward at 128, md_attn_bwd."""
    B, H, Tq, Tk = 2, 2, 64, 300
    hsz = H * HD
    qkv, kv, do = (t.to(DEV) for t in _operands(B, H, Tq, Tk, 3))
    ops = _ops(True)
    names = _calls(ops)
    o = torch.zeros(B * Tq, hsz, dtype=BF16, device=DEV); lse = torch.zeros(B, H, Tq, device=DEV)
    ops.attn_fwd(qkv[:, :hsz], kv[:, :hsz], kv[:, hsz:], o, lse, B, H, Tq, Tk, HD)
    dq = torch.zeros_like(o); dkv = torch.zeros(B * Tk, 2 * hsz, dtype=BF16, device=DEV)
    ops.attn_bwd(do, qkv[:, :hsz], kv[:, :hsz], kv[:, hsz:], o, lse, None, dq, dkv[:, :hsz], dkv[:, hsz:], B, H, Tq, Tk, HD)
    torch.cuda.synchronize()
    assert names == ["md_attn_fwd_tc", "md_attn_bwd"]


@pytest.mark.parametrize("B,H,Tq,Tk", [(2, 2, 64, 64), (2, 3, 64, 77), (1, 2, 256, 120), (3, 2, 130, 33), (1, 1, 64, 1024)])
def test_f32_attention_matches_contract(B, H, Tq, Tk):
    from oracle.emu_ops import EmuOps
    hsz = H * HD
    qkv, kv, do = _operands(B, H, Tq, Tk, 4, torch.float32)
    emu = EmuOps("cpu", exact=True)
    o_ref = torch.zeros(B * Tq, hsz); lse_ref = torch.zeros(B, H, Tq)
    emu.attn_fwd(qkv[:, :hsz], kv[:, :hsz], kv[:, hsz:], o_ref, lse_ref, B, H, Tq, Tk, HD)
    dq_ref = torch.zeros(B * Tq, hsz); dkv_ref = torch.zeros(B * Tk, 2 * hsz)
    emu.attn_bwd(do, qkv[:, :hsz], kv[:, :hsz], kv[:, hsz:], o_ref, lse_ref, torch.zeros(B, H, Tq), dq_ref,
                 dkv_ref[:, :hsz], dkv_ref[:, hsz:], B, H, Tq, Tk, HD)
    ops = _ops(precision="high")
    names = _calls(ops)
    qd, kd, dod = qkv.to(DEV), kv.to(DEV), do.to(DEV)
    o = torch.zeros(B * Tq, hsz, device=DEV); lse = torch.zeros(B, H, Tq, device=DEV)
    ops.attn_fwd(qd[:, :hsz], kd[:, :hsz], kd[:, hsz:], o, lse, B, H, Tq, Tk, HD)
    dq = torch.zeros_like(o); dkv = torch.zeros(B * Tk, 2 * hsz, device=DEV)
    ops.attn_bwd(dod, qd[:, :hsz], kd[:, :hsz], kd[:, hsz:], o, lse, torch.zeros(B, H, Tq, device=DEV), dq,
                 dkv[:, :hsz], dkv[:, hsz:], B, H, Tq, Tk, HD)
    torch.cuda.synchronize()
    assert names == ["md_attn_fwd_f32", "md_attn_bwd_f32"]
    e = (rel(o.cpu(), o_ref), rel(dq.cpu(), dq_ref), rel(dkv.cpu(), dkv_ref))
    print(f"\n[f32 B={B} H={H} Tq={Tq} Tk={Tk}] o {e[0]:.2e} dq {e[1]:.2e} dkv {e[2]:.2e}")
    assert max(e) < 1e-4, e
    assert torch.allclose(lse.cpu(), lse_ref, atol=1e-4, rtol=1e-5)


def test_other_head_widths_stay_unsupported():
    from micro_diffusion_b200._lib import MicroditLibraryError
    B, H, Tq, Tk, hd = 1, 2, 64, 64, 96
    x = torch.zeros(B * Tq, 3 * H * hd, dtype=BF16, device=DEV)
    o = torch.zeros(B * Tq, H * hd, dtype=BF16, device=DEV); lse = torch.zeros(B, H, Tq, device=DEV)
    for tc in (None, False, True):
        with pytest.raises(MicroditLibraryError, match="32, 64 or 128|head_dim 128"):
            _ops(tc).attn_fwd(x[:, :H * hd], x[:, H * hd:2 * H * hd], x[:, 2 * H * hd:], o, lse, B, H, Tq, Tk, hd)


# ------------------------------------------------------------------------------------------------ 2. DiT(head_dim=128)
def _high_ops(device):
    from micro_diffusion_b200.ops import CudaOps
    return CudaOps(device, precision="high")


@pytest.mark.parametrize("name", CASES)
def test_cuda_path_matches_oracle_and_golden(name):
    fx = hc.golden(name)
    loss, grads, den, ld = hc.product_run(name, device=DEV)
    ops = ld.dit.engine.ops
    assert ops.launches > 100 and not ops.is_emulation
    del ld
    _free()
    oloss, ograds, oden = hc.oracle_run(name)
    errs, med, worst = pc.grad_report(grads, ograds)
    amp_F = max(v["ref_amp_bf16"]["F"] for v in fx["vjp"].values())
    print(f"\n[{name}] loss cuda {loss:.6f} golden {fx['loss']:.6f} rel {abs(loss - fx['loss']) / fx['loss']:.2e} | "
          f"D_x relL2 {rel(den, fx['denoised_unmasked']):.2e} | grads median {med:.2e} worst {worst:.2e} ({errs[0][1]}) | "
          f"reference amp-bf16: loss {fx['ref_amp_bf16_loss_rel']:.2e} grads median {fx['ref_amp_bf16_grad_rel_median']:.2e}"
          f" worst {fx['ref_amp_bf16_grad_rel_max']:.2e} F {amp_F:.2e}")
    assert abs(oloss - fx["loss"]) / fx["loss"] < 1e-5
    assert abs(loss - fx["loss"]) / fx["loss"] < 3e-3
    assert rel(den, fx["denoised_unmasked"]) < max(1e-2, amp_F)
    assert med < 1.5 * fx["ref_amp_bf16_grad_rel_median"] + 5e-3
    assert worst < 2 * fx["ref_amp_bf16_grad_rel_max"] + 2e-2, errs[:5]


@pytest.mark.parametrize("name", CASES)
def test_high_precision_mode_meets_1e3(name):
    fx = hc.golden(name)
    loss, grads, den, ld = hc.product_run(name, ops_factory=_high_ops, device=DEV)
    assert ld.dit.engine.ops.prec == 1
    del ld
    _free()
    lrel, drel = abs(loss - fx["loss"]) / fx["loss"], rel(den, fx["denoised_unmasked"])
    errs = sorted((vc.fingerprint_error(k, grads[k], fp), k) for k, fp in fx["grads"].items())
    print(f"\n[{name} high] loss rel {lrel:.2e} D_x relL2 {drel:.2e} grad fingerprints worst {errs[-1][0]:.2e} ({errs[-1][1]})")
    assert lrel < 1e-3 and drel < 1e-3
    assert errs[-1][0] < 1e-3, errs[-3:]


def test_deterministic_mode_reproduces_a_step_bit_for_bit():
    from micro_diffusion_b200.train_step import FlatAdamW

    def one_step():
        _free()
        ld = hc.build_product("HS", device=DEV)
        ops = ld.dit.engine.ops
        ops.set_deterministic(True)
        try:
            opt = FlatAdamW(ld.dit, lr=1e-3, clip_norm=0.25)
            batch = {k: v.to(DEV) for k, v in weights.synth_batch(6, 4, 16, seed=5).items()}
            total = 0.0
            for i, s0 in enumerate(range(0, 6, 3)):
                torch.manual_seed(123 + i)
                loss = ld({k: v[s0:s0 + 3] for k, v in batch.items()})[0]
                (loss * 0.5).backward()
                total += float(loss.detach())
            g = ld.dit.store.grad.cpu()
            opt.step()
            torch.cuda.synchronize()
            return total, g, ld.dit.store.flat.cpu()
        finally:
            ops.set_deterministic(False)
            del ld

    l1, g1, w1 = one_step()
    l2, g2, w2 = one_step()
    assert l1 == l2 and torch.equal(g1, g2) and torch.equal(w1, w2)


@pytest.mark.parametrize("name,mr", [(n, mr) for n in CASES for mr in hc.VJP_MASKS[n]])
def test_vjp_within_reference_amp_class(name, mr):
    fx = hc.golden(name)["vjp"][mr]
    amp = fx["ref_amp_bf16"]
    net = hc.build_dit(name, device=DEV)
    x, t, y, dF, noise = hc.vjp_case(name, mr)
    if mr > 0:  # get_mask draws from the CUDA generator here: the oracle replays that draw
        noise = vc.mask_noise(x.shape[0], noise.shape[1], DEV).cpu()
    F, dx, dt, dy, grads = vc.product_vjp(net, *(v.to(DEV) for v in (x, t, y, dF)), mr)
    del net
    _free()
    oF, odx, odt, ody, ograds = hc.port_vjp(name, x, t, y, dF, mr, noise)
    if mr == 0:
        assert rel(oF, fx["F"]) < 1e-5 and rel(odx, fx["dx"]) < 1e-5
    errs, med, worst = pc.grad_report(grads, ograds)
    ie = {"F": rel(F, oF), "dx": rel(dx, odx), "dt": rel(dt, odt), "dy": rel(dy, ody)}
    print(f"\n[{name} VJP mask {mr}] {ie} grads median {med:.2e} worst {worst:.2e} | reference amp-bf16 {amp}")
    for k, e in ie.items():
        assert e < 2 * amp[k] + 2e-2, (k, e, amp[k])
    assert med < 1.5 * amp["grad_rel_median"] + 5e-3 and worst < 2 * amp["grad_rel_max"] + 2e-2, errs[:5]


@pytest.mark.parametrize("name", CASES)
def test_cfg_sampler_matches_the_oracle_sampler(name):
    """4 Heun steps at guidance 3 against the fp64-state oracle sampler: the high-precision mode to 1e-3; the bf16 path
    compounds its per-call deviation (D_x ~1e-2 above) through the steps and the 1 + 2 x 3 guidance gain."""
    steps, guidance = 4, 3.0
    c = hc.HD128_CONFIGS[name]
    ct = c["ctor"]
    g = torch.Generator().manual_seed(17)
    x = torch.randn(2, ct["in_channels"], ct["input_size"], ct["input_size"], generator=g)
    y = torch.randn(2, 1, 77, 1024, generator=g).half()
    P = weights.synth_state_dict(hc.template(name), seed=pc.WEIGHT_SEED)
    ref = port.edm_sampler(P, pc.port_config(c, ct), x, y.float(), steps, guidance).float()
    errs = {}
    for prec, ops_factory in (("bf16", None), ("high", _high_ops)):
        ld = hc.build_product(name, ops_factory=ops_factory, device=DEV)
        ld.eval()
        errs[prec] = rel(ld.edm_sampler_loop(x.to(DEV), y.to(DEV), steps=steps, cfg=guidance).float().cpu(), ref)
        del ld
        _free()
    print(f"\n[{name} sampler cfg {guidance}] relL2 vs oracle: bf16 {errs['bf16']:.2e} high {errs['high']:.2e}")
    assert errs["high"] < 1e-3 and errs["bf16"] < 5e-2, errs


@pytest.mark.parametrize("widths", ["DiT", "MicroDiT_XL_2"])
def test_full_width_models_train_one_step_and_sample(widths):
    from micro_diffusion_b200.arch import micro_dit_xl_2_kwargs
    from micro_diffusion_b200.models.dit import DiT
    from micro_diffusion_b200.models.model import LatentDiffusion, PrecomputedLatentStubs
    from micro_diffusion_b200.train_step import FlatAdamW
    _free()
    net = DiT(head_dim=128) if widths == "DiT" else DiT(**{**micro_dit_xl_2_kwargs(), "head_dim": 128})
    assert net.cfg.head_dim == 128 and all(b.attn_dim % 128 == 0 for b in net.cfg.all_blocks())
    net.load_state_dict(weights.synth_state_dict(net.state_dict(), seed=7))
    ld = LatentDiffusion(net.to(DEV), *PrecomputedLatentStubs.make(), train_mask_ratio=0.75, latent_res=32)
    ld.train()
    opt = FlatAdamW(ld.dit, lr=1e-4, clip_norm=0.25)
    batch = {k: v.to(DEV) for k, v in weights.synth_batch(4, 4, 32, seed=3).items()}
    torch.manual_seed(0)
    loss = ld(batch)[0]
    loss.backward()
    assert torch.isfinite(loss) and float(ld.dit.store.grad.abs().max()) > 0
    opt.step()
    ld.eval()
    g = torch.Generator(device=DEV).manual_seed(1)
    x = torch.randn(2, 4, 32, 32, device=DEV, generator=g)
    y = torch.randn(2, 1, 77, 1024, device=DEV, generator=g).half()
    out = ld.edm_sampler_loop(x, y, steps=2, cfg=3.0)
    print(f"\n[{widths} head_dim 128] loss {float(loss.detach()):.4f} sample std {float(out.float().std()):.3f}")
    assert torch.isfinite(out).all()
    del ld, opt, net
    _free()
