"""Kernel contracts of use_bias=True on the GPU: the bias of the fused SwiGLU epilogue (MD_EPI_SWIGLU) and
md_colsum_interleaved, against torch fp32 restatements in the interleaved layout (the metric of tests/test_kernels_gpu.py:
relative L2 plus a per-element ulp bound)."""
import pytest
import torch

from oracle.emu_ops import interleave_perm
from tests.test_kernels_gpu import BF16, DEV, F32, close, rnd

pytestmark = pytest.mark.gpu


def _ops():
    from micro_diffusion_b200.ops import CudaOps
    return CudaOps(DEV)


@pytest.mark.parametrize("M,f,K", [(512, 256, 128), (1000, 96, 192), (96, 64, 64), (300, 2816, 64), (77, 160, 256)])
def test_swiglu_epilogue_adds_the_natural_order_bias(M, f, K):
    """u = x W12^T + [b1 | b2] in the interleaved column order, h = silu(u1) * u2, with M and f not tile multiples."""
    ops = _ops()
    perm = interleave_perm(f)
    w12 = rnd((2 * f, K), 1, scale=K ** -0.5).to(BF16)
    b = rnd((2 * f,), 2, scale=0.5)
    x = rnd((M, K), 3, BF16)
    u = torch.zeros(M, 2 * f, dtype=BF16, device=DEV)
    h = torch.zeros(M, f, dtype=BF16, device=DEV)
    ops.gemm(x.to(DEV), w12[perm].contiguous().to(DEV), u, epi=6, C2=h, bias=b.to(DEV))
    # torch fp32 restatement: natural-order u, rounded to bf16 where the kernel stores it, then interleaved
    un = (x.float() @ w12.float().t() + b).to(BF16).float()
    close(u, un[:, perm], "swiglu u + bias")
    close(h, (torch.nn.functional.silu(un[:, :f]) * un[:, f:]).to(BF16), "swiglu hact with bias")


def test_swiglu_gradient_epilogue_still_rejects_a_bias():
    from micro_diffusion_b200._lib import MicroditLibraryError
    ops = _ops()
    dy = torch.zeros(128, 64, dtype=BF16, device=DEV)
    w3t = torch.zeros(64, 64, dtype=BF16, device=DEV)
    u = torch.zeros(128, 128, dtype=BF16, device=DEV)
    with pytest.raises(MicroditLibraryError, match="no bias"):
        ops.gemm(dy, w3t, torch.zeros_like(u), epi=7, aux=u, bias=torch.zeros(64, device=DEV))


@pytest.mark.parametrize("rows,f,dtype", [(1000, 96, BF16), (4096, 2816, BF16), (231, 256, F32), (64, 32, BF16)])
def test_colsum_interleaved_matches_torch_fast_and_deterministic(rows, f, dtype):
    ops = _ops()
    x = rnd((rows, 2 * f), 5, dtype).to(DEV)
    base = rnd((2 * f,), 6)
    ref = base + x.float().cpu().sum(0)[torch.argsort(interleave_perm(f))]
    out = base.to(DEV)
    ops.colsum_interleaved(x, out, f)
    close(out, ref, "colsum_interleaved (fast)", 1e-4)
    ops.set_deterministic(True, workspace_bytes=64 << 20)
    try:
        outs = []
        for _ in range(2):
            o = base.to(DEV)
            ops.colsum_interleaved(x, o, f)
            outs.append(o.cpu())
        torch.cuda.synchronize()
    finally:
        ops.set_deterministic(False)
    assert torch.equal(outs[0], outs[1])
    close(outs[0], ref, "colsum_interleaved (deterministic)", 1e-4)
