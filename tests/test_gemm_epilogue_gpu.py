"""GEMM epilogue tails on interior and edge tiles against the CPU contract (oracle.emu_ops.EmuOps) or a torch
restatement.  Interior tiles (the whole 128 x BLOCK_N tile inside the output) run an unguarded tail that loads its side
inputs in batches ahead of the stores; edge tiles keep the per-pair guarded tail.  The shapes put only interior tiles,
or interior and edge tiles together, into one launch at tile widths 256 and 128: through the checks of the GEMM tests
in test_kernels_gpu.py, and for the residual tail writing in place over its own residual and the bias of the bf16 store
and of the fused SwiGLU forward."""
import pytest
import torch

from tests import test_kernels_gpu as tk
from tests.test_kernels_gpu import BF16, DEV, both, close, rnd

pytestmark = pytest.mark.gpu

@pytest.mark.parametrize("layout,M,N,K,epi", [
    (0, 4352, 1024, 64, 1),   # f32 + bias, 256-wide tiles, all interior
    (0, 4352, 1024, 64, 2),   # residual + gate + res_mod + bias + C2, all interior
    (0, 4400, 1000, 64, 2),   # the same, interior and edge tiles
    (0, 4352, 1024, 64, 4),   # GELU dual store + bias, all interior
    (0, 4400, 1000, 64, 4),   # the same, interior and edge tiles
])
def test_gemm_via_ops_interior_tiles(layout, M, N, K, epi):
    tk.test_gemm_via_ops(layout, M, N, K, epi)


@pytest.mark.parametrize("M,N,K,batch,ld_extra", [
    (4352, 1024, 64, 1, 0),      # 256-wide tiles, every tile interior
    (4400, 1000, 64, 1, 0),      # 256-wide tiles, interior and edge tiles in one launch
    (1024, 512, 128, 17, 0),     # batched, 256-wide interior tiles
])
@pytest.mark.parametrize("act", [0, 1])
def test_gemm_activation_epilogues_interior_tiles(M, N, K, batch, ld_extra, act):
    tk.test_gemm_activation_epilogues(M, N, K, batch, ld_extra, act)


@pytest.mark.parametrize("M,f,K", [
    (4352, 512, 64),   # interior tiles only: 256 wide forward, 128 wide backward
    (4400, 992, 64),   # 256-wide tiles, interior and edge tiles mixed
])
def test_gemm_swiglu_epilogues_interior_tiles(M, f, K):
    tk.test_gemm_swiglu_epilogues(M, f, K)


# (M, N): 256-wide tiles all interior, 256-wide interior + edge, 128-wide all interior, 128-wide interior + edge
SHAPES = [(4352, 1024), (4400, 1000), (512, 768), (600, 768)]


@pytest.mark.parametrize("M,N", SHAPES)
def test_gemm_residual_in_place_with_gate(M, N):
    """C = C + gate * (A B^T + bias) with res = C (the stacked K/V backward's accumulation), plus the bf16 side copy;
    res_mod = M keeps every row reading its own residual row."""
    K, T = 64, 64 if M % 64 == 0 else M
    A = rnd((M, K), 1, BF16); B = rnd((N, K), 2, BF16)
    bias = rnd((N,), 3); gate = rnd((M // T, 2 * N), 5); Cm = rnd((M, N), 4); C2 = torch.zeros(M, N, dtype=BF16)

    def run(o, A, B, Cm, C2, bias, gate):
        o.gemm(A, B, Cm, epi=2, C2=C2, bias=bias, res=Cm, res_mod=M, gate=gate[:, N:], rows_per_gate=T)
    cpu, cu = both(run, [A, B, Cm, C2, bias, gate])
    close(cu[2], cpu[2], "in-place residual", 1e-4); close(cu[3], cpu[3], "in-place residual C2")


@pytest.mark.parametrize("M,N", SHAPES)
def test_gemm_bf16_store_with_bias(M, N):
    K = 64
    A = rnd((M, K), 1, BF16); B = rnd((N, K), 2, BF16); bias = rnd((N,), 3); Cm = torch.zeros(M, N, dtype=BF16)
    cpu, cu = both(lambda o, A, B, Cm, bias: o.gemm(A, B, Cm, epi=0, bias=bias), [A, B, Cm, bias])
    close(cu[2], cpu[2], "bf16 store + bias")


@pytest.mark.parametrize("M,f", [(4352, 512), (4400, 992), (512, 384), (600, 384)])
def test_gemm_swiglu_with_bias(M, f):
    """MD_EPI_SWIGLU with the natural-order [b1 | b2] bias on the interleaved weight stack, against a torch fp32
    restatement rounded to bf16 where the kernel stores."""
    from micro_diffusion_b200.ops import CudaOps
    from oracle.emu_ops import interleave_perm
    K, perm = 64, interleave_perm(f)
    x = rnd((M, K), 1, BF16); w12 = rnd((2 * f, K), 2, scale=K ** -0.5).to(BF16); b = rnd((2 * f,), 3, scale=0.5)
    u = torch.zeros(M, 2 * f, dtype=BF16, device=DEV); h = torch.zeros(M, f, dtype=BF16, device=DEV)
    CudaOps(DEV).gemm(x.to(DEV), w12[perm].contiguous().to(DEV), u, epi=6, C2=h, bias=b.to(DEV))
    un = (x.float() @ w12.float().t() + b).to(BF16).float()
    close(u, un[:, perm], "swiglu u + bias")
    close(h, (torch.nn.functional.silu(un[:, :f]) * un[:, f:]).to(BF16), "swiglu hact + bias")
