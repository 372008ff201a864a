"""Python face of the C ABI: every method takes torch CUDA tensors (device memory + strides are the only
thing torch provides here), checks dtypes/contiguity, and forwards raw pointers and sizes to
libmicrodit_b200.so on the current CUDA stream.  No method computes anything in PyTorch and there is no
fallback: a missing library or a failing call raises `MicroditLibraryError`.

The engine (`engine.py`) is written against this interface; `oracle/emu_ops.py` (test infrastructure)
implements the same interface on CPU tensors so the host-side orchestration can be tested without a GPU.
"""
from __future__ import annotations

import ctypes as C
import os

import torch

from . import _lib
from ._lib import GemmArgs, MicroditLibraryError

NT, TN = 0, 1
EPI_BF16, EPI_F32, EPI_RESID, EPI_ATOMIC, EPI_ACT_DUAL, EPI_ACT_GRAD, EPI_SWIGLU, EPI_SWIGLU_GRAD = 0, 1, 2, 3, 4, 5, 6, 7
ACT_GELU_ERF, ACT_GELU_TANH = 0, 1

_I64 = C.c_int64
_F = C.c_float
_P = C.c_void_p
_I = C.c_int
_D = C.c_double

_PROTOS = {
    "md_ln_fwd": [_P, _I, _P, _P, _P, _P, _P, _P, _P, _I64, _I64, _P, _P, _P, _I64, _I64, _F, _I, _P],
    "md_ln_bwd": [_P, _P, _I, _P, _P, _P, _I64, _I64, _P, _P, _P, _I, _P, _P, _P, _P, _P, _P, _P, _I64, _I64, _I, _P],
    "md_rownorm_fwd": [_P, _I64, _P, _I64, _I64, _I64, _F, _I, _P],
    "md_rownorm_bwd": [_P, _I64, _P, _I64, _P, _I64, _I64, _I64, _I, _P],
    "md_gate_bwd": [_P, _P, _P, _I64, _I64, _P, _P, _I64, _I64, _I, _P],
    "md_attn_fwd": [_P, _I64, _P, _I64, _P, _I64, _P, _I64, _P, _I64, _I64, _I64, _I64, _I64, _P],
    "md_attn_fwd_tc": [_P, _I64, _P, _I64, _P, _I64, _P, _I64, _P, _I64, _I64, _I64, _I64, _I64, _P],
    "md_attn_bwd_tc": [_P, _I64, _P, _I64, _P, _I64, _P, _I64, _P, _I64, _P, _P, _P, _I64, _P, _I64, _P, _I64,
                       _I64, _I64, _I64, _I64, _I64, _P],
    "md_attn_fwd_mma": [_P, _I64, _P, _I64, _P, _I64, _P, _I64, _P, _I64, _I64, _I64, _I64, _I64, _P],
    "md_attn_bwd_mma": [_P, _I64, _P, _I64, _P, _I64, _P, _I64, _P, _I64, _P, _P, _P, _I64, _P, _I64, _P, _I64,
                        _I64, _I64, _I64, _I64, _I64, _P],
    "md_attn_fwd_f32": [_P, _I64, _P, _I64, _P, _I64, _P, _I64, _P, _I64, _I64, _I64, _I64, _I64, _P],
    "md_attn_bwd_f32": [_P, _I64, _P, _I64, _P, _I64, _P, _I64, _P, _I64, _P, _P, _P, _I64, _P, _I64, _P, _I64,
                        _I64, _I64, _I64, _I64, _I64, _P],
    "md_split3_bf16": [_P, _I64, _I64, _P, _I64, _I64, _I64, _I, _I, _P],
    "md_attn_bwd": [_P, _I64, _P, _I64, _P, _I64, _P, _I64, _P, _I64, _P, _P, _P, _I64, _P, _I64, _P, _I64,
                    _I64, _I64, _I64, _I64, _I64, _P],
    "md_swiglu_fwd": [_P, _P, _I64, _I64, _I, _P],
    "md_swiglu_bwd": [_P, _P, _P, _I64, _I64, _I, _P],
    "md_act_fwd": [_P, _P, _I64, _I, _I, _P],
    "md_act_bwd": [_P, _P, _P, _I64, _I, _I, _P],
    "md_gelu_tanh_f32_fwd": [_P, _P, _I64, _I, _P],
    "md_gelu_tanh_f32_bwd": [_P, _P, _P, _I, _I64, _P],
    "md_moe_gate_fwd": [_P, _P, _P, _I64, _I64, _I64, _I, _P],
    "md_moe_topk": [_P, _P, _P, _P, _I64, _I64, _I64, _I64, _P],
    "md_moe_gather": [_P, _P, _P, _I64, _I64, _I64, _I64, _I64, _I, _P],
    "md_moe_combine_fwd": [_P, _P, _P, _P, _P, _I64, _P, _P, _I64, _I64, _I64, _I64, _I64, _I, _P],
    "md_moe_combine_bwd": [_P, _P, _P, _P, _P, _P, _I64, _I64, _I64, _I64, _I64, _I, _P],
    "md_moe_dx_bwd": [_P, _P, _P, _P, _P, _P, _P, _I64, _I64, _I64, _I64, _I64, _I, _P],
    "md_moe_gate_wgrad": [_P, _P, _P, _I64, _I64, _I64, _I, _P],
    "md_mask_sort": [_P, _P, _P, _P, _P, _I64, _I64, _I64, _P],
    "md_gather_rows_f32": [_P, _P, _P, _I64, _I64, _P],
    "md_scatter_rows_f32": [_P, _P, _P, _I64, _I64, _P],
    "md_cond_prepare": [_P, _P, _P, _P, _I64, _I64, _I, _P],
    "md_patchify": [_P, _P, _P, _I64, _I64, _I64, _I64, _I64, _I, _P],
    "md_edm_prepare": [_P, _I, _P, _P, _P, _F, _F, _F, _P, _P, _P, _I64, _I64, _I64, _I64, _I64, _I, _P],
    "md_timestep_embed": [_P, _P, _I64, _I64, _I, _P],
    "md_edm_loss_fwd": [_P, _P, _P, _I, _P, _P, _P, _P, _I64, _I64, _I64, _I64, _I64, _I64, _P],
    "md_edm_loss_bwd": [_P, _P, _P, _I, _P, _P, _P, _P, _I64, _I64, _I64, _I64, _I64, _I64, _I, _P],
    "md_edm_output": [_P, _P, _P, _P, _P, _P, _P, _I64, _I64, _I64, _I64, _I64, _I64, _P],
    "md_edm_heun": [_I, _P, _P, _P, _P, _P, _P, _P, _P, _P, _I64, _I64, _I64, _I64, _D, _P],
    "md_edm_output_cfg": [_P, _P, _P, _P, _P, _F, _F, _I64, _I64, _I64, _I64, _I64, _P],
    "md_unpatchify_bwd": [_P, _P, _P, _I64, _I64, _I64, _I64, _I64, _I64, _I, _P],
    "md_patchify_bwd": [_P, _P, _P, _I64, _I64, _I64, _I64, _I64, _I, _P],
    "md_timestep_embed_bwd": [_P, _P, _P, _I64, _I64, _I, _P],
    "md_mean_tokens_fwd": [_P, _P, _I64, _I64, _I64, _I, _P],
    "md_mean_tokens_bwd": [_P, _P, _I64, _I64, _I64, _P],
    "md_cast_f32_bf16": [_P, _P, _I64, _I, _P],
    "md_colsum": [_P, _I, _I64, _P, _I64, _I64, _P],
    "md_colsum_interleaved": [_P, _I, _I64, _P, _I64, _I64, _I64, _P],
    "md_cast_transpose": [_P, _P, _P, _I64, _I64, _I64, _I64, _I, _P],
    "md_cast_transpose_multi": [_P, _P, _P, _P, _I64, _I64, _I, _P],
    "md_set_deterministic": [_P, _I64],
    "md_sumsq": [_P, _P, _I64, _P],
    "md_adamw": [_P, _P, _P, _P, _P, _F, _F, _F, _F, _F, _F, _I64, _P, _I64, _P],
    "md_adamw_ema": [_P, _P, _P, _P, _P, _F, _F, _F, _F, _F, _F, _I64, _P, _F, _P, _I64, _P],
    "md_swap_f32": [_P, _P, _I64, _P],
}

_TAKES_PREC = frozenset(['md_ln_fwd', 'md_ln_bwd', 'md_rownorm_fwd', 'md_rownorm_bwd', 'md_gate_bwd', 'md_swiglu_fwd', 'md_swiglu_bwd', 'md_act_fwd', 'md_act_bwd', 'md_gelu_tanh_f32_fwd', 'md_moe_gate_fwd', 'md_moe_gather', 'md_moe_combine_fwd', 'md_moe_combine_bwd', 'md_moe_dx_bwd', 'md_moe_gate_wgrad', 'md_cond_prepare', 'md_edm_prepare', 'md_patchify', 'md_timestep_embed', 'md_edm_loss_bwd', 'md_unpatchify_bwd', 'md_patchify_bwd', 'md_timestep_embed_bwd', 'md_mean_tokens_fwd', 'md_cast_f32_bf16', 'md_cast_transpose', 'md_cast_transpose_multi'])

EXPORTED_SYMBOLS = ["md_last_error", "md_abi_version", "md_gemm_bf16", *_PROTOS.keys()]


def _ptr(t):
    return None if t is None else t.data_ptr()


_DET_WORKSPACE = {}  # the deterministic-mode scratch registered with the library (md_set_deterministic), kept alive here


def _mod(t):
    """(pointer, row pitch) of a per-sample modulation view [samples, D] (a column slice of the adaLN buffer)."""
    if t is None:
        return None, 0
    assert t.dim() == 2 and t.stride(1) == 1 and t.dtype == torch.float32
    return t.data_ptr(), t.stride(0)


class CudaOps:
    """Launches the sm_90a kernels.  One instance per device."""

    is_emulation = False

    def __init__(self, device, precision=None):
        """precision: "bf16" (default; the product path) or "high" (MD_PRECISION=high): GEMM operands / saved activations
        stay fp32, every GEMM runs as a 3-way bf16 split on the same wgmma kernel, attention in plain fp32 -- the mode
        the 1e-3 parity gate of north_star is taken in (tests/test_parity_gpu.py)."""
        self.device = torch.device(device)
        precision = precision or os.environ.get("MD_PRECISION", "bf16")
        if precision not in ("bf16", "high"):
            raise ValueError(f"MD_PRECISION must be 'bf16' or 'high', got {precision!r}")
        self.precision = precision
        self.prec = 1 if precision == "high" else 0
        self.lowp_dtype = torch.float32 if self.prec else torch.bfloat16
        if self.device.type != "cuda":
            raise MicroditLibraryError("the MicroDiT hot path runs on an H100 (CUDA) device only; there is no CPU path")
        self.lib = _lib.load()
        for name, argtypes in _PROTOS.items():
            fn = getattr(self.lib, name)
            fn.restype = C.c_int
            fn.argtypes = argtypes
        self.launches = 0
        self.poison_kinds = os.environ.get("MD_DEBUG_POISON", "0")
        self.poison = self.poison_kinds != "0"
        self._det_ws = None
        if os.environ.get("MD_DETERMINISTIC", "0") == "1":
            self.set_deterministic(True)
        self.gemm_flops = 0      # algorithmic FLOPs of every md_gemm_bf16 launched (2*M*N*K*batch)
        # None: md_attn_fwd chooses the forward kernel per shape; True: the wgmma kernel (md_attn_fwd_tc) wherever its
        # envelope allows (head_dim 64 with Tk <= 256, or head_dim 128) and the wgmma backward (md_attn_bwd_tc, head_dim
        # 64; head_dim 128 has none and takes md_attn_bwd); False: the mma.sync kernels (md_attn_fwd_mma /
        # md_attn_bwd_mma), for A/B runs.
        self.attn_tc = None
        self.sm_limit = 0        # > 0: persistent GEMM grids use at most this many SMs (set while a collective overlaps)
        self.profile = None      # set to a list to record (name, start_event, end_event, flops) per launch

    # ------------------------------------------------------------------ helpers
    def _stream(self):
        return torch.cuda.current_stream(self.device).cuda_stream

    def _call(self, name, *args, label=None, flops=0):
        if name in _TAKES_PREC:
            args = (*args, self.prec)
        prof = self.profile
        if prof is not None:
            e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
            e0.record()
        rc = getattr(self.lib, name)(*args, self._stream())
        if prof is not None:
            e1.record()
            prof.append((name + (" " + label if label else ""), e0, e1, flops))
        self.launches += 1
        if rc != 0:
            raise MicroditLibraryError(f"{name} failed ({rc}): {self.lib.md_last_error().decode()}")

    def set_deterministic(self, on: bool = True, workspace_bytes: int = 1 << 30):
        """Deterministic mode of the library (include/microdit_b200.h: md_set_deterministic): every cross-block floating-point
        atomic accumulation goes through per-block partials in a workspace and a fixed-order reduction, so identical inputs
        give bit-identical gradients and weights (MD_DETERMINISTIC=1 turns it on at construction).  Process-wide switch."""
        if on:
            ws = _DET_WORKSPACE.get("ws")
            if ws is None or ws.numel() < workspace_bytes or ws.device != self.device:
                ws = torch.empty(workspace_bytes, dtype=torch.uint8, device=self.device)
            ws.fill_(0xFF)   # NaN pattern: a reduction that read a partial nobody wrote would show up at once
            rc = self.lib.md_set_deterministic(ws.data_ptr(), ws.numel())
            # the library keeps the pointer (process-wide switch): the buffer must outlive this CudaOps instance
            _DET_WORKSPACE["ws"] = ws
            self._det_ws = ws
        else:
            rc = self.lib.md_set_deterministic(None, 0)
            torch.cuda.synchronize(self.device)   # no launch may still be writing partials when the buffer is released
            _DET_WORKSPACE.pop("ws", None)
            self._det_ws = None
        if rc != 0:
            raise MicroditLibraryError(f"md_set_deterministic failed ({rc}): {self.lib.md_last_error().decode()}")

    def profile_summary(self):
        """{op: (launches, total_ms, flops)} from the recorded events (call after torch.cuda.synchronize())."""
        out = {}
        for name, e0, e1, fl in self.profile or []:
            n, ms, f = out.get(name, (0, 0.0, 0))
            out[name] = (n + 1, ms + e0.elapsed_time(e1), f + fl)
        return out

    def empty(self, shape, dtype):
        if self.prec and dtype == torch.bfloat16:
            dtype = torch.float32
        if self.poison and self.poison_kinds in ("1", {torch.bfloat16: "bf16", torch.float32: "f32"}.get(dtype, "int")):
            # MD_DEBUG_POISON=1|bf16|f32|int: scratch / output buffers start as NaN (-1 for indices), so that a kernel reading
            # an element nobody wrote cannot go unnoticed (tools/det_diag_s.py --poison)
            return torch.full(shape, float("nan") if dtype.is_floating_point else -1, dtype=dtype, device=self.device)
        return torch.empty(shape, dtype=dtype, device=self.device)

    def zeros(self, shape, dtype):
        if self.prec and dtype == torch.bfloat16:
            dtype = torch.float32
        return torch.zeros(shape, dtype=dtype, device=self.device)

    # ------------------------------------------------------------------ GEMM
    def _split3(self, x, role, along):
        """fp32 operand -> bf16 [hi | lo | hi] (role 0) or [hi | hi | lo] (role 1) stacked along the contraction."""
        x3 = x if x.dim() == 3 else x.unsqueeze(0)
        assert x3.dtype == torch.float32 and x3.stride(2) == 1
        b, r, c = x3.shape
        out = torch.empty((b, r, 3 * c) if along == 0 else (b, 3 * r, c), dtype=torch.bfloat16, device=self.device)
        self._call("md_split3_bf16", x3.data_ptr(), x3.stride(1), x3.stride(0), out.data_ptr(), b, r, c, role, along)
        return out if x.dim() == 3 else out[0]

    def gemm(self, A, B, Cm, *, layout=NT, epi=EPI_BF16, C2=None, bias=None, res=None, gate=None, rows_per_gate=0,
             res_mod=0, splits=1, act=0, alpha=1.0, aux=None, row_interleave=0):
        if self.prec:
            assert epi not in (EPI_SWIGLU, EPI_SWIGLU_GRAD) and not row_interleave, "fused SwiGLU is a bf16-mode layout"
            # high precision: the same wgmma kernel at 3x the contraction depth over bf16 (hi, lo) splits of the fp32
            # operands; outputs stay fp32 (the bf16-store epilogues become fp32 stores, the fused activation a second pass)
            along = 0 if layout == NT else 1
            A3, B3 = self._split3(A, 0, along), self._split3(B, 1, along)
            if epi == EPI_ACT_DUAL:
                self._gemm_lowp(A3, B3, Cm, layout=layout, epi=EPI_F32, bias=bias, alpha=alpha)
                self.act_fwd(Cm, C2, act)
                return
            if epi == EPI_ACT_GRAD:
                tmp = torch.empty_like(Cm)
                self._gemm_lowp(A3, B3, tmp, layout=layout, epi=EPI_F32, alpha=alpha)
                self.act_bwd(tmp, aux, Cm, act)
                return
            if epi == EPI_RESID and C2 is not None:
                raise MicroditLibraryError("high-precision GEMM: the bf16 side copy of the residual epilogue is not available")
            self._gemm_lowp(A3, B3, Cm, layout=layout, epi=EPI_F32 if epi == EPI_BF16 else epi, bias=bias, res=res,
                            gate=gate, rows_per_gate=rows_per_gate, res_mod=res_mod, splits=splits, alpha=alpha)
            return
        self._gemm_lowp(A, B, Cm, layout=layout, epi=epi, C2=C2, bias=bias, res=res, gate=gate,
                        rows_per_gate=rows_per_gate, res_mod=res_mod, splits=splits, act=act, alpha=alpha, aux=aux,
                        row_interleave=row_interleave)

    def _gemm_lowp(self, A, B, Cm, *, layout=NT, epi=EPI_BF16, C2=None, bias=None, res=None, gate=None, rows_per_gate=0,
                   res_mod=0, splits=1, act=0, alpha=1.0, aux=None, row_interleave=0):
        a = GemmArgs()
        batched = A.dim() == 3
        A3, B3, C3 = (A, B, Cm) if batched else (A.unsqueeze(0), B.unsqueeze(0), Cm.unsqueeze(0))
        assert A3.dtype == torch.bfloat16 and B3.dtype == torch.bfloat16
        assert A3.stride(2) == 1 and B3.stride(2) == 1 and C3.stride(2) == 1
        if layout == NT:
            M, K = A3.shape[1], A3.shape[2]
            N = B3.shape[1]
            assert B3.shape[2] == K
        else:
            K, M = A3.shape[1], A3.shape[2]
            N = B3.shape[2]
            assert B3.shape[1] == K
        # the SwiGLU backward epilogue turns the N = f columns of d h into the 2f interleaved columns of d u
        assert C3.shape[1] == M and C3.shape[2] == (2 * N if epi == EPI_SWIGLU_GRAD else N), (C3.shape, M, N)
        a.A, a.B, a.C, a.C2 = A3.data_ptr(), B3.data_ptr(), C3.data_ptr(), _ptr(C2)
        a.bias, a.res, a.aux = _ptr(bias), _ptr(res), _ptr(aux)
        a.M, a.N, a.K = M, N, K
        a.lda, a.ldb, a.ldc = A3.stride(1), B3.stride(1), C3.stride(1)
        a.batch = A3.shape[0]
        a.strideA, a.strideB, a.strideC = A3.stride(0), B3.stride(0), C3.stride(0)
        # [batch, N]: one bias per batch entry; [N]: one bias shared by every batch entry (stride 0)
        a.strideBias = bias.stride(0) if (bias is not None and bias.dim() == 2) else 0
        a.gate, a.ldgate = _mod(gate)
        a.rows_per_gate = rows_per_gate
        a.res_mod = res_mod
        a.layout, a.epilogue, a.splits, a.act, a.alpha = layout, epi, splits, act, alpha
        a.sm_limit = self.sm_limit
        a.row_interleave = row_interleave
        a.ldc2 = a.strideC2 = 0
        if epi == EPI_SWIGLU:
            assert C2 is not None and C2.dtype == torch.bfloat16 and C2.shape[-1] == N // 2 and C2.stride(-1) == 1
            # the bias is the natural-order [b1 | b2] vector; the epilogue maps it onto the interleaved columns
            assert bias is None or (bias.dtype == torch.float32 and bias.shape[-1] == N and bias.stride(-1) == 1)
            a.ldc2 = C2.stride(-2)
            a.strideC2 = C2.stride(0) if C2.dim() == 3 else 0
        elif C2 is not None:
            # the kernel writes C2 at C's offsets (batch stride, row pitch): any other layout lands in the wrong place
            assert C2.shape == Cm.shape and C2.stride() == Cm.stride(), (C2.shape, C2.stride(), Cm.shape, Cm.stride())
        if aux is not None:
            assert aux.dtype == torch.bfloat16 and aux.shape == Cm.shape and aux.stride() == Cm.stride()
        if res is not None:
            assert res.dtype == torch.float32 and res.stride(-1) == 1 and res.stride(-2) == C3.stride(1)
        want = torch.bfloat16 if epi in (EPI_BF16, EPI_ACT_DUAL, EPI_ACT_GRAD, EPI_SWIGLU, EPI_SWIGLU_GRAD) else torch.float32
        assert Cm.dtype == want, (Cm.dtype, epi)
        flops = 2 * M * N * K * int(a.batch)
        self.gemm_flops += flops
        prof = self.profile
        if prof is not None:
            e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
            e0.record()
        rc = self.lib.md_gemm_bf16(C.byref(a), self._stream())
        if prof is not None:
            e1.record()
            prof.append((f"md_gemm_bf16/{'tn' if layout == TN else 'nt'} M={M} N={N} K={K} b={int(a.batch)} epi={epi} s={splits}", e0, e1, flops))
        self.launches += 1
        if rc != 0:
            raise MicroditLibraryError(f"md_gemm_bf16 failed ({rc}): {self.lib.md_last_error().decode()} "
                                       f"[M={M} N={N} K={K} layout={layout} epi={epi}]")

    # ------------------------------------------------------------------ norms
    def ln_fwd(self, x, y, mean, rstd, *, gamma=None, shift=None, scale=None, T, src_rows=None, eps=1e-6,
               y_add=None, gate_add=None, x_new=None):
        rows, D = y.shape
        sh, ld1 = _mod(shift)
        sc, ld2 = _mod(scale)
        ga, ld3 = _mod(gate_add)
        self._call("md_ln_fwd", x.data_ptr(), int(x.dtype == torch.bfloat16), _ptr(src_rows), _ptr(y_add), ga,
                   _ptr(x_new), _ptr(gamma), sh, sc, ld1 or ld2 or ld3, T, y.data_ptr(), _ptr(mean), _ptr(rstd), rows,
                   D, eps)

    def ln_bwd(self, dy, x, mean, rstd, *, gamma=None, scale=None, T, src_rows=None, dx=None, dx_mode=0,
               dgamma=None, dshift=None, dscale=None, dy_next=None, y_next=None, gate_next=None, dgate_next=None):
        """dy_next (bf16 [rows, D]): also emit the next branch's gated-residual backward from the updated dx
        (dy_next = gate_next * dx, dgate_next += sum_t dx * y_next) -- what a separate gate_bwd pass would compute."""
        rows, D = dy.shape
        sc, ld = _mod(scale)
        dsh, ld2 = _mod(dshift)
        dsc, ld3 = _mod(dscale)
        gn, ld4 = _mod(gate_next)
        dgn, ld5 = _mod(dgate_next)
        lds = {v for v in (ld, ld2, ld3, ld4, ld5) if v}
        assert len(lds) <= 1, "all per-sample vectors of one call are views of the same modulation buffer"
        self._call("md_ln_bwd", dy.data_ptr(), x.data_ptr(), int(x.dtype == torch.bfloat16), _ptr(src_rows),
                   _ptr(gamma), sc, lds.pop() if lds else 0, T, mean.data_ptr(), rstd.data_ptr(), _ptr(dx), dx_mode,
                   _ptr(dgamma), dsh, dsc, _ptr(y_next), gn, dgn, _ptr(dy_next), rows, D)

    def rownorm_fwd(self, x, rstd, eps=1e-6, nslice=1):
        """x [rows, nslice*W]: every W-wide slice normalised on its own; rstd [nslice, rows] ([rows] for one slice)."""
        rows, W = x.shape[0], x.shape[1] // nslice
        assert rstd.numel() == nslice * rows and x.shape[1] == nslice * W
        self._call("md_rownorm_fwd", x.data_ptr(), x.stride(0), rstd.data_ptr(), rows, W, nslice, eps)

    def rownorm_bwd(self, dy, xhat, rstd, nslice=1):
        rows, W = dy.shape[0], dy.shape[1] // nslice
        assert rstd.numel() == nslice * rows and xhat.shape[1] == dy.shape[1] == nslice * W
        self._call("md_rownorm_bwd", dy.data_ptr(), dy.stride(0), xhat.data_ptr(), xhat.stride(0), rstd.data_ptr(),
                   rows, W, nslice)

    def gate_bwd(self, dres, dy, *, y=None, gate=None, dgate=None, T):
        rows, D = dres.shape
        g, ld = _mod(gate)
        dg, ld2 = _mod(dgate)
        self._call("md_gate_bwd", dres.data_ptr(), _ptr(y), g, ld or ld2, T, dy.data_ptr(), dg, rows, D)

    # ------------------------------------------------------------------ attention
    def attn_fwd(self, q, k, v, o, lse, B, H, Tq, Tk, hd):
        if self.prec:
            name = "md_attn_fwd_f32"
        else:
            tc_ok = (hd == 64 and Tk <= 256) or hd == 128
            name = "md_attn_fwd_tc" if (self.attn_tc and tc_ok) else "md_attn_fwd"
            if self.attn_tc is False:
                name = "md_attn_fwd_mma"
        self._call(name, q.data_ptr(), q.stride(0), k.data_ptr(), k.stride(0), v.data_ptr(), v.stride(0),
                   o.data_ptr(), o.stride(0), lse.data_ptr(), B, H, Tq, Tk, hd,
                   label=f"B={B} H={H} Tq={Tq} Tk={Tk}", flops=4 * B * H * Tq * Tk * hd)

    def attn_bwd(self, dout, q, k, v, o, lse, delta, dq, dk, dv, B, H, Tq, Tk, hd):
        if self.prec:
            self._call("md_attn_bwd_f32", dout.data_ptr(), dout.stride(0), q.data_ptr(), q.stride(0), k.data_ptr(),
                       k.stride(0), v.data_ptr(), v.stride(0), o.data_ptr(), o.stride(0), lse.data_ptr(),
                       delta.data_ptr(), dq.data_ptr(), dq.stride(0), dk.data_ptr(), dk.stride(0), dv.data_ptr(),
                       dv.stride(0), B, H, Tq, Tk, hd, label=f"B={B} H={H} Tq={Tq} Tk={Tk}")
            return
        if delta is None:  # scratch of the many-key kernels
            delta = self.empty((B, H, Tq), torch.float32)
        name = "md_attn_bwd_tc" if (self.attn_tc and hd == 64) else "md_attn_bwd"
        if self.attn_tc is False:
            name = "md_attn_bwd_mma"
        self._call(name, dout.data_ptr(), dout.stride(0),
                   q.data_ptr(), q.stride(0), k.data_ptr(),
                   k.stride(0), v.data_ptr(), v.stride(0), o.data_ptr(), o.stride(0), lse.data_ptr(),
                   delta.data_ptr(), dq.data_ptr(), dq.stride(0), dk.data_ptr(), dk.stride(0), dv.data_ptr(),
                   dv.stride(0), B, H, Tq, Tk, hd,
                   label=f"B={B} H={H} Tq={Tq} Tk={Tk}", flops=10 * B * H * Tq * Tk * hd)

    # ------------------------------------------------------------------ feed-forward tails
    def swiglu_fwd(self, u, h):
        self._call("md_swiglu_fwd", u.data_ptr(), h.data_ptr(), h.shape[0], h.shape[1])

    def swiglu_bwd(self, dh, u, du):
        self._call("md_swiglu_bwd", dh.data_ptr(), u.data_ptr(), du.data_ptr(), dh.shape[0], dh.shape[1])

    def act_fwd(self, pre, out, act):
        self._call("md_act_fwd", pre.data_ptr(), out.data_ptr(), pre.numel(), act)

    def act_bwd(self, dact, pre, dpre, act):
        self._call("md_act_bwd", dact.data_ptr(), pre.data_ptr(), dpre.data_ptr(), dact.numel(), act)

    def gelu_tanh_f32_fwd(self, c, out):
        self._call("md_gelu_tanh_f32_fwd", c.data_ptr(), out.data_ptr(), c.numel())

    def gelu_tanh_f32_bwd(self, dact, c, dc, accumulate):
        self._call("md_gelu_tanh_f32_bwd", dact.data_ptr(), c.data_ptr(), dc.data_ptr(), int(accumulate), c.numel())

    # ------------------------------------------------------------------ MoE
    def moe_gate_fwd(self, x, wg, probs):
        self._call("md_moe_gate_fwd", x.data_ptr(), wg.data_ptr(), probs.data_ptr(), x.shape[0], x.shape[1],
                   wg.shape[0])

    def moe_topk(self, probs, idx, gval, inv, B, T, E, k):
        self._call("md_moe_topk", probs.data_ptr(), idx.data_ptr(), gval.data_ptr(), inv.data_ptr(), B, T, E, k)

    def moe_gather(self, x, idx, xin, B, T, E, k):
        self._call("md_moe_gather", x.data_ptr(), idx.data_ptr(), xin.data_ptr(), B, T, E, k, x.shape[1])

    def moe_combine_fwd(self, h2, gval, inv, xres, gate, xout, ymoe, B, T, E, k):
        g, ld = _mod(gate)
        self._call("md_moe_combine_fwd", h2.data_ptr(), gval.data_ptr(), inv.data_ptr(), _ptr(xres), g, ld,
                   _ptr(xout), _ptr(ymoe), B, T, E, k, h2.shape[-1])

    def moe_combine_bwd(self, dy, h2, gval, idx, dh2, dgval, B, T, E, k):
        self._call("md_moe_combine_bwd", dy.data_ptr(), h2.data_ptr(), gval.data_ptr(), idx.data_ptr(),
                   dh2.data_ptr(), dgval.data_ptr(), B, T, E, k, h2.shape[-1])

    def moe_dx_bwd(self, dxin, inv, dgval, probs, wg, dscores, dx, B, T, E, k):
        self._call("md_moe_dx_bwd", dxin.data_ptr(), inv.data_ptr(), dgval.data_ptr(), probs.data_ptr(),
                   wg.data_ptr(), dscores.data_ptr(), dx.data_ptr(), B, T, E, k, dx.shape[-1])

    def moe_gate_wgrad(self, dscores, x, dwg):
        self._call("md_moe_gate_wgrad", dscores.data_ptr(), x.data_ptr(), dwg.data_ptr(), x.shape[0], x.shape[1],
                   dwg.shape[0])

    # ------------------------------------------------------------------ masking
    def mask_sort(self, noise, ids_shuffle, ids_restore, mask, keep_rows, keep):
        B, T = noise.shape
        self._call("md_mask_sort", noise.data_ptr(), _ptr(ids_shuffle), _ptr(ids_restore), _ptr(mask),
                   _ptr(keep_rows), B, T, keep)

    def gather_rows(self, x, src_rows, y):
        self._call("md_gather_rows_f32", x.data_ptr(), src_rows.data_ptr(), y.data_ptr(), y.shape[0], y.shape[1])

    def scatter_rows(self, dy, src_rows, dx):
        self._call("md_scatter_rows_f32", dy.data_ptr(), src_rows.data_ptr(), dx.data_ptr(), dy.shape[0], dy.shape[1])

    # ------------------------------------------------------------------ EDM
    def cond_prepare(self, cap, keep, out, cap_out=None):
        assert cap.dtype == torch.float16 and cap.is_contiguous()
        B = cap.shape[0]
        self._call("md_cond_prepare", cap.data_ptr(), _ptr(keep), out.data_ptr(), _ptr(cap_out), B, cap.numel() // B)

    def patchify(self, x, scale, patches, p):
        B, Cc, H, W = x.shape
        assert x.is_contiguous() and x.dtype == torch.float32
        self._call("md_patchify", x.data_ptr(), _ptr(scale), patches.data_ptr(), B, Cc, H, W, p)

    def edm_prepare(self, lat, eps, rnd, sigma_in, p_mean, p_std, sigma_data, xn, patches, coef, p):
        B, Cc, H, W = lat.shape
        assert lat.is_contiguous() and eps.is_contiguous() and lat.dtype in (torch.float16, torch.float32)
        self._call("md_edm_prepare", lat.data_ptr(), int(lat.dtype == torch.float16), eps.data_ptr(), _ptr(rnd),
                   _ptr(sigma_in), p_mean, p_std, sigma_data, xn.data_ptr(), patches.data_ptr(), coef.data_ptr(),
                   B, Cc, H, W, p)

    def timestep_embed(self, t, out):
        self._call("md_timestep_embed", t.data_ptr(), out.data_ptr(), out.shape[0], out.shape[1])

    def edm_loss_fwd(self, ftok, keep_tok, lat, xn, coef, per_sample, loss, p, Tk):
        B, Cc, H, W = lat.shape
        self._call("md_edm_loss_fwd", ftok.data_ptr(), _ptr(keep_tok), lat.data_ptr(),
                   int(lat.dtype == torch.float16), xn.data_ptr(), coef.data_ptr(), per_sample.data_ptr(),
                   loss.data_ptr(), B, Cc, H, W, p, Tk)

    def edm_loss_bwd(self, ftok, keep_tok, lat, xn, coef, gscale, dftok, p, Tk):
        B, Cc, H, W = lat.shape
        self._call("md_edm_loss_bwd", ftok.data_ptr(), _ptr(keep_tok), lat.data_ptr(),
                   int(lat.dtype == torch.float16), xn.data_ptr(), coef.data_ptr(), gscale.data_ptr(),
                   dftok.data_ptr(), B, Cc, H, W, p, Tk)

    def edm_output(self, ftok, ids_restore, mask_token, xn, coef, fx, dx, p, Tk):
        ref = fx if fx is not None else dx
        B, Cc, H, W = ref.shape
        self._call("md_edm_output", ftok.data_ptr(), _ptr(ids_restore), _ptr(mask_token), _ptr(xn), _ptr(coef),
                   _ptr(fx), _ptr(dx), B, Cc, H, W, p, Tk)

    HEUN_IN, HEUN_EULER, HEUN_CORRECT, HEUN_NEXT = 0, 1, 2, 3

    def edm_heun(self, stage, x, x_hat, d_cur, den, noise, xin, sigma, table, step, s_noise):
        """One stage of the fp64 Heun step (md_edm_heun) on the state x, x_hat, d_cur (f64 [B,C,H,W]).  table: f64
        [2*max_steps+1] (t_steps | t_hat), step: int32 [1] device index, noise: f64 [max_steps, B,C,H,W], xin: f32 [copies*B,
        C,H,W], sigma: f32 [copies*B], den: f32 [B,C,H,W].  HEUN_NEXT only advances `step`."""
        assert step.dtype == torch.int32 and step.numel() == 1
        if stage == self.HEUN_NEXT:
            self._call("md_edm_heun", stage, *([None] * 8), step.data_ptr(), 1, 1, 1, 1, 1.0)
            return
        B = x.shape[0]
        n = x[0].numel()
        assert table.dtype == torch.float64 and table.numel() % 2 == 1 and table.is_contiguous()
        max_steps = table.numel() // 2
        for t in (x, x_hat, d_cur):
            assert t is None or (t.dtype == torch.float64 and t.shape == x.shape and t.is_contiguous())
        assert den is None or (den.dtype == torch.float32 and den.shape == x.shape and den.is_contiguous())
        assert noise is None or (noise.dtype == torch.float64 and noise.is_contiguous() and
                                 tuple(noise.shape) == (max_steps, *x.shape))
        copies = 1
        if xin is not None:
            copies = xin.shape[0] // B
            assert xin.dtype == torch.float32 and xin.is_contiguous() and tuple(xin.shape) == (copies * B, *x.shape[1:])
            assert sigma.dtype == torch.float32 and sigma.numel() == copies * B
        self._call("md_edm_heun", stage, x.data_ptr(), _ptr(x_hat), _ptr(d_cur), _ptr(den), _ptr(noise), _ptr(xin),
                   _ptr(sigma), table.data_ptr(), step.data_ptr(), max_steps, B, n, copies, float(s_noise))

    def edm_output_cfg(self, ftok, x, sigma, cfg, dx, sigma_data, p):
        """dx = c_skip*x + c_out*(unc + cfg*(cond - unc)) for a doubled (cond | uncond) batch, md_edm_output_cfg: ftok f32
        [2B*T, p*p*C], x / dx f32 [B,C,H,W], sigma f32 [B], cfg f32 [1] on the device.  sigma_data is the Python float of
        the EDM config: its fp32 value and the fp32 value of its square enter like torch's scalar operands."""
        B, Cc, H, W = dx.shape
        assert x.shape == dx.shape and x.is_contiguous() and dx.is_contiguous() and x.dtype == dx.dtype == torch.float32
        assert ftok.dtype == torch.float32 and ftok.is_contiguous() and tuple(ftok.shape) == (2 * B * (H // p) * (W // p),
                                                                                               p * p * Cc)
        assert sigma.dtype == torch.float32 and sigma.numel() >= B and cfg.dtype == torch.float32 and cfg.numel() == 1
        self._call("md_edm_output_cfg", ftok.data_ptr(), x.data_ptr(), sigma.data_ptr(), cfg.data_ptr(), dx.data_ptr(),
                   float(sigma_data), float(sigma_data) ** 2, B, Cc, H, W, p)

    # ------------------------------------------------------------------ adjoints of the DiT input / output maps
    def unpatchify_bwd(self, dF, keep_rows, dftok, p, Tk):
        """dftok [B*Tk, p*p*C] = adjoint of edm_output's un-mask + unpatchify at the kept tokens (all when keep_rows is None)."""
        B, Cc, H, W = dF.shape
        assert dF.is_contiguous() and dF.dtype == torch.float32 and dftok.shape == (B * Tk, p * p * Cc)
        self._call("md_unpatchify_bwd", dF.data_ptr(), _ptr(keep_rows), dftok.data_ptr(), B, Cc, H, W, p, Tk)

    def patchify_bwd(self, dpatches, scale, dx, p):
        """dx f32 [B,C,H,W] = adjoint of patchify (col2im) of dpatches f32 [B*T, C*p*p]."""
        B, Cc, H, W = dx.shape
        assert dpatches.is_contiguous() and dpatches.dtype == torch.float32 and dx.is_contiguous()
        assert dpatches.shape == (B * (H // p) * (W // p), Cc * p * p)
        self._call("md_patchify_bwd", dpatches.data_ptr(), _ptr(scale), dx.data_ptr(), B, Cc, H, W, p)

    def timestep_embed_bwd(self, dfreq, t, dt):
        """dt f32 [B] = adjoint of timestep_embed at t for the cotangent dfreq f32 [B, dim]."""
        assert dfreq.is_contiguous() and dfreq.dtype == torch.float32 and t.dtype == torch.float32 and t.is_contiguous()
        self._call("md_timestep_embed_bwd", dfreq.data_ptr(), t.data_ptr(), dt.data_ptr(), dfreq.shape[0], dfreq.shape[1])

    # ------------------------------------------------------------------ utilities
    def mean_tokens_fwd(self, x, out, B, L):
        self._call("md_mean_tokens_fwd", x.data_ptr(), out.data_ptr(), B, L, out.shape[1])

    def mean_tokens_bwd(self, d, dx, B, L):
        self._call("md_mean_tokens_bwd", d.data_ptr(), dx.data_ptr(), B, L, d.shape[1])

    def cast_bf16(self, x, y):
        assert x.is_contiguous() and y.is_contiguous()
        self._call("md_cast_f32_bf16", x.data_ptr(), y.data_ptr(), x.numel())

    def colsum(self, x, out):
        rows, N = x.shape
        self._call("md_colsum", x.data_ptr(), int(x.dtype == torch.bfloat16), x.stride(0), out.data_ptr(), rows, N)

    def colsum_interleaved(self, x, out, half):
        """out(f32 [2 half]) += column sums of x [rows, 2 half] (32-interleaved w1 | w2 columns), in [b1 | b2] order."""
        rows, N = x.shape
        assert N == 2 * half and out.numel() == N and out.dtype == torch.float32
        self._call("md_colsum_interleaved", x.data_ptr(), int(x.dtype == torch.bfloat16), x.stride(0), out.data_ptr(), rows,
                   N, half)

    def cast_transpose(self, w, wb, wbt, interleave_half=0):
        if w.dim() == 2:
            batch, (rows, cols) = 1, w.shape
        else:
            batch, rows, cols = w.shape
        self._call("md_cast_transpose", w.data_ptr(), _ptr(wb), _ptr(wbt), batch, rows, cols, interleave_half)

    def cast_transpose_multi(self, flat, wb, wbt, desc, total_tiles):
        """desc: int64 [n, 8] device tensor of md_cast_desc rows (offset, rows, cols, half, need_t, tile_start, tiles_x, 0)."""
        assert desc.dtype == torch.int64 and desc.dim() == 2 and desc.shape[1] == 8 and desc.is_contiguous()
        self._call("md_cast_transpose_multi", flat.data_ptr(), wb.data_ptr(), wbt.data_ptr(), desc.data_ptr(), desc.shape[0],
                   total_tiles)

    def sumsq(self, x, out):
        self._call("md_sumsq", x.data_ptr(), out.data_ptr(), x.numel())

    def adamw(self, p, g, m, v, sumsq, clip, lr, beta1, beta2, eps, wd, step, nonfinite=None):
        self._call("md_adamw", p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), _ptr(sumsq), clip, lr, beta1,
                   beta2, eps, wd, step, _ptr(nonfinite), p.numel())

    def adamw_ema(self, p, g, m, v, sumsq, clip, lr, beta1, beta2, eps, wd, step, ema, smoothing, nonfinite=None):
        """adamw(...) and, in the same pass, ema = smoothing * ema + (1 - smoothing) * p_new."""
        assert ema.numel() == p.numel() and ema.dtype == torch.float32
        self._call("md_adamw_ema", p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), _ptr(sumsq), clip, lr, beta1,
                   beta2, eps, wd, step, ema.data_ptr(), smoothing, _ptr(nonfinite), p.numel())

    def swap(self, a, b):
        """Exchange the contents of two fp32 buffers of the same size in place (md_swap_f32; they may not overlap)."""
        assert a.numel() == b.numel() and a.dtype == b.dtype == torch.float32 and a.is_contiguous() and b.is_contiguous()
        self._call("md_swap_f32", a.data_ptr(), b.data_ptr(), a.numel())
