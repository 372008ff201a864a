/* microdit_b200 -- C ABI of the H100 (sm_90a) MicroDiT training hot path.
 *
 * Every entry point takes plain device pointers, integer sizes and a CUDA stream handle
 * (cudaStream_t passed as void*), returns 0 on success or a negative MD_ERR_* code, never allocates
 * device memory and keeps no global state besides cached function attributes; all calls are
 * asynchronous on the given stream and re-entrant per stream.  md_last_error() returns the message of
 * the last failure on the calling thread.
 *
 * The reference (SonyResearch/micro_diffusion) has no FFI: its hot path is Python calling torch ops.
 * Each function below names the reference code it replaces (file:line under the reference root).
 * The Python binding a maintainer would add is the ctypes stub in INTEGRATION.md.
 *
 * Conventions: "rows" are tokens (sample-major: row = sample * T + token); bf16 = __nv_bfloat16;
 * per-sample modulation vectors (shift / scale / gate) are passed as a pointer to sample 0 plus a row
 * pitch `ldmod` in elements (they are column slices of one [samples, sum(6*D)] adaLN buffer);
 * `T` = rows per sample.
 *
 * `prec` selects the storage type of the GEMM-operand / saved-activation tensors an entry point reads or writes (the
 * arguments documented as bf16): 0 = bf16, the product path (the reference's amp_bf16 regime, train.py:113);
 * 1 = fp32, the high-precision mode (MD_PRECISION=high) in which the same kernels and the same host sequencing are
 * gated against the fp32 oracle at 1e-3 on loss and denoiser output.  Statistics, the residual stream, router
 * probabilities, the loss and every parameter gradient are fp32 in both modes.
 */
#ifndef MICRODIT_B200_H_
#define MICRODIT_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(MD_BUILDING_LIB)
#define MD_API __attribute__((visibility("default")))
#else
#define MD_API
#endif

#define MD_OK 0
#define MD_ERR_INVALID (-1)     /* bad argument (null pointer, misaligned operand, bad size) */
#define MD_ERR_CUDA (-2)        /* CUDA runtime / driver error */
#define MD_ERR_UNSUPPORTED (-3) /* device is not sm_90a, or shape outside the kernel's envelope */

MD_API const char* md_last_error(void);
MD_API int md_abi_version(void);
/* Deterministic mode.  The fast path accumulates some gradients with floating-point atomics across thread blocks (split-K
 * weight gradients, the per-column reductions of the LayerNorm / gate / router / bias gradients, the gradient norm), so
 * two runs differ in the last bits.  With a workspace registered here those accumulations go through per-block partial
 * sums in the workspace and a fixed-order reduction: the same inputs give bit-identical outputs (what the reference gets
 * from cuBLAS + torch's deterministic reductions).  The workspace (device memory, >= 1 MiB, 256-byte aligned, owned by
 * the caller; 1 GiB covers MicroDiT_XL_2 at microbatch 512) is reused by consecutive launches: issue all calls on one
 * stream.  NULL turns the mode off.  Requests that do not fit fall back to an unsplit (slower, still deterministic) form. */
MD_API int md_set_deterministic(void* workspace, int64_t bytes);

/* ------------------------------------------------------------------------------------------ GEMM */
#define MD_GEMM_NT 0 /* C[M,N] = A[M,K] . B[N,K]^T   (A, B row-major, K contiguous)                 */
#define MD_GEMM_TN 1 /* C[M,N] = A[K,M]^T . B[K,N]   (A, B row-major, reduction index K strided)    */
#define MD_EPI_STORE_BF16 0 /* C(bf16) = alpha*acc (+bias)                                           */
#define MD_EPI_STORE_F32 1  /* C(f32)  = alpha*acc (+bias)                                           */
#define MD_EPI_RESID_F32 2  /* C(f32)  = res[row % res_mod] + gate[row/rows_per_gate]*(alpha*acc+bias) */
                            /*           C2(bf16, optional) = alpha*acc+bias                         */
#define MD_EPI_ATOMIC_F32 3 /* C(f32) += alpha*acc   (red.global.add; the only mode allowing splits; no bias:
                             * a bias is MD_ERR_INVALID) */
#define MD_EPI_ACT_DUAL 4   /* C(bf16) = pre = alpha*acc+bias ; C2(bf16) = act(pre); act: 0 gelu-erf, 1 gelu-tanh */
#define MD_EPI_ACT_GRAD 5   /* C(bf16) = alpha*acc * act'(aux) (no bias): the dgrad GEMM of an activation's output applies the
                             * activation's derivative at the saved pre-activation aux (bf16, indexed like C) */

#define MD_EPI_SWIGLU 6     /* N = 2f columns in the 32-interleaved order (w1 block j, w2 block j, ...): C(bf16) = u = alpha*acc
                             * (+bias), C2(bf16 [M, f], pitch ldc2) = silu(u1) * u2 (FeedForward, dit.py:84-89).  bias (optional,
                             * f32 [batch][2f]) is in the natural [b1 | b2] order: interleaved column c = 64 j + r takes
                             * bias[32 j + r] for r < 32 and bias[f + 32 j + r - 32] otherwise, and is added before u is
                             * rounded and stored, so the u that MD_EPI_SWIGLU_GRAD reads back includes it */
#define MD_EPI_SWIGLU_GRAD 7 /* N = f: acc = d h; C(bf16 [M, 2f] interleaved) = (d h * u2 * silu'(u1) | d h * silu(u1)) with
                              * u = aux (bf16 [M, 2f] interleaved, indexed like C); no bias */

typedef struct md_gemm_args {
  const void* A; /* bf16 */
  const void* B; /* bf16 */
  void* C;
  void* C2;
  const void* bias; /* f32 [batch][N] or NULL */
  const void* res;  /* f32, indexed like C (may alias C); row taken modulo res_mod when res_mod > 0 */
  const void* gate; /* f32 [M / rows_per_gate][ldgate] or NULL (=1) */
  const void* aux;  /* bf16, indexed like C: the saved pre-activation of MD_EPI_ACT_GRAD */
  int64_t M, N, K;
  int64_t lda, ldb, ldc; /* row pitches in elements */
  int64_t batch;         /* >= 1; batch strides in elements */
  int64_t strideA, strideB, strideC, strideBias;
  int64_t ldgate, rows_per_gate;
  int64_t res_mod;  /* 0: res row == C row */
  int32_t layout;   /* MD_GEMM_* */
  int32_t epilogue; /* MD_EPI_*  */
  int32_t splits;   /* split of the reduction dimension (>=1) */
  int32_t act;      /* activation of MD_EPI_ACT_DUAL */
  float alpha;      /* 0 is treated as 1 */
  int32_t sm_limit; /* > 0: use at most this many SMs (persistent grid) -- leaves room for a concurrent collective */
  int64_t ldc2, strideC2;   /* pitch / batch stride of C2 for MD_EPI_SWIGLU (0: N / 2, unbatched) */
  int64_t row_interleave;   /* f > 0 (atomic epilogue, M == 2f): output row p is the gradient of row
                             * (p % 64 < 32 ? 0 : f) + 32 * (p / 64) + p % 32 -- the weight gradient of a 32-row-interleaved
                             * w1 | w2 stack lands in the parameters' own order */
} md_gemm_args;

/* Dense / batched bf16 GEMM, fp32 accumulation, wgmma tensor cores fed by TMA.
 * Replaces nn.Linear under autocast -- qkv/proj utils.py:172-173, cross-attn q/kv/proj utils.py:109-111,
 * SwiGLU dit.py:84-89, adaLN dit.py:227-230, stem/mixer maps dit.py:377-388, final linear utils.py:226-230,
 * patch-embed conv dit.py:312-314 (as a K=C*p*p GEMM) -- the expert einsums dit.py:135-137 (batch =
 * experts) and the autograd dgrad/wgrad of all of them. */
MD_API int md_gemm_bf16(const md_gemm_args* args, void* stream);

/* --------------------------------------------------------------------------- LayerNorm (+modulate) */
/* y = LN(x; gamma, eps) * (1 + scale[sample]) + shift[sample]   (create_norm utils.py:71-78 +
 * modulate utils.py:28-30; call sites dit.py:236-238, utils.py:238).  x: f32 (x_bf16=0) or bf16 (1),
 * [rows, D]; src_rows (optional, int32 [rows]) gathers input rows (mask_out_token utils.py:406-414 fused
 * into the patch_mixer_map_xout norm, dit.py:504-508).  gamma / shift / scale may be NULL.  y bf16 [rows,D];
 * mean, rstd f32 [rows].  D % 8 == 0, D <= 2048.
 * y_add (optional, bf16 [rows_src, D]): the pending gated residual update of the previous sub-block is applied first,
 * x_new[src] = x[src] + gate_add[sample] * y_add[src] (dit.py:236-238), written to x_new (f32) and then normalised --
 * the branch GEMM then stores plain bf16 instead of doing the fp32 read-modify-write in its epilogue. */
MD_API int md_ln_fwd(const void* x, int x_bf16, const int32_t* src_rows, const void* y_add, const float* gate_add,
                     float* x_new, const float* gamma, const float* shift, const float* scale, int64_t ldmod,
                     int64_t T, void* y, float* mean, float* rstd, int64_t rows, int64_t D, float eps,
                     int prec, void* stream);
/* Backward of the above.  dy bf16 [rows, D].  dx_mode: 0 = dx(f32)[r] += , 1 = dx(bf16)[r] = ,
 * 2 = dx(f32)[src_rows[r]] += (scatter).  dgamma f32 [D] += (atomic); dshift / dscale f32 [samples, D]
 * pitched by ldmod, += (atomic; caller zeroes them once per step).  NULL outputs are skipped.
 * Fused tail (dy_next != NULL; needs dx_mode 0): the updated dx is the gradient entering the NEXT branch of the backward
 * chain, so its gated-residual backward (md_gate_bwd below) rides along instead of re-reading dx:
 * dy_next(bf16) = gate_next[sample] * dx_new, dgate_next[sample] += sum_t dx_new * y_next (atomic); y_next / gate_next /
 * dgate_next may be NULL (plain cast). */
MD_API int md_ln_bwd(const void* dy, const void* x, int x_bf16, const int32_t* src_rows, const float* gamma,
                     const float* scale, int64_t ldmod, int64_t T, const float* mean, const float* rstd,
                     void* dx, int dx_mode, float* dgamma, float* dshift, float* dscale, const void* y_next,
                     const float* gate_next, float* dgate_next, void* dy_next, int64_t rows, int64_t D, int prec,
                     void* stream);
/* Non-affine LayerNorm over W-wide column slices, in place on bf16 (QK-norm: ln_q / ln_k utils.py:183-186,
 * 122-125).  fwd: x <- (x-mean)*rstd, rstd out.  bwd: dy <- rstd*(dy - mean(dy) - xhat*mean(dy*xhat)).
 * nslice (1..4) adjacent slices [s*W, (s+1)*W) of every row are normalised independently in ONE launch (q and k of
 * the packed qkv projection); rstd is [nslice][rows]. */
MD_API int md_rownorm_fwd(void* x, int64_t ld, float* rstd, int64_t rows, int64_t W, int64_t nslice, float eps, int prec,
                          void* stream);
MD_API int md_rownorm_bwd(void* dy, int64_t ld_dy, const void* xhat, int64_t ld_x, const float* rstd, int64_t rows,
                          int64_t W, int64_t nslice, int prec, void* stream);
/* Backward of x_new = x + gate[sample] * y (dit.py:236,238): dy(bf16) = gate * dres;
 * dgate[sample] += sum_t dres * y (atomic).  y / gate / dgate may be NULL (plain f32->bf16 cast). */
MD_API int md_gate_bwd(const float* dres, const void* y, const float* gate, int64_t ldmod, int64_t T, void* dy,
                       float* dgate, int64_t rows, int64_t D, int prec, void* stream);

/* ------------------------------------------------------------------------------------- attention */
/* softmax(Q K^T / sqrt(hd)) V, non-causal (F.scaled_dot_product_attention at utils.py:188-193 self,
 * 127-132 cross).  q [B*Tq, *] pitch ldq, k / v [B*Tk, *] pitch ldk / ldv, head h at column h*hd;
 * o bf16 [B*Tq, H*hd] pitch ldo; lse f32 [B,H,Tq] (log2 domain).  hd 32, 64 or 128 (any other: MD_ERR_UNSUPPORTED).
 * Every bf16 attention entry point needs q / k / v / o (and dout / dq / dk / dv) 16-byte aligned and every row pitch a
 * multiple of 8 elements; anything else is MD_ERR_INVALID. */
MD_API int md_attn_fwd(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, void* o,
                       int64_t ldo, float* lse, int64_t B, int64_t H, int64_t Tq, int64_t Tk, int64_t hd,
                       void* stream);
/* delta scratch f32 [B,H,Tq]; dq/dk/dv bf16 with the pitches of q/k/v.  hd 32, 64 or 128; where the backward runs a
 * delta pass (every hd-128 shape, and more than 80 keys at hd 32 / 64) H*hd must be <= 2048: at most 16 heads at hd 128,
 * 32 at hd 64. */
MD_API int md_attn_bwd(const void* dout, int64_t lddo, const void* q, int64_t ldq, const void* k, int64_t ldk,
                       const void* v, int64_t ldv, const void* o, int64_t ldo, const float* lse, float* delta,
                       void* dq, int64_t lddq, void* dk, int64_t lddk, void* dv, int64_t lddv, int64_t B, int64_t H,
                       int64_t Tq, int64_t Tk, int64_t hd, void* stream);
/* The same backward on wgmma (csrc/attn_wgmma.cu) for head_dim 64, any Tk: a dK / dV kernel role per 64-key block and a
 * dQ role per 64-query block (no atomics); delta is scratch.  md_attn_bwd dispatches here above 128 keys.  H*hd must be
 * <= 2048 (at most 32 heads), as for the generic split; more is MD_ERR_UNSUPPORTED. */
MD_API int md_attn_bwd_tc(const void* dout, int64_t lddo, const void* q, int64_t ldq, const void* k, int64_t ldk,
                          const void* v, int64_t ldv, const void* o, int64_t ldo, const float* lse, float* delta,
                          void* dq, int64_t lddq, void* dk, int64_t lddk, void* dv, int64_t lddv, int64_t B, int64_t H,
                          int64_t Tq, int64_t Tk, int64_t hd, void* stream);
/* The mma.sync (m16n8k16) flash-style kernels (csrc/attn.cu), head_dim 32, 64 or 128: the whole backward, and the
 * forward outside the wgmma envelope (head_dim 32; head_dim 64 with Tk > 256); callable directly for A/B runs. */
MD_API int md_attn_fwd_mma(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, void* o,
                           int64_t ldo, float* lse, int64_t B, int64_t H, int64_t Tq, int64_t Tk, int64_t hd,
                           void* stream);
MD_API int md_attn_bwd_mma(const void* dout, int64_t lddo, const void* q, int64_t ldq, const void* k, int64_t ldk,
                           const void* v, int64_t ldv, const void* o, int64_t ldo, const float* lse, float* delta,
                           void* dq, int64_t lddq, void* dk, int64_t lddk, void* dv, int64_t lddv, int64_t B, int64_t H,
                           int64_t Tq, int64_t Tk, int64_t hd, void* stream);
/* The same forward on the warpgroup tensor cores (TMA + wgmma, csrc/attn_wgmma.cu) for head_dim 64 with Tk <= 256 (one
 * 64-query tile per CTA, whole-row softmax in registers, P fed back to the tensor core from registers) and for head_dim
 * 128 with any Tk (online softmax over 64-key chunks streamed through a two-stage TMA ring).  md_attn_fwd dispatches here
 * whenever the shape is inside this envelope. */
MD_API int md_attn_fwd_tc(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, void* o,
                          int64_t ldo, float* lse, int64_t B, int64_t H, int64_t Tq, int64_t Tk, int64_t hd,
                          void* stream);
/* High-precision mode (prec = 1): the same contract with fp32 q / k / v / o / gradients, plain fp32 FMAs; hd 32, 64
 * or 128. */
MD_API int md_attn_fwd_f32(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, void* o,
                           int64_t ldo, float* lse, int64_t B, int64_t H, int64_t Tq, int64_t Tk, int64_t hd,
                           void* stream);
MD_API int md_attn_bwd_f32(const void* dout, int64_t lddo, const void* q, int64_t ldq, const void* k, int64_t ldk,
                           const void* v, int64_t ldv, const void* o, int64_t ldo, const float* lse, float* delta,
                           void* dq, int64_t lddq, void* dk, int64_t lddk, void* dv, int64_t lddv, int64_t B, int64_t H,
                           int64_t Tq, int64_t Tk, int64_t hd, void* stream);
/* High-precision GEMM operands: fp32 x [batch][rows][cols] (row pitch ldx, batch pitch batch_stride, elements) ->
 * bf16 triples hi = bf16(x), lo = bf16(x - hi) stacked along the contraction, so that md_gemm_bf16 at 3x the depth
 * accumulates a_hi b_hi + a_lo b_hi + a_hi b_lo in fp32 (the high-precision mode runs on the same wgmma kernel).
 * role 0 (A operand): [hi | lo | hi]; role 1 (B operand): [hi | hi | lo].
 * along 0: out [batch][rows][3*cols] (K-major operands); along 1: out [batch][3*rows][cols] (MN-major operands). */
MD_API int md_split3_bf16(const float* x, int64_t ldx, int64_t batch_stride, void* out, int64_t batch, int64_t rows,
                          int64_t cols, int role, int along, void* stream);

/* ------------------------------------------------------------------------------ feed-forward tails */
/* SwiGLU (dit.py:88-89): u bf16 [rows, 2f] = [w1 x | w2 x];  h = silu(u[:, :f]) * u[:, f:]. */
MD_API int md_swiglu_fwd(const void* u, void* h, int64_t rows, int64_t f, int prec, void* stream);
MD_API int md_swiglu_bwd(const void* dh, const void* u, void* du, int64_t rows, int64_t f, int prec, void* stream);
/* act = act(pre), bf16 -> bf16 (the expert GELU, dit.py:136, as its own HBM-bound pass: in the GEMM epilogue it
 * made the expert GEMM epilogue-bound) */
MD_API int md_act_fwd(const void* pre, void* out, int64_t n, int act, int prec, void* stream);
/* dpre = dact * act'(pre), bf16 (act: 0 gelu-erf dit.py:136, 1 gelu-tanh utils.py:65). */
MD_API int md_act_bwd(const void* dact, const void* pre, void* dpre, int64_t n, int act, int prec, void* stream);
/* c_act(bf16) = gelu_tanh(c f32)  (the nn.GELU in every adaLN_modulation, dit.py:227-230);
 * bwd: dc(f32) (+)= dc_act(f32) * gelu_tanh'(c). */
MD_API int md_gelu_tanh_f32_fwd(const float* c, void* out_bf16, int64_t n, int prec, void* stream);
MD_API int md_gelu_tanh_f32_bwd(const float* dact, const float* c, float* dc, int accumulate, int64_t n, void* stream);

/* -------------------------------------------------------------------------- expert-choice MoE */
/* FeedForwardECMoe (dit.py:126-143).  E <= 16, D % 8 == 0. */
/* probs(f32 [rows,E]) = softmax(x(bf16 [rows,D]) . Wg(f32 [E,D])^T)   (dit.py:130-131) */
MD_API int md_moe_gate_fwd(const void* x, const float* wg, float* probs, int64_t rows, int64_t D, int64_t E,
                           int prec, void* stream);
/* per (sample, expert) top-k over the T tokens (dit.py:132): idx int32 [B,E,k], gval f32 [B,E,k],
 * inv int32 [B,T,E] = slot of token t in expert e's list or -1.  T <= 4096. */
MD_API int md_moe_topk(const float* probs, int32_t* idx, float* gval, int32_t* inv, int64_t B, int64_t T, int64_t E,
                       int64_t k, void* stream);
/* dispatch (the one-hot einsum dit.py:134 as a gather): xin bf16 [E, B*k, D] */
MD_API int md_moe_gather(const void* x, const int32_t* idx, void* xin, int64_t B, int64_t T, int64_t E, int64_t k,
                         int64_t D, int prec, void* stream);
/* combine (dit.py:139-140) fused with the gated residual (dit.py:238):
 * ymoe(bf16 [rows,D]) = sum_e g*h2 ; xout(f32) = xres + gate[sample]*ymoe */
MD_API int md_moe_combine_fwd(const void* h2, const float* gval, const int32_t* inv, const float* xres,
                              const float* gate, int64_t ldmod, float* xout, void* ymoe, int64_t B, int64_t T,
                              int64_t E, int64_t k, int64_t D, int prec, void* stream);
/* dh2(bf16 [E,B*k,D]) = g * dy[token] ; dgval(f32 [B,E,k]) = <h2, dy[token]> */
MD_API int md_moe_combine_bwd(const void* dy, const void* h2, const float* gval, const int32_t* idx, void* dh2,
                              float* dgval, int64_t B, int64_t T, int64_t E, int64_t k, int64_t D,
                              int prec, void* stream);
/* softmax/top-k backward + un-dispatch: dscores f32 [rows,E]; dx(bf16 [rows,D]) = sum_e dxin[slot] + dscores.Wg */
MD_API int md_moe_dx_bwd(const void* dxin, const int32_t* inv, const float* dgval, const float* probs,
                         const float* wg, float* dscores, void* dx, int64_t B, int64_t T, int64_t E, int64_t k,
                         int64_t D, int prec, void* stream);
/* dWg(f32 [E,D]) += dscores^T . x  (atomic) */
MD_API int md_moe_gate_wgrad(const float* dscores, const void* x, float* dwg, int64_t rows, int64_t D, int64_t E,
                             int prec, void* stream);

/* ------------------------------------------------------------------------- masking (utils.py:382-426) */
/* get_mask with the uniform noise given: ascending argsort per sample (ties by index).
 * ids_shuffle, ids_restore int32 [B,T]; mask f32 [B,T] (0 keep, 1 drop); keep_rows int32 [B*keep] = global
 * row (b*T + token) of every kept token in shuffle order.  T <= 4096. */
MD_API int md_mask_sort(const float* noise, int32_t* ids_shuffle, int32_t* ids_restore, float* mask,
                        int32_t* keep_rows, int64_t B, int64_t T, int64_t keep, void* stream);
/* f32 row gather / scatter-add (mask_out_token when the mixer maps are Identity, dit.py:386-388,504) */
MD_API int md_gather_rows_f32(const float* x, const int32_t* src_rows, float* y, int64_t rows, int64_t D, void* stream);
MD_API int md_scatter_rows_f32(const float* dy, const int32_t* src_rows, float* dx, int64_t rows, int64_t D,
                               void* stream);

/* ---------------------------------------------------------- EDM noise / preconditioning / loss */
/* conditioning *= drop_caption_mask; .float() (model.py:132-139): cap fp16 [B, L*Dc] -> bf16.  keep f64 or NULL;
 * cap_out_f16 (optional, may alias cap_f16) receives the masked fp16 captions (the reference's in-place `*=`). */
MD_API int md_cond_prepare(const void* cap_f16, const double* keep, void* out_bf16, void* cap_out_f16, int64_t B,
                           int64_t per_sample, int prec, void* stream);
/* model.py:182-188,153-166 + the im2col of the patch-embed conv (dit.py:479):
 * sigma = exp(rnd*P_std+P_mean); xn = x + sigma*eps; patches(bf16 [B*T, Kp]) = c_in * xn, column
 * (c*p+i)*p+j, Kp = C*p*p; coef f32 [6,B] = sigma, c_skip, c_out, c_in, c_noise, weight.
 * lat: fp16 (lat_f16=1) or f32.  sigma_in (optional) overrides the draw (sampler path). */
MD_API int md_edm_prepare(const void* lat, int lat_f16, const float* eps, const float* rnd, const float* sigma_in,
                          float p_mean, float p_std, float sigma_data, float* xn, void* patches, float* coef,
                          int64_t B, int64_t C, int64_t H, int64_t W, int64_t p, int prec, void* stream);
/* im2col of the patch-embed conv for the plain DiT.forward entry (dit.py:479,552): patches(bf16 [B*T, C*p*p]) =
 * scale[b] * x, scale f32 [B] or NULL. */
MD_API int md_patchify(const float* x, const float* scale, void* patches, int64_t B, int64_t C, int64_t H, int64_t W,
                       int64_t p, int prec, void* stream);
/* TimestepEmbedder.timestep_embedding (utils.py:265-281): out bf16 [B, dim] = [cos | sin](t * freqs) */
MD_API int md_timestep_embed(const float* t, void* out, int64_t B, int64_t dim, int prec, void* stream);
/* weighted masked MSE (model.py:199-210) straight from the final-layer tokens ftok f32 [B*Tk, p*p*C]
 * (column (i*p+j)*C+c, unpatchify dit.py:566-575); keep_tok int32 [B,Tk] = global rows (b*T + token) of the kept
 * tokens (md_mask_sort's keep_rows) or NULL (all tokens).
 * per_sample f32 [B]; loss f32 [1] += mean (caller zeroes). */
MD_API int md_edm_loss_fwd(const float* ftok, const int32_t* keep_tok, const void* lat, int lat_f16, const float* xn,
                           const float* coef, float* per_sample, float* loss, int64_t B, int64_t C, int64_t H,
                           int64_t W, int64_t p, int64_t Tk, void* stream);
/* d loss / d ftok * gscale[0] (f32 device scalar: the incoming grad_output) -> bf16 [B*Tk, p*p*C] */
MD_API int md_edm_loss_bwd(const float* ftok, const int32_t* keep_tok, const void* lat, int lat_f16, const float* xn,
                           const float* coef, const float* gscale, void* dftok, int64_t B, int64_t C, int64_t H,
                           int64_t W, int64_t p, int64_t Tk, int prec, void* stream);
/* unmask_tokens + unpatchify (utils.py:417-426, dit.py:566-575) + D = c_skip*xn + c_out*F (model.py:173-178).
 * ids_restore int32 [B,T] or NULL; mask_token f32 [p*p*C]; fx (raw network output) and dx (denoised), f32
 * [B,C,H,W]; either may be NULL. */
MD_API int md_edm_output(const float* ftok, const int32_t* ids_restore, const float* mask_token, const float* xn,
                         const float* coef, float* fx, float* dx, int64_t B, int64_t C, int64_t H, int64_t W,
                         int64_t p, int64_t Tk, void* stream);
/* One stage of the fp64 Heun sampler (LatentDiffusion._heun, model.py:260-276) on the state x, x_hat, d_cur (f64
 * [B * sample_numel] each).  The step k is read from *step (device int32) and t_cur = table[k], t_next = table[k+1],
 * t_hat = table[max_steps+1+k] from table (device f64 [2*max_steps+1]), so one captured graph serves every step.
 *   stage 0 (in):      x_hat = x + sqrt(t_hat^2 - t_cur^2) * s_noise * noise[k]   (noise f64 [max_steps, B*sample_numel])
 *   stage 1 (euler):   d_cur = (x_hat - den) / t_hat; x = x_hat + (t_next - t_hat) * d_cur
 *   stage 2 (correct): x = x_hat + (t_next - t_hat) * (0.5 * d_cur + 0.5 * (x - den) / t_next)
 *   stage 3 (next):    *step += 1 (one thread; only `step` is read)
 * Stages 0 and 1 also write the next denoiser input: xin f32 = the new x_hat / x, `copies` (1, or 2 for a CFG batch) times
 * back to back, and sigma f32 [copies*B] = t_hat / t_next.  den: f32 [B * sample_numel] denoiser output.  Every operation
 * is rounded on its own in the association order of the torch expressions (no FMA contraction), so the result is bit-for-bit
 * the eager loop's.  A step index outside [0, max_steps) writes NaN instead of reading outside the table. */
MD_API int md_edm_heun(int stage, double* x, double* x_hat, double* d_cur, const float* den, const double* noise,
                       float* xin, float* sigma, const double* table, int32_t* step, int64_t max_steps, int64_t B,
                       int64_t sample_numel, int64_t copies, double s_noise, void* stream);
/* Classifier-free guidance + EDM preconditioning of a doubled batch (model.py:197-201): ftok f32 [2B*T, p*p*C] holds the
 * cond samples [0, B) then the uncond samples [B, 2B) (no masking), x f32 [B,C,H,W] the denoiser input, sigma f32 [B],
 * cfg f32 [1] (device) the guidance scale.  dx = c_skip*x + c_out*(unc + cfg*(cond - unc)) with c_skip =
 * (1 / (sigma^2 + sigma_data_sq)) * sigma_data_sq and c_out = sigma*sigma_data / sqrt(sigma^2 + sigma_data_sq), each
 * operation rounded on its own like the torch expression it replaces. */
MD_API int md_edm_output_cfg(const float* ftok, const float* x, const float* sigma, const float* cfg, float* dx,
                             float sigma_data, float sigma_data_sq, int64_t B, int64_t C, int64_t H, int64_t W, int64_t p,
                             void* stream);

/* ----------------------------------------------- adjoints for the differentiable DiT.forward (VJP) */
/* adjoint of the unmask_tokens + unpatchify of md_edm_output for the raw output F (utils.py:417-426,
 * dit.py:566-575): dF f32 [B,C,H,W] -> dftok [B*Tk, p*p*C] (column (i*p+j)*C+c; bf16, f32 with prec=1) for the kept
 * tokens only: keep_rows int32 [B*Tk] (md_mask_sort's keep_rows) or NULL (Tk = T).  Masked tokens output the
 * non-trainable mask_token buffer (dit.py:440-443) and receive no gradient. */
MD_API int md_unpatchify_bwd(const float* dF, const int32_t* keep_rows, void* dftok, int64_t B, int64_t C, int64_t H,
                             int64_t W, int64_t p, int64_t Tk, int prec, void* stream);
/* adjoint of md_patchify (col2im of the patch-embed conv, dit.py:479; column (c*p+i)*p+j): dpatches f32 [B*T, C*p*p],
 * scale f32 [B] or NULL -> dx f32 [B,C,H,W] (written, not accumulated).  Inputs are f32 in both precisions. */
MD_API int md_patchify_bwd(const float* dpatches, const float* scale, float* dx, int64_t B, int64_t C, int64_t H,
                           int64_t W, int64_t p, int prec, void* stream);
/* adjoint of md_timestep_embed (utils.py:265-281): dt[b] = sum_i dfreq[b,i] * d[cos|sin](t[b]*w_i)/dt; dfreq f32
 * [B, dim], t f32 [B], dt f32 [B] (written).  One block per sample with a fixed reduction order: deterministic. */
MD_API int md_timestep_embed_bwd(const float* dfreq, const float* t, float* dt, int64_t B, int64_t dim, int prec,
                                 void* stream);

/* ------------------------------------------------------------------------------------ utilities */
/* mean over the L tokens of each sample (dit.py:484): x f32 [B,L,D] -> bf16 [B,D]; bwd: dx[b,l,:] += d[b,:]/L */
MD_API int md_mean_tokens_fwd(const float* x, void* out, int64_t B, int64_t L, int64_t D, int prec, void* stream);
MD_API int md_mean_tokens_bwd(const float* d, float* dx, int64_t B, int64_t L, int64_t D, void* stream);
MD_API int md_cast_f32_bf16(const float* x, void* y, int64_t n, int prec, void* stream);
/* out(f32 [N]) += column sums of x [rows, N] (bf16 if x_bf16 else f32), pitch ld (bias gradients) */
MD_API int md_colsum(const void* x, int x_bf16, int64_t ld, float* out, int64_t rows, int64_t N, void* stream);
/* The same for a fused-SwiGLU gradient du [rows, N = 2 half] in the 32-interleaved column order of MD_EPI_SWIGLU
 * (half % 32 == 0): out(f32 [2 half]) += the column sums in the natural [b1 | b2] order -- column c = 64 j + r goes to
 * 32 j + r (r < 32) or half + 32 j + r - 32, the row map of md_gemm_args.row_interleave -- i.e. the bias gradient of
 * a w1 | w2 stack (dit.py:84-86 with use_bias).  Deterministic mode as md_colsum. */
MD_API int md_colsum_interleaved(const void* x, int x_bf16, int64_t ld, float* out, int64_t rows, int64_t N, int64_t half,
                                 void* stream);
/* W f32 [batch, rows, cols] -> wb bf16 same layout (optional) and wbt bf16 [batch, cols, rows] (optional):
 * the per-step bf16 operand copies of the fp32 master weights (what autocast does per call in the reference).
 * interleave_half = f > 0 (rows == 2f, f % 32 == 0): both copies hold the rows in the 32-interleaved order of the fused
 * SwiGLU GEMMs (w1 rows 0-31, w2 rows 0-31, w1 rows 32-63, ...; MD_EPI_SWIGLU). */
MD_API int md_cast_transpose(const float* w, void* wb, void* wbt, int64_t batch, int64_t rows, int64_t cols,
                             int64_t interleave_half, int prec, void* stream);
/* The same for many matrices of one flat buffer in a single launch: desc (device memory) has one row per matrix, sorted by
 * tile_start; matrix i lives at element `offset` of flat / wb / wbt and owns the 64 x 64 tiles
 * [tile_start, tile_start + tiles_x * ceil(rows / 64)), tiles_x = ceil(cols / 64). */
typedef struct md_cast_desc {
  int64_t offset, rows, cols, half; /* half = interleave_half of md_cast_transpose */
  int64_t need_t;                   /* 0: no transposed copy for this matrix */
  int64_t tile_start, tiles_x;
  int64_t reserved;
} md_cast_desc;
MD_API int md_cast_transpose_multi(const float* flat, void* wb, void* wbt, const md_cast_desc* desc, int64_t n_desc,
                                   int64_t total_tiles, int prec, void* stream);
/* sumsq(f32 [1]) += sum x^2  (gradient-norm clipping, train.py:85-86) */
MD_API int md_sumsq(const float* x, float* sumsq, int64_t n, void* stream);
/* fused (clip-scaled) AdamW on flat fp32 buffers (train.py:39, configs/res_256_pretrain.yaml:50-57):
 * g *= min(1, clip / (sqrt(sumsq[0]) + 1e-6)) if sumsq != NULL and clip > 0; decoupled weight decay; bias correction by
 * step.  If sumsq[0] is not finite (a NaN / Inf gradient, cf. NaNCatcher callbacks.py:47-64) nothing is written and
 * *nonfinite (nullable, i32) is set to 1.  p/g/m/v may be any 16-byte aligned slice of the flat buffers (sharded step). */
MD_API int md_adamw(float* p, const float* g, float* m, float* v, const float* sumsq, float clip, float lr,
                    float beta1, float beta2, float eps, float wd, int64_t step, int32_t* nonfinite, int64_t n,
                    void* stream);
/* md_adamw plus an exponential moving average of the weights in the same pass: p / m / v get the same update as
 * md_adamw (bit-identical: one shared device function), then ema = smoothing * ema + (1 - smoothing) * p_new from the
 * register holding p_new -- 8 more bytes per parameter, p is not read twice.  smoothing in [0, 1].  A non-finite
 * sumsq[0] writes nothing (p, m, v and ema) and sets *nonfinite.  All five pointers 16-byte aligned (float4 body,
 * scalar tail).  Element-wise, no reduction: bit-reproducible with or without deterministic mode. */
MD_API int md_adamw_ema(float* p, const float* g, float* m, float* v, const float* sumsq, float clip, float lr,
                        float beta1, float beta2, float eps, float wd, int64_t step, float* ema, float smoothing,
                        int32_t* nonfinite, int64_t n, void* stream);
/* Exchange a[0, n) and b[0, n) in place (swapping EMA and training weights without a full-size temporary).  a == b and
 * any other overlap of the two ranges are rejected.  Element-wise, no reduction: deterministic mode needs nothing. */
MD_API int md_swap_f32(float* a, float* b, int64_t n, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* MICRODIT_B200_H_ */
