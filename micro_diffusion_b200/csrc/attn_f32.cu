// fp32 attention for the high-precision mode (prec = 1, MD_PRECISION=high): q / k / v / o and their gradients are
// fp32 tensors and every product is an fp32 FMA -- no tensor cores, because this mode exists to gate the host
// sequencing and the hand-derived backward against the fp32 oracle at 1e-3 (it is never the timed path).
// Same contract as md_attn_fwd / md_attn_bwd (F.scaled_dot_product_attention, reference utils.py:188-193, 127-132):
// column-slice operands with row pitches, lse in the log2 domain, delta = rowsum(dO * O) written to the scratch.
//
// One warp per query row (forward, dQ) or per key row (dK / dV): lanes take one key (query) each for the score, then
// the weighted sum over the 32 scores is accumulated with each lane owning head_dim / 32 output columns.  The backward
// kernels read two whole rows in every lane (q and dO, or k and v); up to head_dim 64 they sit in registers, at 128 they
// would spill, so there they live in a per-warp shared-memory copy that the lanes read by broadcast.
#include "common.cuh"

namespace md {
namespace attn_f32 {

constexpr float kLog2e = 1.4426950408889634f;

template <int HD>
__global__ void __launch_bounds__(128)
fwd_kernel(const float* __restrict__ q, long long ldq, const float* __restrict__ k, long long ldk,
           const float* __restrict__ v, long long ldv, float* __restrict__ o, long long ldo, float* __restrict__ lse,
           int H, int Tq, int Tk, long long rows, float scale) {
  constexpr int DPL = HD / 32;  // output columns per lane
  const int lane = threadIdx.x & 31;
  const long long w = 1LL * blockIdx.x * 4 + (threadIdx.x >> 5);
  if (w >= rows) return;
  const int qi = static_cast<int>(w % Tq);
  const int h = static_cast<int>((w / Tq) % H);
  const long long b = w / (1LL * Tq * H);
  const float* qr = q + (b * Tq + qi) * ldq + h * HD;
  float qv[HD];
#pragma unroll
  for (int d = 0; d < HD; ++d) qv[d] = qr[d] * scale;
  float m = -INFINITY, l = 0.f, acc[DPL];
#pragma unroll
  for (int e = 0; e < DPL; ++e) acc[e] = 0.f;
  for (int j0 = 0; j0 < Tk; j0 += 32) {
    const int j = j0 + lane;
    float s = -INFINITY;
    if (j < Tk) {
      const float* kr = k + (b * Tk + j) * ldk + h * HD;
      float a = 0.f;
#pragma unroll
      for (int d = 0; d < HD; ++d) a = fmaf(qv[d], kr[d], a);
      s = a;
    }
    const float mn = fmaxf(m, warp_max(s));
    const float corr = __expf(m - mn);  // exp(-inf) = 0 on the first block
    const float pj = j < Tk ? __expf(s - mn) : 0.f;
    l = l * corr + warp_sum(pj);
#pragma unroll
    for (int e = 0; e < DPL; ++e) acc[e] *= corr;
    const int nj = min(32, Tk - j0);
    for (int t = 0; t < nj; ++t) {
      const float pt = __shfl_sync(0xffffffffu, pj, t);
      const float* vr = v + (b * Tk + j0 + t) * ldv + h * HD;
#pragma unroll
      for (int e = 0; e < DPL; ++e) acc[e] = fmaf(pt, vr[lane + 32 * e], acc[e]);
    }
    m = mn;
  }
  float* orow = o + (b * Tq + qi) * ldo + h * HD;
#pragma unroll
  for (int e = 0; e < DPL; ++e) orow[lane + 32 * e] = acc[e] / l;
  if (lane == 0) lse[(b * H + h) * Tq + qi] = (m + logf(l)) * kLog2e;
}

// dQ (+ delta): warp per query row
template <int HD>
__global__ void __launch_bounds__(128)
dq_kernel(const float* __restrict__ dout, long long lddo, const float* __restrict__ q, long long ldq,
          const float* __restrict__ k, long long ldk, const float* __restrict__ v, long long ldv,
          const float* __restrict__ o, long long ldo, const float* __restrict__ lse, float* __restrict__ delta,
          float* __restrict__ dq, long long lddq, int H, int Tq, int Tk, long long rows, float scale) {
  constexpr int DPL = HD / 32;
  const int lane = threadIdx.x & 31;
  const long long w = 1LL * blockIdx.x * 4 + (threadIdx.x >> 5);
  if (w >= rows) return;
  const int qi = static_cast<int>(w % Tq);
  const int h = static_cast<int>((w / Tq) % H);
  const long long b = w / (1LL * Tq * H);
  const float* qr = q + (b * Tq + qi) * ldq + h * HD;
  const float* dor = dout + (b * Tq + qi) * lddo + h * HD;
  const float* orow = o + (b * Tq + qi) * ldo + h * HD;
  constexpr bool kSmemRows = HD == 128;
  __shared__ float srows[kSmemRows ? 4 * 2 * HD : 1];
  float qreg[kSmemRows ? 1 : HD], doreg[kSmemRows ? 1 : HD];
  float* qv = kSmemRows ? srows + (threadIdx.x >> 5) * 2 * HD : qreg;
  float* dov = kSmemRows ? qv + HD : doreg;
  float dl = 0.f;
  if constexpr (kSmemRows) {
#pragma unroll
    for (int e = 0; e < DPL; ++e) {
      qv[lane + 32 * e] = qr[lane + 32 * e] * scale;
      dov[lane + 32 * e] = dor[lane + 32 * e];
    }
    __syncwarp();
#pragma unroll
    for (int d = 0; d < HD; ++d) dl = fmaf(dov[d], orow[d], dl);
  } else {
#pragma unroll
    for (int d = 0; d < HD; ++d) {
      qv[d] = qr[d] * scale;
      dov[d] = dor[d];
      dl = fmaf(dov[d], orow[d], dl);
    }
  }
  const float lrow = lse[(b * H + h) * Tq + qi];
  if (lane == 0) delta[(b * H + h) * Tq + qi] = dl;
  float acc[DPL];
#pragma unroll
  for (int e = 0; e < DPL; ++e) acc[e] = 0.f;
  for (int j0 = 0; j0 < Tk; j0 += 32) {
    const int j = j0 + lane;
    float ds = 0.f;
    if (j < Tk) {
      const float* kr = k + (b * Tk + j) * ldk + h * HD;
      const float* vr = v + (b * Tk + j) * ldv + h * HD;
      float s = 0.f, dp = 0.f;
#pragma unroll
      for (int d = 0; d < HD; ++d) {
        s = fmaf(qv[d], kr[d], s);
        dp = fmaf(dov[d], vr[d], dp);
      }
      const float pj = exp2f(s * kLog2e - lrow);
      ds = pj * (dp - dl);
    }
    const int nj = min(32, Tk - j0);
    for (int t = 0; t < nj; ++t) {
      const float dt = __shfl_sync(0xffffffffu, ds, t);
      const float* kr = k + (b * Tk + j0 + t) * ldk + h * HD;
#pragma unroll
      for (int e = 0; e < DPL; ++e) acc[e] = fmaf(dt, kr[lane + 32 * e], acc[e]);
    }
  }
  float* dqr = dq + (b * Tq + qi) * lddq + h * HD;
#pragma unroll
  for (int e = 0; e < DPL; ++e) dqr[lane + 32 * e] = acc[e] * scale;
}

// dK, dV: warp per key row
template <int HD>
__global__ void __launch_bounds__(128)
dkdv_kernel(const float* __restrict__ dout, long long lddo, const float* __restrict__ q, long long ldq,
            const float* __restrict__ k, long long ldk, const float* __restrict__ v, long long ldv,
            const float* __restrict__ lse, const float* __restrict__ delta, float* __restrict__ dk, long long lddk,
            float* __restrict__ dv, long long lddv, int H, int Tq, int Tk, long long rows, float scale) {
  constexpr int DPL = HD / 32;
  const int lane = threadIdx.x & 31;
  const long long w = 1LL * blockIdx.x * 4 + (threadIdx.x >> 5);
  if (w >= rows) return;
  const int kj = static_cast<int>(w % Tk);
  const int h = static_cast<int>((w / Tk) % H);
  const long long b = w / (1LL * Tk * H);
  const float* kr = k + (b * Tk + kj) * ldk + h * HD;
  const float* vr = v + (b * Tk + kj) * ldv + h * HD;
  constexpr bool kSmemRows = HD == 128;
  __shared__ float srows[kSmemRows ? 4 * 2 * HD : 1];
  float kreg[kSmemRows ? 1 : HD], vreg[kSmemRows ? 1 : HD];
  float* kv = kSmemRows ? srows + (threadIdx.x >> 5) * 2 * HD : kreg;
  float* vv = kSmemRows ? kv + HD : vreg;
  if constexpr (kSmemRows) {
#pragma unroll
    for (int e = 0; e < DPL; ++e) {
      kv[lane + 32 * e] = kr[lane + 32 * e] * scale;
      vv[lane + 32 * e] = vr[lane + 32 * e];
    }
    __syncwarp();
  } else {
#pragma unroll
    for (int d = 0; d < HD; ++d) {
      kv[d] = kr[d] * scale;
      vv[d] = vr[d];
    }
  }
  float ak[DPL], av[DPL];
#pragma unroll
  for (int e = 0; e < DPL; ++e) ak[e] = av[e] = 0.f;
  for (int i0 = 0; i0 < Tq; i0 += 32) {
    const int i = i0 + lane;
    float pi = 0.f, ds = 0.f;
    if (i < Tq) {
      const float* qr = q + (b * Tq + i) * ldq + h * HD;
      const float* dor = dout + (b * Tq + i) * lddo + h * HD;
      float s = 0.f, dp = 0.f;
#pragma unroll
      for (int d = 0; d < HD; ++d) {
        s = fmaf(qr[d], kv[d], s);
        dp = fmaf(dor[d], vv[d], dp);
      }
      pi = exp2f(s * kLog2e - lse[(b * H + h) * Tq + i]);
      ds = pi * (dp - delta[(b * H + h) * Tq + i]);
    }
    const int ni = min(32, Tq - i0);
    for (int t = 0; t < ni; ++t) {
      const float pt = __shfl_sync(0xffffffffu, pi, t);
      const float dt = __shfl_sync(0xffffffffu, ds, t);
      const float* qr = q + (b * Tq + i0 + t) * ldq + h * HD;
      const float* dor = dout + (b * Tq + i0 + t) * lddo + h * HD;
#pragma unroll
      for (int e = 0; e < DPL; ++e) {
        av[e] = fmaf(pt, dor[lane + 32 * e], av[e]);
        ak[e] = fmaf(dt, qr[lane + 32 * e], ak[e]);
      }
    }
  }
  float* dkr = dk + (b * Tk + kj) * lddk + h * HD;
  float* dvr = dv + (b * Tk + kj) * lddv + h * HD;
#pragma unroll
  for (int e = 0; e < DPL; ++e) {
    dkr[lane + 32 * e] = ak[e] * scale;
    dvr[lane + 32 * e] = av[e];
  }
}

}  // namespace attn_f32
}  // namespace md

using namespace md;
#define ST(s) reinterpret_cast<cudaStream_t>(s)
#define CF(p) reinterpret_cast<const float*>(p)
#define F(p) reinterpret_cast<float*>(p)

extern "C" int md_attn_fwd_f32(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, void* o,
                               int64_t ldo, float* lse, int64_t B, int64_t H, int64_t Tq, int64_t Tk, int64_t hd,
                               void* stream) {
  if (B <= 0 || H <= 0 || Tq <= 0 || Tk <= 0) return B == 0 ? 0 : md_set_error(MD_ERR_INVALID, "md_attn_fwd_f32: bad sizes");
  if (hd != 32 && hd != 64 && hd != 128)
    return md_set_error(MD_ERR_UNSUPPORTED, "md_attn_fwd_f32: head_dim must be 32, 64 or 128");
  if (!q || !k || !v || !o || !lse) return md_set_error(MD_ERR_INVALID, "md_attn_fwd_f32: null pointer");
  const long long rows = B * H * Tq;
  const unsigned grid = static_cast<unsigned>((rows + 3) / 4);
  const float scale = 1.f / sqrtf(static_cast<float>(hd));
  if (hd == 128)
    attn_f32::fwd_kernel<128><<<grid, 128, 0, ST(stream)>>>(CF(q), ldq, CF(k), ldk, CF(v), ldv, F(o), ldo, lse, (int)H, (int)Tq,
                                                            (int)Tk, rows, scale);
  else if (hd == 64)
    attn_f32::fwd_kernel<64><<<grid, 128, 0, ST(stream)>>>(CF(q), ldq, CF(k), ldk, CF(v), ldv, F(o), ldo, lse, (int)H, (int)Tq,
                                                           (int)Tk, rows, scale);
  else
    attn_f32::fwd_kernel<32><<<grid, 128, 0, ST(stream)>>>(CF(q), ldq, CF(k), ldk, CF(v), ldv, F(o), ldo, lse, (int)H, (int)Tq,
                                                           (int)Tk, rows, scale);
  return check_launch("md_attn_fwd_f32");
}

extern "C" int md_attn_bwd_f32(const void* dout, int64_t lddo, const void* q, int64_t ldq, const void* k, int64_t ldk,
                               const void* v, int64_t ldv, const void* o, int64_t ldo, const float* lse, float* delta,
                               void* dq, int64_t lddq, void* dk, int64_t lddk, void* dv, int64_t lddv, int64_t B, int64_t H,
                               int64_t Tq, int64_t Tk, int64_t hd, void* stream) {
  if (B <= 0 || H <= 0 || Tq <= 0 || Tk <= 0) return B == 0 ? 0 : md_set_error(MD_ERR_INVALID, "md_attn_bwd_f32: bad sizes");
  if (hd != 32 && hd != 64 && hd != 128)
    return md_set_error(MD_ERR_UNSUPPORTED, "md_attn_bwd_f32: head_dim must be 32, 64 or 128");
  if (!dout || !q || !k || !v || !o || !lse || !delta || !dq || !dk || !dv)
    return md_set_error(MD_ERR_INVALID, "md_attn_bwd_f32: null pointer");
  const long long qrows = B * H * Tq, krows = B * H * Tk;
  const float scale = 1.f / sqrtf(static_cast<float>(hd));
#define BWD(HD_)                                                                                                       \
  do {                                                                                                                 \
    attn_f32::dq_kernel<HD_><<<(unsigned)((qrows + 3) / 4), 128, 0, ST(stream)>>>(                                     \
        CF(dout), lddo, CF(q), ldq, CF(k), ldk, CF(v), ldv, CF(o), ldo, lse, delta, F(dq), lddq, (int)H, (int)Tq,      \
        (int)Tk, qrows, scale);                                                                                        \
    attn_f32::dkdv_kernel<HD_><<<(unsigned)((krows + 3) / 4), 128, 0, ST(stream)>>>(                                   \
        CF(dout), lddo, CF(q), ldq, CF(k), ldk, CF(v), ldv, lse, delta, F(dk), lddk, F(dv), lddv, (int)H, (int)Tq,     \
        (int)Tk, krows, scale);                                                                                        \
  } while (0)
  if (hd == 128) BWD(128);
  else if (hd == 64) BWD(64);
  else BWD(32);
#undef BWD
  return check_launch("md_attn_bwd_f32");
}

// ------------------------------------------------------------------------------------------------ 3-way bf16 split
// High-precision GEMMs run on the SAME wgmma kernel: an fp32 operand x is written as bf16 triples hi = bf16(x),
// lo = bf16(x - hi), laid out along the contraction so that one bf16 GEMM of 3x the depth accumulates
//   a_hi b_hi + a_lo b_hi + a_hi b_lo      (error ~2^-17 relative: the missing a_lo b_lo term)
// in fp32 registers.  role 0 (the "A" pattern) emits [hi | lo | hi], role 1 (the "B" pattern) [hi | hi | lo].
//   along == 0: x [batch][rows][cols] -> out [batch][rows][3*cols]   (K-major operands: contraction = columns)
//   along == 1: x [batch][rows][cols] -> out [batch][3*rows][cols]   (MN-major operands: contraction = rows)
namespace md {
__global__ void split3_kernel(const float* __restrict__ x, long long ldx, long long bstride, __nv_bfloat16* __restrict__ out,
                              long long rows, long long cols, int role, int along) {
  const long long b = blockIdx.y;
  const long long total = rows * cols;
  for (long long i = 1LL * blockIdx.x * blockDim.x + threadIdx.x; i < total; i += 1LL * gridDim.x * blockDim.x) {
    const long long r = i / cols, c = i % cols;
    const float v = x[b * bstride + r * ldx + c];
    const __nv_bfloat16 hi = __float2bfloat16_rn(v);
    const __nv_bfloat16 lo = __float2bfloat16_rn(v - __bfloat162float(hi));
    const __nv_bfloat16 p1 = role == 0 ? lo : hi, p2 = role == 0 ? hi : lo;
    if (along == 0) {
      __nv_bfloat16* o = out + (b * rows + r) * 3 * cols;
      o[c] = hi; o[cols + c] = p1; o[2 * cols + c] = p2;
    } else {
      __nv_bfloat16* o = out + b * 3 * rows * cols;
      o[r * cols + c] = hi; o[(rows + r) * cols + c] = p1; o[(2 * rows + r) * cols + c] = p2;
    }
  }
}
}  // namespace md

extern "C" int md_split3_bf16(const float* x, int64_t ldx, int64_t batch_stride, void* out, int64_t batch, int64_t rows,
                              int64_t cols, int role, int along, void* stream) {
  if (batch * rows * cols == 0) return 0;
  if (!x || !out || role < 0 || role > 1 || along < 0 || along > 1)
    return md_set_error(MD_ERR_INVALID, "md_split3_bf16: bad argument");
  long long blocks = (rows * cols + 255) / 256;
  if (blocks > 132 * 8) blocks = 132 * 8;
  dim3 grid(static_cast<unsigned>(blocks), static_cast<unsigned>(batch));
  split3_kernel<<<grid, 256, 0, ST(stream)>>>(x, ldx, batch_stride, reinterpret_cast<__nv_bfloat16*>(out), rows, cols, role,
                                              along);
  return check_launch("md_split3_bf16");
}
