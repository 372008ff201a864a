// HBM-bound element-wise / reduction tails of the MicroDiT hot path: SwiGLU, activation backward,
// conditioning GELU, token mean, casts, bias gradients (column sums), per-step bf16 weight copies,
// timestep sinusoid, caption-drop cast, gradient sum-of-squares and fused AdamW.
// 16-byte vector accesses, grids sized as multiples of the SM count with grid-stride loops.
#include <cuda_fp16.h>

#include "act.cuh"

namespace md {

static int grid_for(long long work_items, int threads) {
  long long blocks = (work_items + threads - 1) / threads;
  const long long cap = 132LL * 16;  // 16 resident 256-thread CTAs worth of waves per SM
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  return static_cast<int>(blocks);
}

__device__ __forceinline__ void unpack8(const uint4& r, float (&f)[8]) {
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&r);
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    f[2 * e] = __low2float(h[e]);
    f[2 * e + 1] = __high2float(h[e]);
  }
}
__device__ __forceinline__ uint4 pack8(const float (&f)[8]) {
  uint4 r;
  __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&r);
#pragma unroll
  for (int e = 0; e < 4; ++e) h[e] = __floats2bfloat162_rn(f[2 * e], f[2 * e + 1]);
  return r;
}
__device__ __forceinline__ float silu_f(float x) { return x / (1.f + __expf(-x)); }

// ------------------------------------------------------------------------------------------ SwiGLU
template <typename AT>
__global__ void swiglu_fwd_kernel(const AT* __restrict__ u, AT* __restrict__ h, long long rows, int f) {
  const int fv = f >> 3;
  const long long total = rows * fv;
  for (long long i = 1LL * blockIdx.x * blockDim.x + threadIdx.x; i < total; i += 1LL * gridDim.x * blockDim.x) {
    const long long r = i / fv;
    const int c = static_cast<int>(i % fv) * 8;
    float a[8], b[8], o[8];
    ld8(u + r * 2 * f + c, a);
    ld8(u + r * 2 * f + f + c, b);
#pragma unroll
    for (int e = 0; e < 8; ++e) o[e] = silu_f(a[e]) * b[e];
    st8(h + r * f + c, o);
  }
}
template <typename AT>
__global__ void swiglu_bwd_kernel(const AT* __restrict__ dh, const AT* __restrict__ u, AT* __restrict__ du, long long rows,
                                  int f) {
  const int fv = f >> 3;
  const long long total = rows * fv;
  for (long long i = 1LL * blockIdx.x * blockDim.x + threadIdx.x; i < total; i += 1LL * gridDim.x * blockDim.x) {
    const long long r = i / fv;
    const int c = static_cast<int>(i % fv) * 8;
    float a[8], b[8], d[8], da[8], db[8];
    ld8(u + r * 2 * f + c, a);
    ld8(u + r * 2 * f + f + c, b);
    ld8(dh + r * f + c, d);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const float sg = 1.f / (1.f + __expf(-a[e]));
      const float sl = a[e] * sg;
      da[e] = d[e] * b[e] * (sg * (1.f + a[e] * (1.f - sg)));
      db[e] = d[e] * sl;
    }
    st8(du + r * 2 * f + c, da);
    st8(du + r * 2 * f + f + c, db);
  }
}

// ---------------------------------------------------------------------------------------- act fwd
template <typename AT>
__global__ void act_fwd_kernel(const AT* __restrict__ pre, AT* __restrict__ out, long long nvec, int act) {
  for (long long i = 1LL * blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += 1LL * gridDim.x * blockDim.x) {
    float x[8], o[8];
    ld8(pre + 8 * i, x);
#pragma unroll
    for (int e = 0; e < 8; ++e) o[e] = act ? gelu_tanh_f(x[e]) : gelu_erf_f(x[e]);
    st8(out + 8 * i, o);
  }
}

// ---------------------------------------------------------------------------------------- act bwd
template <typename AT>
__global__ void act_bwd_kernel(const AT* __restrict__ dact, const AT* __restrict__ pre, AT* __restrict__ dpre,
                               long long nvec, int act) {
  for (long long i = 1LL * blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += 1LL * gridDim.x * blockDim.x) {
    float d[8], x[8], o[8];
    ld8(dact + 8 * i, d);
    ld8(pre + 8 * i, x);
#pragma unroll
    for (int e = 0; e < 8; ++e) o[e] = d[e] * (act ? gelu_tanh_grad_f(x[e]) : gelu_erf_grad_f(x[e]));
    st8(dpre + 8 * i, o);
  }
}
template <typename AT>
__global__ void gelu_tanh_f32_fwd_kernel(const float* __restrict__ c, AT* __restrict__ out, long long n) {
  for (long long i = 1LL * blockIdx.x * blockDim.x + threadIdx.x; i < n; i += 1LL * gridDim.x * blockDim.x)
    st1a(out + i, gelu_tanh_f(c[i]));
}
__global__ void gelu_tanh_f32_bwd_kernel(const float* __restrict__ dact, const float* __restrict__ c,
                                         float* __restrict__ dc, int accumulate, long long n) {
  for (long long i = 1LL * blockIdx.x * blockDim.x + threadIdx.x; i < n; i += 1LL * gridDim.x * blockDim.x) {
    const float v = dact[i] * gelu_tanh_grad_f(c[i]);
    dc[i] = accumulate ? dc[i] + v : v;
  }
}

// -------------------------------------------------------------------------------------- token mean
template <typename AT>
__global__ void mean_tokens_fwd_kernel(const float* __restrict__ x, AT* __restrict__ out, int L, int D) {
  const long long b = blockIdx.y;
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= D) return;
  float s = 0.f;
  for (int l = 0; l < L; ++l) s += x[(b * L + l) * D + c];
  st1a(out + b * D + c, s / L);
}
__global__ void mean_tokens_bwd_kernel(const float* __restrict__ d, float* __restrict__ dx, int L, int D) {
  const long long b = blockIdx.y;
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= D) return;
  const float v = d[b * D + c] / L;
  for (int l = 0; l < L; ++l) dx[(b * L + l) * D + c] += v;
}

__global__ void cast_f32_bf16_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ y, long long n) {
  const long long nv = n >> 2;
  for (long long i = 1LL * blockIdx.x * blockDim.x + threadIdx.x; i < nv; i += 1LL * gridDim.x * blockDim.x) {
    const float4 v = *reinterpret_cast<const float4*>(x + 4 * i);
    __nv_bfloat162 a = __floats2bfloat162_rn(v.x, v.y), b = __floats2bfloat162_rn(v.z, v.w);
    uint2 raw;
    raw.x = *reinterpret_cast<uint32_t*>(&a);
    raw.y = *reinterpret_cast<uint32_t*>(&b);
    *reinterpret_cast<uint2*>(y + 4 * i) = raw;
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
    const long long i = (nv << 2) + threadIdx.x;
    y[i] = __float2bfloat16_rn(x[i]);
  }
}

__global__ void copy_f32_kernel(const float* __restrict__ x, float* __restrict__ y, long long n) {
  for (long long i = 1LL * blockIdx.x * blockDim.x + threadIdx.x; i < n; i += 1LL * gridDim.x * blockDim.x) y[i] = x[i];
}

// ------------------------------------------------------------------------------------------ colsum
// grid (ceil(N/256), ceil(rows/256)): each thread owns one column of a 256-row slab.
// half > 0: x holds the 2 half columns of a fused-SwiGLU output in the 32-interleaved order (u1 block j, u2 block j, ...);
// column c = 64 j + r lands at 32 j + r (r < 32, b1) or half + 32 j + r - 32 (b2) of out, the [b1 | b2] order.
template <bool kInterleaved>
__global__ void colsum_kernel(const void* __restrict__ x, int x_bf16, long long ld, float* __restrict__ out,
                              long long rows, long long N, float* __restrict__ ws, long long half) {
  const long long c = 1LL * blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= N) return;
  long long oc = c;
  if constexpr (kInterleaved) {
    const long long j = c >> 6, r = c & 63;
    oc = (r < 32 ? 0 : half - 32) + 32 * j + r;
  }
  const long long r0 = 1LL * blockIdx.y * 256, r1 = min(rows, r0 + 256);
  float s = 0.f;
  if (x_bf16) {
    const __nv_bfloat16* p = reinterpret_cast<const __nv_bfloat16*>(x);
    for (long long r = r0; r < r1; ++r) s += __bfloat162float(p[r * ld + c]);
  } else {
    const float* p = reinterpret_cast<const float*>(x);
    for (long long r = r0; r < r1; ++r) s += p[r * ld + c];
  }
  if (ws != nullptr) ws[1LL * blockIdx.y * N + oc] = s;   // deterministic mode: slab partials, fixed-order reduction afterwards
  else atomicAdd(out + oc, s);
}

// ---------------------------------------------------------------------------------- cast_transpose
// 64x64 tiles, 256 threads: 16-byte fp32 loads, 8-byte bf16 stores in both orientations (the transposed one through
// a padded smem tile).  HBM-bound: 4 B read + 2 x 2 B written per element.
template <typename AT>
__device__ __forceinline__ void cast_transpose_tile(const float* __restrict__ wsrc, AT* __restrict__ wb_, AT* __restrict__ wbt_,
                                                    long long rows, long long cols, long long half, long long c0,
                                                    long long r0, float (&tile)[64][65]) {
  // half > 0 (rows == 2 * half, half % 32 == 0): the copies hold the rows in the 32-interleaved order of the fused SwiGLU
  // GEMMs -- input row r (< half: w1, else w2) becomes row 64 * (r' / 32) + (w2 ? 32 : 0) + r' % 32, r' = r mod half
  auto prow = [&](long long r) -> long long {
    if (half <= 0) return r;
    const long long rr = r < half ? r : r - half;
    return 64 * (rr >> 5) + (r < half ? 0 : 32) + (rr & 31);
  };
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;  // 16 x 16 threads, 4 columns each, 4 row passes
  const bool vec = ((cols & 3) == 0) && ((rows & 3) == 0);
#pragma unroll
  for (int pass = 0; pass < 4; ++pass) {
    const long long r = r0 + ty + 16 * pass, c = c0 + 4 * tx;
    float v[4] = {0.f, 0.f, 0.f, 0.f};
    if (r < rows) {
      if (vec && c + 3 < cols) {
        const float4 f = *reinterpret_cast<const float4*>(wsrc + r * cols + c);
        v[0] = f.x; v[1] = f.y; v[2] = f.z; v[3] = f.w;
        if (wb_) st4a(wb_ + prow(r) * cols + c, f);
      } else {
        for (int e = 0; e < 4; ++e)
          if (c + e < cols) {
            v[e] = wsrc[r * cols + c + e];
            if (wb_) st1a(wb_ + prow(r) * cols + c + e, v[e]);
          }
      }
    }
#pragma unroll
    for (int e = 0; e < 4; ++e) tile[ty + 16 * pass][4 * tx + e] = v[e];
  }
  __syncthreads();
  if (wbt_ == nullptr) return;
#pragma unroll
  for (int pass = 0; pass < 4; ++pass) {
    const long long c = c0 + ty + 16 * pass;  // output row = original column
    const long long r = r0 + 4 * tx;          // output columns = original rows r .. r+3
    if (c >= cols) continue;
    float v[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) v[e] = tile[4 * tx + e][ty + 16 * pass];
    AT* dst = wbt_ + c * rows;
    if (vec && r + 3 < rows) {   // r % 4 == 0: the four rows stay adjacent under the 32-row interleave
      st4a(dst + prow(r), make_float4(v[0], v[1], v[2], v[3]));
    } else {
      for (int e = 0; e < 4; ++e)
        if (r + e < rows) st1a(dst + prow(r + e), v[e]);
    }
  }
}

template <typename AT>
__global__ void __launch_bounds__(256)
cast_transpose_kernel(const float* __restrict__ w, AT* __restrict__ wb, AT* __restrict__ wbt, long long rows,
                      long long cols, long long half) {
  __shared__ float tile[64][65];
  const long long o = 1LL * blockIdx.z * rows * cols;
  cast_transpose_tile<AT>(w + o, wb ? wb + o : nullptr, wbt ? wbt + o : nullptr, rows, cols, half, 1LL * blockIdx.x * 64,
                          1LL * blockIdx.y * 64, tile);
}

// All weight matrices of a range in ONE launch: a table of (offset, shape, first tile) rows, one per matrix, and a
// binary search from the block index to its matrix.  Per optimizer step the bf16 copies were 222 launches of mostly
// tiny matrices -- 3.7 ms of a 125 ms rank step at 8 GPUs.
template <typename AT>
__global__ void __launch_bounds__(256)
cast_transpose_multi_kernel(const float* __restrict__ flat, AT* __restrict__ wb, AT* __restrict__ wbt,
                            const md_cast_desc* __restrict__ desc, int n_desc) {
  __shared__ float tile[64][65];
  int lo = 0, hi = n_desc - 1;
  const long long id = blockIdx.x;
  while (lo < hi) {  // last descriptor whose tile_start <= id
    const int mid = (lo + hi + 1) >> 1;
    if (desc[mid].tile_start <= id) lo = mid;
    else hi = mid - 1;
  }
  const md_cast_desc d = desc[lo];
  const long long local = id - d.tile_start;
  const long long bx = local % d.tiles_x, by = local / d.tiles_x;
  cast_transpose_tile<AT>(flat + d.offset, wb + d.offset, d.need_t ? wbt + d.offset : nullptr, d.rows, d.cols, d.half,
                          bx * 64, by * 64, tile);
}

// -------------------------------------------------------------------------------- timestep / cond
template <typename AT>
__global__ void timestep_embed_kernel(const float* __restrict__ t, AT* __restrict__ out, int dim) {
  const long long b = blockIdx.x;
  const int half = dim / 2;
  const float tv = t[b];
  for (int i = threadIdx.x; i < half; i += blockDim.x) {
    const float freq = expf(-9.210340371976184f * static_cast<float>(i) / static_cast<float>(half));
    const float a = tv * freq;
    st1a(out + b * dim + i, cosf(a));
    st1a(out + b * dim + half + i, sinf(a));
  }
  if ((dim & 1) && threadIdx.x == 0) st1a(out + b * dim + dim - 1, 0.f);
}

template <typename AT>
__global__ void cond_prepare_kernel(const __half* cap, const double* __restrict__ keep, AT* __restrict__ out,
                                    __half* cap_out, long long per_sample) {
  const long long b = blockIdx.y;
  const float k = keep ? static_cast<float>(keep[b]) : 1.f;
  const long long nv = per_sample >> 3;
  for (long long i = 1LL * blockIdx.x * blockDim.x + threadIdx.x; i < nv; i += 1LL * gridDim.x * blockDim.x) {
    const uint4 raw = *reinterpret_cast<const uint4*>(cap + b * per_sample + 8 * i);
    const __half2* h = reinterpret_cast<const __half2*>(&raw);
    float o[8];
    uint4 masked;
    __half2* mh = reinterpret_cast<__half2*>(&masked);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      // the reference multiplies in fp16 (in-place `conditioning *= mask`, model.py:132-135), then .float()
      const __half2 m = __hmul2(h[e], __float2half2_rn(k));
      mh[e] = m;
      const float2 f = __half22float2(m);
      o[2 * e] = f.x;
      o[2 * e + 1] = f.y;
    }
    st8(out + b * per_sample + 8 * i, o);
    if (cap_out) *reinterpret_cast<uint4*>(cap_out + b * per_sample + 8 * i) = masked;
  }
}

// ----------------------------------------------------------------------------------- sumsq / AdamW
__global__ void sumsq_kernel(const float* __restrict__ x, float* __restrict__ out, long long n, float* __restrict__ ws) {
  float s = 0.f;
  const long long nv = n >> 2;
  for (long long i = 1LL * blockIdx.x * blockDim.x + threadIdx.x; i < nv; i += 1LL * gridDim.x * blockDim.x) {
    const float4 v = *reinterpret_cast<const float4*>(x + 4 * i);
    s += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
    const float v = x[(nv << 2) + threadIdx.x];
    s += v * v;
  }
  s = warp_sum(s);
  __shared__ float part[32];
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 32) {
    float v = threadIdx.x < (blockDim.x >> 5) ? part[threadIdx.x] : 0.f;
    v = warp_sum(v);
    if (threadIdx.x == 0) {
      if (ws != nullptr) ws[blockIdx.x] = v;   // deterministic mode
      else atomicAdd(out, v);
    }
  }
}

// One parameter's AdamW update, in place.  md_adamw and md_adamw_ema both run exactly this, so their p / m / v agree
// bit for bit.  The moment updates spell out their FMA (m = b1 m + (1 - b1) gg, v = b2 v + (1 - b2) gg^2), which the
// compiler would otherwise contract differently at different call sites.
__device__ __forceinline__ void adamw_elem(float& p, float g, float& m, float& v, float gs, float lr, float b1, float b2,
                                           float eps, float wd, float bc1, float bc2) {
  const float gg = g * gs;
  p *= 1.f - lr * wd;
  m = __fmaf_rn(1.f - b1, gg, b1 * m);
  v = __fmaf_rn(gg, (1.f - b2) * gg, b2 * v);
  const float denom = sqrtf(v) / sqrtf(bc2) + eps;
  p -= (lr / bc1) * m / denom;
}

// kEma: also ema = s * ema + (1 - s) * p_new, from the register that holds p_new (8 more bytes per parameter).
template <bool kEma>
__global__ void adamw_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                             float* __restrict__ v, const float* __restrict__ sumsq, float clip, float lr, float b1,
                             float b2, float eps, float wd, float bc1, float bc2, int* __restrict__ nonfinite,
                             long long n, float* __restrict__ ema, float s) {
  float gs = 1.f;
  if (sumsq != nullptr) {
    const float ss = sumsq[0];
    if (!isfinite(ss)) {  // a NaN / Inf gradient anywhere: leave weights, moments and EMA untouched (NaNCatcher, callbacks.py:47-64)
      if (nonfinite != nullptr && blockIdx.x == 0 && threadIdx.x == 0) *nonfinite = 1;
      return;
    }
    if (clip > 0.f) gs = fminf(1.f, clip / (sqrtf(ss) + 1e-6f));
  }
  const float s1 = 1.f - s;
  const long long nv = n >> 2;
  for (long long i = 1LL * blockIdx.x * blockDim.x + threadIdx.x; i < nv; i += 1LL * gridDim.x * blockDim.x) {
    float4 pv = *reinterpret_cast<float4*>(p + 4 * i);
    const float4 gv = *reinterpret_cast<const float4*>(g + 4 * i);
    float4 mv = *reinterpret_cast<float4*>(m + 4 * i);
    float4 vv = *reinterpret_cast<float4*>(v + 4 * i);
    float* pp = reinterpret_cast<float*>(&pv);
    const float* gp = reinterpret_cast<const float*>(&gv);
    float* mp = reinterpret_cast<float*>(&mv);
    float* vp = reinterpret_cast<float*>(&vv);
#pragma unroll
    for (int e = 0; e < 4; ++e) adamw_elem(pp[e], gp[e], mp[e], vp[e], gs, lr, b1, b2, eps, wd, bc1, bc2);
    *reinterpret_cast<float4*>(p + 4 * i) = pv;
    *reinterpret_cast<float4*>(m + 4 * i) = mv;
    *reinterpret_cast<float4*>(v + 4 * i) = vv;
    if (kEma) {
      float4 ev = *reinterpret_cast<float4*>(ema + 4 * i);
      ev.x = s * ev.x + s1 * pv.x;
      ev.y = s * ev.y + s1 * pv.y;
      ev.z = s * ev.z + s1 * pv.z;
      ev.w = s * ev.w + s1 * pv.w;
      *reinterpret_cast<float4*>(ema + 4 * i) = ev;
    }
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
    const long long i = (nv << 2) + threadIdx.x;
    float pp = p[i], mm = m[i], vv = v[i];
    adamw_elem(pp, g[i], mm, vv, gs, lr, b1, b2, eps, wd, bc1, bc2);
    p[i] = pp; m[i] = mm; v[i] = vv;
    if (kEma) ema[i] = s * ema[i] + s1 * pp;
  }
}

// a <-> b, element by element (kVec: both 16-byte aligned, float4 body + scalar tail)
template <bool kVec>
__global__ void swap_f32_kernel(float* __restrict__ a, float* __restrict__ b, long long n) {
  const long long stride = 1LL * gridDim.x * blockDim.x;
  long long i = 1LL * blockIdx.x * blockDim.x + threadIdx.x;
  if (kVec) {
    const long long nv = n >> 2;
    for (; i < nv; i += stride) {
      const float4 x = *reinterpret_cast<const float4*>(a + 4 * i);
      const float4 y = *reinterpret_cast<const float4*>(b + 4 * i);
      *reinterpret_cast<float4*>(a + 4 * i) = y;
      *reinterpret_cast<float4*>(b + 4 * i) = x;
    }
    if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
      const long long j = (nv << 2) + threadIdx.x;
      const float x = a[j];
      a[j] = b[j];
      b[j] = x;
    }
  } else {
    for (; i < n; i += stride) {
      const float x = a[i];
      a[i] = b[i];
      b[i] = x;
    }
  }
}

}  // namespace md

using namespace md;
#define ST(s) reinterpret_cast<cudaStream_t>(s)
#define BF(p) reinterpret_cast<__nv_bfloat16*>(p)
#define CBF(p) reinterpret_cast<const __nv_bfloat16*>(p)

extern "C" int md_swiglu_fwd(const void* u, void* h, int64_t rows, int64_t f, int prec, void* stream) {
  if (rows == 0) return 0;
  if (!u || !h || f % 8 != 0) return md_set_error(MD_ERR_INVALID, "md_swiglu_fwd: null pointer or f % 8 != 0");
  MD_WITH_ACT(prec, swiglu_fwd_kernel<AT><<<grid_for(rows * (f / 8), 256), 256, 0, ST(stream)>>>(CAP(AT, u), AP(AT, h), rows, (int)f));
  return check_launch("md_swiglu_fwd");
}
extern "C" int md_swiglu_bwd(const void* dh, const void* u, void* du, int64_t rows, int64_t f, int prec, void* stream) {
  if (rows == 0) return 0;
  if (!dh || !u || !du || f % 8 != 0) return md_set_error(MD_ERR_INVALID, "md_swiglu_bwd: null pointer or f % 8 != 0");
  MD_WITH_ACT(prec, swiglu_bwd_kernel<AT><<<grid_for(rows * (f / 8), 256), 256, 0, ST(stream)>>>(CAP(AT, dh), CAP(AT, u), AP(AT, du), rows, (int)f));
  return check_launch("md_swiglu_bwd");
}
extern "C" int md_act_fwd(const void* pre, void* out, int64_t n, int act, int prec, void* stream) {
  if (n == 0) return 0;
  if (!pre || !out || n % 8 != 0) return md_set_error(MD_ERR_INVALID, "md_act_fwd: null pointer or n % 8 != 0");
  MD_WITH_ACT(prec, act_fwd_kernel<AT><<<grid_for(n / 8, 256), 256, 0, ST(stream)>>>(CAP(AT, pre), AP(AT, out), n / 8, act));
  return check_launch("md_act_fwd");
}
extern "C" int md_act_bwd(const void* dact, const void* pre, void* dpre, int64_t n, int act, int prec, void* stream) {
  if (n == 0) return 0;
  if (!dact || !pre || !dpre || n % 8 != 0) return md_set_error(MD_ERR_INVALID, "md_act_bwd: null pointer or n % 8 != 0");
  MD_WITH_ACT(prec, act_bwd_kernel<AT><<<grid_for(n / 8, 256), 256, 0, ST(stream)>>>(CAP(AT, dact), CAP(AT, pre), AP(AT, dpre), n / 8, act));
  return check_launch("md_act_bwd");
}
extern "C" int md_gelu_tanh_f32_fwd(const float* c, void* out, int64_t n, int prec, void* stream) {
  if (n == 0) return 0;
  if (!c || !out) return md_set_error(MD_ERR_INVALID, "md_gelu_tanh_f32_fwd: null pointer");
  MD_WITH_ACT(prec, gelu_tanh_f32_fwd_kernel<AT><<<grid_for(n, 256), 256, 0, ST(stream)>>>(c, AP(AT, out), n));
  return check_launch("md_gelu_tanh_f32_fwd");
}
extern "C" int md_gelu_tanh_f32_bwd(const float* dact, const float* c, float* dc, int accumulate, int64_t n,
                                    void* stream) {
  if (n == 0) return 0;
  if (!dact || !c || !dc) return md_set_error(MD_ERR_INVALID, "md_gelu_tanh_f32_bwd: null pointer");
  gelu_tanh_f32_bwd_kernel<<<grid_for(n, 256), 256, 0, ST(stream)>>>(dact, c, dc, accumulate, n);
  return check_launch("md_gelu_tanh_f32_bwd");
}
extern "C" int md_mean_tokens_fwd(const float* x, void* out, int64_t B, int64_t L, int64_t D, int prec, void* stream) {
  if (B == 0) return 0;
  if (!x || !out) return md_set_error(MD_ERR_INVALID, "md_mean_tokens_fwd: null pointer");
  dim3 grid((unsigned)((D + 127) / 128), (unsigned)B);
  MD_WITH_ACT(prec, mean_tokens_fwd_kernel<AT><<<grid, 128, 0, ST(stream)>>>(x, AP(AT, out), (int)L, (int)D));
  return check_launch("md_mean_tokens_fwd");
}
extern "C" int md_mean_tokens_bwd(const float* d, float* dx, int64_t B, int64_t L, int64_t D, void* stream) {
  if (B == 0) return 0;
  if (!d || !dx) return md_set_error(MD_ERR_INVALID, "md_mean_tokens_bwd: null pointer");
  dim3 grid((unsigned)((D + 127) / 128), (unsigned)B);
  mean_tokens_bwd_kernel<<<grid, 128, 0, ST(stream)>>>(d, dx, (int)L, (int)D);
  return check_launch("md_mean_tokens_bwd");
}
extern "C" int md_cast_f32_bf16(const float* x, void* y, int64_t n, int prec, void* stream) {
  if (n == 0) return 0;
  if (!x || !y) return md_set_error(MD_ERR_INVALID, "md_cast_f32_bf16: null pointer");
  if (prec) copy_f32_kernel<<<grid_for(n, 256), 256, 0, ST(stream)>>>(x, reinterpret_cast<float*>(y), n);
  else cast_f32_bf16_kernel<<<grid_for(n / 4 + 1, 256), 256, 0, ST(stream)>>>(x, BF(y), n);
  return check_launch("md_cast_f32_bf16");
}
extern "C" int md_colsum(const void* x, int x_bf16, int64_t ld, float* out, int64_t rows, int64_t N, void* stream) {
  if (rows == 0 || N == 0) return 0;
  if (!x || !out) return md_set_error(MD_ERR_INVALID, "md_colsum: null pointer");
  dim3 grid((unsigned)((N + 255) / 256), (unsigned)((rows + 255) / 256));
  float* ws = nullptr;
  if (det_enabled()) {
    ws = det_workspace(static_cast<size_t>(grid.y) * N * sizeof(float));
    if (ws == nullptr) return md_set_error(MD_ERR_INVALID, "md_colsum: deterministic workspace too small");
  }
  colsum_kernel<false><<<grid, 256, 0, ST(stream)>>>(x, x_bf16, ld, out, rows, N, ws, 0);
  if (int rc = check_launch("md_colsum")) return rc;
  return ws ? det_reduce(ws, out, grid.y, N, 1, ST(stream)) : 0;
}
extern "C" int md_colsum_interleaved(const void* x, int x_bf16, int64_t ld, float* out, int64_t rows, int64_t N,
                                     int64_t half, void* stream) {
  if (rows == 0 || N == 0) return 0;
  if (!x || !out) return md_set_error(MD_ERR_INVALID, "md_colsum_interleaved: null pointer");
  if (half <= 0 || half % 32 != 0 || N != 2 * half)
    return md_set_error(MD_ERR_INVALID, "md_colsum_interleaved: needs N == 2 half and half % 32 == 0");
  dim3 grid((unsigned)((N + 255) / 256), (unsigned)((rows + 255) / 256));
  float* ws = nullptr;
  if (det_enabled()) {
    ws = det_workspace(static_cast<size_t>(grid.y) * N * sizeof(float));
    if (ws == nullptr) return md_set_error(MD_ERR_INVALID, "md_colsum_interleaved: deterministic workspace too small");
  }
  colsum_kernel<true><<<grid, 256, 0, ST(stream)>>>(x, x_bf16, ld, out, rows, N, ws, half);
  if (int rc = check_launch("md_colsum_interleaved")) return rc;
  return ws ? det_reduce(ws, out, grid.y, N, 1, ST(stream)) : 0;
}
extern "C" int md_cast_transpose(const float* w, void* wb, void* wbt, int64_t batch, int64_t rows, int64_t cols,
                                 int64_t interleave_half, int prec, void* stream) {
  if (batch * rows * cols == 0) return 0;
  if (!w) return md_set_error(MD_ERR_INVALID, "md_cast_transpose: null pointer");
  if (interleave_half != 0 && (interleave_half % 32 != 0 || rows != 2 * interleave_half))
    return md_set_error(MD_ERR_INVALID, "md_cast_transpose: interleave_half = f needs f % 32 == 0 and rows == 2 f");
  dim3 grid((unsigned)((cols + 63) / 64), (unsigned)((rows + 63) / 64), (unsigned)batch);
  MD_WITH_ACT(prec, cast_transpose_kernel<AT><<<grid, 256, 0, ST(stream)>>>(w, AP(AT, wb), AP(AT, wbt), rows, cols, interleave_half));
  return check_launch("md_cast_transpose");
}
extern "C" int md_cast_transpose_multi(const float* flat, void* wb, void* wbt, const md_cast_desc* desc, int64_t n_desc,
                                       int64_t total_tiles, int prec, void* stream) {
  if (n_desc == 0 || total_tiles == 0) return 0;
  if (!flat || !wb || !wbt || !desc) return md_set_error(MD_ERR_INVALID, "md_cast_transpose_multi: null pointer");
  MD_WITH_ACT(prec, cast_transpose_multi_kernel<AT><<<(unsigned)total_tiles, 256, 0, ST(stream)>>>(flat, AP(AT, wb), AP(AT, wbt), desc,
                                                                                               (int)n_desc));
  return check_launch("md_cast_transpose_multi");
}
extern "C" int md_timestep_embed(const float* t, void* out, int64_t B, int64_t dim, int prec, void* stream) {
  if (B == 0) return 0;
  if (!t || !out) return md_set_error(MD_ERR_INVALID, "md_timestep_embed: null pointer");
  MD_WITH_ACT(prec, timestep_embed_kernel<AT><<<(unsigned)B, 128, 0, ST(stream)>>>(t, AP(AT, out), (int)dim));
  return check_launch("md_timestep_embed");
}
extern "C" int md_cond_prepare(const void* cap_f16, const double* keep, void* out_bf16, void* cap_out_f16, int64_t B,
                               int64_t per_sample, int prec, void* stream) {
  if (B == 0) return 0;
  if (!cap_f16 || !out_bf16 || per_sample % 8 != 0)
    return md_set_error(MD_ERR_INVALID, "md_cond_prepare: null pointer or per_sample % 8 != 0");
  dim3 grid((unsigned)min((long long)((per_sample / 8 + 255) / 256), 64LL), (unsigned)B);
  MD_WITH_ACT(prec, cond_prepare_kernel<AT><<<grid, 256, 0, ST(stream)>>>(reinterpret_cast<const __half*>(cap_f16), keep,
                                                                          AP(AT, out_bf16),
                                                                          reinterpret_cast<__half*>(cap_out_f16), per_sample));
  return check_launch("md_cond_prepare");
}
extern "C" int md_sumsq(const float* x, float* sumsq, int64_t n, void* stream) {
  if (n == 0) return 0;
  if (!x || !sumsq) return md_set_error(MD_ERR_INVALID, "md_sumsq: null pointer");
  const int grid = grid_for(n / 4 + 1, 256);
  float* ws = det_enabled() ? det_workspace(static_cast<size_t>(grid) * sizeof(float)) : nullptr;
  sumsq_kernel<<<grid, 256, 0, ST(stream)>>>(x, sumsq, n, ws);
  if (int rc = check_launch("md_sumsq")) return rc;
  return ws ? det_reduce(ws, sumsq, grid, 1, 1, ST(stream)) : 0;
}
extern "C" int md_adamw(float* p, const float* g, float* m, float* v, const float* sumsq, float clip, float lr,
                        float beta1, float beta2, float eps, float wd, int64_t step, int32_t* nonfinite, int64_t n,
                        void* stream) {
  if (n == 0) return 0;
  if (!p || !g || !m || !v || step < 1) return md_set_error(MD_ERR_INVALID, "md_adamw: null pointer or step < 1");
  const float bc1 = 1.f - powf(beta1, (float)step), bc2 = 1.f - powf(beta2, (float)step);
  adamw_kernel<false><<<grid_for(n / 4 + 1, 256), 256, 0, ST(stream)>>>(p, g, m, v, sumsq, clip, lr, beta1, beta2, eps,
                                                                        wd, bc1, bc2, nonfinite, n, nullptr, 0.f);
  return check_launch("md_adamw");
}
extern "C" int md_adamw_ema(float* p, const float* g, float* m, float* v, const float* sumsq, float clip, float lr,
                            float beta1, float beta2, float eps, float wd, int64_t step, float* ema, float smoothing,
                            int32_t* nonfinite, int64_t n, void* stream) {
  if (n == 0) return 0;
  if (!p || !g || !m || !v || !ema || step < 1)
    return md_set_error(MD_ERR_INVALID, "md_adamw_ema: null pointer or step < 1");
  if (!(smoothing >= 0.f && smoothing <= 1.f))
    return md_set_error(MD_ERR_INVALID, "md_adamw_ema: smoothing must lie in [0, 1]");
  if ((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(m) |
       reinterpret_cast<uintptr_t>(v) | reinterpret_cast<uintptr_t>(ema)) & 15)
    return md_set_error(MD_ERR_INVALID, "md_adamw_ema: p, g, m, v and ema must be 16-byte aligned");
  const float bc1 = 1.f - powf(beta1, (float)step), bc2 = 1.f - powf(beta2, (float)step);
  adamw_kernel<true><<<grid_for(n / 4 + 1, 256), 256, 0, ST(stream)>>>(p, g, m, v, sumsq, clip, lr, beta1, beta2, eps,
                                                                       wd, bc1, bc2, nonfinite, n, ema, smoothing);
  return check_launch("md_adamw_ema");
}
extern "C" int md_swap_f32(float* a, float* b, int64_t n, void* stream) {
  if (n == 0) return 0;
  if (!a || !b || n < 0) return md_set_error(MD_ERR_INVALID, "md_swap_f32: null pointer or n < 0");
  if (a == b) return md_set_error(MD_ERR_INVALID, "md_swap_f32: a and b are the same range");
  if (a < b + n && b < a + n) return md_set_error(MD_ERR_INVALID, "md_swap_f32: the two ranges overlap");
  if (((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b)) & 15) == 0)
    swap_f32_kernel<true><<<grid_for(n / 4 + 1, 256), 256, 0, ST(stream)>>>(a, b, n);
  else
    swap_f32_kernel<false><<<grid_for(n, 256), 256, 0, ST(stream)>>>(a, b, n);
  return check_launch("md_swap_f32");
}
