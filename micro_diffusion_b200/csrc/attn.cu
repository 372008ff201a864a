// Non-causal multi-head attention forward / backward for short sequences (T in {64, 77, 256, 1024}),
// head_dim 32, 64 or 128: F.scaled_dot_product_attention at utils.py:188-193 (self) and utils.py:127-132
// (cross, 77 caption tokens) and its autograd backward.
//
// This file: the mma.sync kernels -- flash-style tiles of 64 queries x 64 keys per CTA (4 warps x 16 rows), bf16
// mma.sync m16n8k16 with fp32 accumulation and online softmax in the log2 domain; backward is the deterministic
// two-kernel split (dK/dV per key tile, dQ per query tile; no atomics) plus fused few-key variants (head_dim 32 / 64;
// head_dim 128 always takes the split).  md_attn_fwd runs them for head_dim 32 and head_dim 64 beyond 256 keys;
// md_attn_bwd for head_dim 32 / 128 and head_dim 64 up to 128 keys (the rest: attn_wgmma.cu).  Every entry point
// requires 16-byte aligned operands: the tiles move in 16-byte loads (uint4, cp.async 16).
#include <stdlib.h>

#include <initializer_list>

#include "common.cuh"

namespace md {

constexpr int kTile = 64;

__device__ __forceinline__ void ldsm_x4(uint32_t (&r)[4], const void* p) {
  const uint32_t a = static_cast<uint32_t>(__cvta_generic_to_shared(p));
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(a));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t (&r)[4], const void* p) {
  const uint32_t a = static_cast<uint32_t>(__cvta_generic_to_shared(p));
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(a));
}
__device__ __forceinline__ void mma16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint32_t pack2(float a, float b) {
  __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&v);
}

template <int HD>
struct Smem {
  static constexpr int kPitch = HD + 8;  // bf16 elements; 16-byte row skew -> conflict-free ldmatrix
};

// Load rows [row0, row0+64) x HD columns (starting at column col0) of a [*, ld] bf16 matrix; rows >= nrows -> 0.
template <int HD, int ROWS = kTile>
__device__ __forceinline__ void load_tile(__nv_bfloat16* s, const __nv_bfloat16* g, long long ld, long long row0,
                                          long long nrows, int col0) {
  constexpr int kChunks = HD / 8;
  for (int i = threadIdx.x; i < ROWS * kChunks; i += blockDim.x) {
    const int r = i / kChunks, c = (i % kChunks) * 8;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (row0 + r < nrows) v = *reinterpret_cast<const uint4*>(g + (row0 + r) * ld + col0 + c);
    *reinterpret_cast<uint4*>(s + r * Smem<HD>::kPitch + c) = v;
  }
}

// cp.async variants: the next tile streams into the other buffer while the tensor cores work on this one.
__device__ __forceinline__ void cp_async16(void* smem, const void* gmem, int src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(static_cast<uint32_t>(__cvta_generic_to_shared(smem))),
               "l"(gmem), "r"(src_bytes)
               : "memory");
}
__device__ __forceinline__ void cp_async4(void* smem, const void* gmem, int src_bytes) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(static_cast<uint32_t>(__cvta_generic_to_shared(smem))),
               "l"(gmem), "r"(src_bytes)
               : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

template <int HD, int ROWS = kTile>
__device__ __forceinline__ void load_tile_async(__nv_bfloat16* s, const __nv_bfloat16* g, long long ld, long long row0,
                                                long long nrows, int col0) {
  constexpr int kChunks = HD / 8;
  for (int i = threadIdx.x; i < ROWS * kChunks; i += blockDim.x) {
    const int r = i / kChunks, c = (i % kChunks) * 8;
    const bool ok = row0 + r < nrows;
    cp_async16(s + r * Smem<HD>::kPitch + c, ok ? g + (row0 + r) * ld + col0 + c : g, ok ? 16 : 0);  // 0 -> zero fill
  }
}

// A fragments of a 16 x HD row block starting at smem row r0.
template <int HD>
__device__ __forceinline__ void load_a_frags(uint32_t (&a)[HD / 16][4], const __nv_bfloat16* s, int r0, int lane) {
#pragma unroll
  for (int ks = 0; ks < HD / 16; ++ks)
    ldsm_x4(a[ks], s + (r0 + (lane & 15)) * Smem<HD>::kPitch + ks * 16 + (lane >> 4) * 8);
}

// acc[nt] (16 x KT, nt = KT/8 tiles of 8 columns) = A(16 x HD) . M^T where M is a KT x HD smem tile ([n][k]).
template <int HD, int KT = kTile>
__device__ __forceinline__ void mma_a_bt(float (&acc)[KT / 8][4], const uint32_t (&a)[HD / 16][4], const __nv_bfloat16* m,
                                         int lane) {
#pragma unroll
  for (int np = 0; np < KT / 16; ++np) {
#pragma unroll
    for (int ks = 0; ks < HD / 16; ++ks) {
      uint32_t b[4];
      const int mi = lane >> 3;
      ldsm_x4(b, m + (np * 16 + (lane & 7) + (mi >> 1) * 8) * Smem<HD>::kPitch + ks * 16 + (mi & 1) * 8);
      mma16816(acc[2 * np], a[ks], b[0], b[1]);
      mma16816(acc[2 * np + 1], a[ks], b[2], b[3]);
    }
  }
}

// out[dt] (16 x HD) += P(16 x KT, given as KT/16 k-steps of A fragments) . M where M is a KT x HD smem tile ([k][n]).
template <int HD, int KT = kTile>
__device__ __forceinline__ void mma_p_m(float (&out)[HD / 8][4], const uint32_t (&pa)[KT / 16][4], const __nv_bfloat16* m,
                                        int lane) {
#pragma unroll
  for (int kt = 0; kt < KT / 16; ++kt) {
#pragma unroll
    for (int dp = 0; dp < HD / 16; ++dp) {
      uint32_t b[4];
      const int mi = lane >> 3;
      ldsm_x4_t(b, m + (kt * 16 + (lane & 7) + (mi & 1) * 8) * Smem<HD>::kPitch + dp * 16 + (mi >> 1) * 8);
      mma16816(out[2 * dp], pa[kt], b[0], b[1]);
      mma16816(out[2 * dp + 1], pa[kt], b[2], b[3]);
    }
  }
}

// mma_a_bt with the A operand (16 x HD, smem rows r0..r0+15) read from shared memory one k-step at a time instead of
// held in registers: what the dK / dV kernel needs at head_dim 128, where K / V fragments next to the dK / dV
// accumulators would not fit in the register file.
template <int HD, int KT = kTile>
__device__ __forceinline__ void mma_sa_bt(float (&acc)[KT / 8][4], const __nv_bfloat16* sa, int r0, const __nv_bfloat16* m,
                                          int lane) {
#pragma unroll
  for (int ks = 0; ks < HD / 16; ++ks) {
    uint32_t a[4];
    ldsm_x4(a, sa + (r0 + (lane & 15)) * Smem<HD>::kPitch + ks * 16 + (lane >> 4) * 8);
#pragma unroll
    for (int np = 0; np < KT / 16; ++np) {
      uint32_t b[4];
      const int mi = lane >> 3;
      ldsm_x4(b, m + (np * 16 + (lane & 7) + (mi >> 1) * 8) * Smem<HD>::kPitch + ks * 16 + (mi & 1) * 8);
      mma16816(acc[2 * np], a, b[0], b[1]);
      mma16816(acc[2 * np + 1], a, b[2], b[3]);
    }
  }
}

template <int KS = 4>
__device__ __forceinline__ void acc_to_afrag(uint32_t (&pa)[KS][4], const float (&s)[2 * KS][4]) {
#pragma unroll
  for (int kt = 0; kt < KS; ++kt) {
    pa[kt][0] = pack2(s[2 * kt][0], s[2 * kt][1]);
    pa[kt][1] = pack2(s[2 * kt][2], s[2 * kt][3]);
    pa[kt][2] = pack2(s[2 * kt + 1][0], s[2 * kt + 1][1]);
    pa[kt][3] = pack2(s[2 * kt + 1][2], s[2 * kt + 1][3]);
  }
}

// ------------------------------------------------------------------------------------------ forward
template <int HD, int KT>
__global__ void __launch_bounds__(128)
attn_fwd_kernel(const __nv_bfloat16* __restrict__ q, long long ldq, const __nv_bfloat16* __restrict__ k, long long ldk,
                const __nv_bfloat16* __restrict__ v, long long ldv, __nv_bfloat16* __restrict__ o, long long ldo,
                float* __restrict__ lse, int H, int Tq, int Tk, float scale_log2) {
  constexpr int P = Smem<HD>::kPitch;
  extern __shared__ __align__(16) unsigned char smem_fwd[];
  __nv_bfloat16* sq = reinterpret_cast<__nv_bfloat16*>(smem_fwd);
  __nv_bfloat16* skv = sq + kTile * P;  // [2 buffers][K | V][KT * P]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const int h = blockIdx.y;
  const long long b = blockIdx.z;
  const int q0 = blockIdx.x * kTile;
  const __nv_bfloat16* kg = k + b * Tk * ldk;
  const __nv_bfloat16* vg = v + b * Tk * ldv;

  load_tile_async<HD, KT>(skv, kg, ldk, 0, Tk, h * HD);
  load_tile_async<HD, KT>(skv + KT * P, vg, ldv, 0, Tk, h * HD);
  cp_async_commit();
  load_tile<HD>(sq, q + b * Tq * ldq, ldq, q0, Tq, h * HD);
  __syncthreads();
  uint32_t qa[HD / 16][4];
  load_a_frags<HD>(qa, sq, warp * 16, lane);

  float oacc[HD / 8][4];
#pragma unroll
  for (int i = 0; i < HD / 8; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) oacc[i][j] = 0.f;
  float mrow[2] = {-INFINITY, -INFINITY}, lrow[2] = {0.f, 0.f};

  for (int k0 = 0, it = 0; k0 < Tk; k0 += KT, ++it) {
    __nv_bfloat16* sk = skv + (it & 1) * (2 * KT * P);
    __nv_bfloat16* sv = sk + KT * P;
    if (k0 + KT < Tk) {  // prefetch the next K/V tile into the other buffer
      __nv_bfloat16* nk = skv + ((it + 1) & 1) * (2 * KT * P);
      load_tile_async<HD, KT>(nk, kg, ldk, k0 + KT, Tk, h * HD);
      load_tile_async<HD, KT>(nk + KT * P, vg, ldv, k0 + KT, Tk, h * HD);
      cp_async_commit();
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    float s[KT / 8][4];
#pragma unroll
    for (int i = 0; i < KT / 8; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) s[i][j] = 0.f;
    mma_a_bt<HD, KT>(s, qa, sk, lane);
    float mx[2] = {mrow[0], mrow[1]};
#pragma unroll
    for (int nt = 0; nt < KT / 8; ++nt)
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int key = k0 + nt * 8 + 2 * t + (j & 1);
        s[nt][j] = key < Tk ? s[nt][j] * scale_log2 : -INFINITY;
        mx[j >> 1] = fmaxf(mx[j >> 1], s[nt][j]);
      }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
    }
    float corr[2], rs[2] = {0.f, 0.f};
#pragma unroll
    for (int r = 0; r < 2; ++r) corr[r] = exp2f(mrow[r] - mx[r]);  // first tile: exp2(-inf) = 0
#pragma unroll
    for (int nt = 0; nt < KT / 8; ++nt)
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        s[nt][j] = exp2f(s[nt][j] - mx[j >> 1]);
        rs[j >> 1] += s[nt][j];
      }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      lrow[r] = lrow[r] * corr[r] + rs[r];
      mrow[r] = mx[r];
    }
#pragma unroll
    for (int i = 0; i < HD / 8; ++i) {
      oacc[i][0] *= corr[0]; oacc[i][1] *= corr[0];
      oacc[i][2] *= corr[1]; oacc[i][3] *= corr[1];
    }
    uint32_t pa[KT / 16][4];
    acc_to_afrag<KT / 16>(pa, s);
    mma_p_m<HD, KT>(oacc, pa, sv, lane);
    __syncthreads();  // all warps are done with this buffer before the prefetch of tile it+2 lands in it
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    lrow[r] += __shfl_xor_sync(0xffffffffu, lrow[r], 1);
    lrow[r] += __shfl_xor_sync(0xffffffffu, lrow[r], 2);
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int row = q0 + warp * 16 + g + r * 8;
    if (row < Tq) {
      const float inv = 1.f / lrow[r];
      __nv_bfloat16* dst = o + (b * Tq + row) * ldo + h * HD;
#pragma unroll
      for (int i = 0; i < HD / 8; ++i)
        *reinterpret_cast<uint32_t*>(dst + i * 8 + 2 * t) = pack2(oacc[i][2 * r] * inv, oacc[i][2 * r + 1] * inv);
      if (t == 0) lse[(b * H + h) * Tq + row] = mrow[r] + log2f(lrow[r]);
    }
  }
}

// -------------------------------------------------------------------------------------------- delta
// delta[b,h,q] = sum_d dO * O.  One warp per token row covering all heads with 16-byte loads issued up front;
// a head's HD/8 chunks sit in adjacent lanes, so the per-head sum is a short shuffle reduction.
template <int HD>
__global__ void __launch_bounds__(256)
attn_delta_kernel(const __nv_bfloat16* __restrict__ dout, long long lddo, const __nv_bfloat16* __restrict__ o,
                  long long ldo, float* __restrict__ delta, long long rows, int H, int Tq) {
  constexpr int kLanesPerHead = HD / 8;  // 16 (HD=128), 8 (HD=64) or 4 (HD=32)
  constexpr int kMaxChunks = 8;          // uint4 chunks per lane: H*HD <= 2048
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nchunks = H * kLanesPerHead;
  for (long long row = 1LL * blockIdx.x * 8 + warp; row < rows; row += 1LL * gridDim.x * 8) {
    uint4 a[kMaxChunks], c[kMaxChunks];
#pragma unroll
    for (int j = 0; j < kMaxChunks; ++j) {
      const int i = lane + 32 * j;
      const bool ok = i < nchunks;
      a[j] = ok ? *reinterpret_cast<const uint4*>(dout + row * lddo + 8 * i) : make_uint4(0, 0, 0, 0);
      c[j] = ok ? *reinterpret_cast<const uint4*>(o + row * ldo + 8 * i) : make_uint4(0, 0, 0, 0);
    }
    const long long b = row / Tq;
    const int qq = static_cast<int>(row % Tq);
#pragma unroll
    for (int j = 0; j < kMaxChunks; ++j) {
      const int i = lane + 32 * j;
      const __nv_bfloat162* pa = reinterpret_cast<const __nv_bfloat162*>(&a[j]);
      const __nv_bfloat162* pc = reinterpret_cast<const __nv_bfloat162*>(&c[j]);
      float s = 0.f;
#pragma unroll
      for (int e = 0; e < 4; ++e)
        s += __low2float(pa[e]) * __low2float(pc[e]) + __high2float(pa[e]) * __high2float(pc[e]);
#pragma unroll
      for (int off = kLanesPerHead / 2; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
      if (i < nchunks && (lane % kLanesPerHead) == 0) delta[(b * H + i / kLanesPerHead) * Tq + qq] = s;
    }
  }
}

// ------------------------------------------------------------------------------------- dK / dV kernel
template <int HD>
__global__ void __launch_bounds__(128)
attn_bwd_dkdv_kernel(const __nv_bfloat16* __restrict__ dout, long long lddo, const __nv_bfloat16* __restrict__ q,
                     long long ldq, const __nv_bfloat16* __restrict__ k, long long ldk,
                     const __nv_bfloat16* __restrict__ v, long long ldv, const float* __restrict__ lse,
                     const float* __restrict__ delta, __nv_bfloat16* __restrict__ dk, long long lddk,
                     __nv_bfloat16* __restrict__ dv, long long lddv, int H, int Tq, int Tk, float scale,
                     float scale_log2) {
  constexpr int P = Smem<HD>::kPitch;
  __shared__ __align__(16) __nv_bfloat16 sk[kTile * P];
  __shared__ __align__(16) __nv_bfloat16 sv[kTile * P];
  extern __shared__ __align__(16) unsigned char smem_dkdv[];
  __nv_bfloat16* sqdo = reinterpret_cast<__nv_bfloat16*>(smem_dkdv);                 // [2 buffers][Q | dO][64 * P]
  float* sstat = reinterpret_cast<float*>(sqdo + 4 * kTile * P);                       // [2 buffers][lse | delta][64]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const int h = blockIdx.y;
  const long long b = blockIdx.z;
  const int k0 = blockIdx.x * kTile;
  const __nv_bfloat16* qg = q + b * Tq * ldq;
  const __nv_bfloat16* dog = dout + b * Tq * lddo;
  const float* lseg = lse + (b * H + h) * Tq;
  const float* delg = delta + (b * H + h) * Tq;
  auto prefetch = [&](int q0, int buf) {
    __nv_bfloat16* dstq = sqdo + buf * (2 * kTile * P);
    load_tile_async<HD>(dstq, qg, ldq, q0, Tq, h * HD);
    load_tile_async<HD>(dstq + kTile * P, dog, lddo, q0, Tq, h * HD);
    if (threadIdx.x < kTile) {  // padded queries: zero-filled stats are harmless here (their Q and dO rows are zero)
      const bool ok = q0 + threadIdx.x < Tq;
      cp_async4(sstat + buf * 2 * kTile + threadIdx.x, ok ? lseg + q0 + threadIdx.x : lseg, ok ? 4 : 0);
      cp_async4(sstat + buf * 2 * kTile + kTile + threadIdx.x, ok ? delg + q0 + threadIdx.x : delg, ok ? 4 : 0);
    }
    cp_async_commit();
  };
  prefetch(0, 0);

  load_tile<HD>(sk, k + b * Tk * ldk, ldk, k0, Tk, h * HD);
  load_tile<HD>(sv, v + b * Tk * ldv, ldv, k0, Tk, h * HD);
  __syncthreads();
  // head_dim 128: the K / V A fragments stay in shared memory (read per k-step), so that the 2 x 64 dK / dV accumulators
  // and the S^T / dP^T tiles fit in registers without spilling
  constexpr bool kFragsInSmem = HD == 128;
  uint32_t ka[HD / 16][4], va[HD / 16][4];
  if constexpr (!kFragsInSmem) {
    load_a_frags<HD>(ka, sk, warp * 16, lane);
    load_a_frags<HD>(va, sv, warp * 16, lane);
  }

  float dkacc[HD / 8][4], dvacc[HD / 8][4];
#pragma unroll
  for (int i = 0; i < HD / 8; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) dkacc[i][j] = dvacc[i][j] = 0.f;

  for (int q0 = 0, it = 0; q0 < Tq; q0 += kTile, ++it) {
    const __nv_bfloat16* sq = sqdo + (it & 1) * (2 * kTile * P);
    const __nv_bfloat16* sdo = sq + kTile * P;
    const float* slse = sstat + (it & 1) * 2 * kTile;
    const float* sdelta = slse + kTile;
    if (q0 + kTile < Tq) {
      prefetch(q0 + kTile, (it + 1) & 1);
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    float st[8][4], dpt[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) st[i][j] = dpt[i][j] = 0.f;
    if constexpr (kFragsInSmem) {
      mma_sa_bt<HD>(st, sk, warp * 16, sq, lane);
      mma_sa_bt<HD>(dpt, sv, warp * 16, sdo, lane);
    } else {
      mma_a_bt<HD>(st, ka, sq, lane);    // S^T  = K . Q^T     (16 keys x 64 queries)
      mma_a_bt<HD>(dpt, va, sdo, lane);  // dP^T = V . dO^T
    }
#pragma unroll
    for (int nt = 0; nt < 8; ++nt)
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int qc = nt * 8 + 2 * t + (j & 1);
        const float p = exp2f(st[nt][j] * scale_log2 - slse[qc]);
        st[nt][j] = p;
        dpt[nt][j] = p * (dpt[nt][j] - sdelta[qc]);
      }
    uint32_t pa[4][4];
    acc_to_afrag(pa, st);
    mma_p_m<HD>(dvacc, pa, sdo, lane);  // dV += P^T . dO
    acc_to_afrag(pa, dpt);
    mma_p_m<HD>(dkacc, pa, sq, lane);   // dK += dS^T . Q
    __syncthreads();
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int key = k0 + warp * 16 + g + r * 8;
    if (key < Tk) {
      __nv_bfloat16* pk = dk + (b * Tk + key) * lddk + h * HD;
      __nv_bfloat16* pv = dv + (b * Tk + key) * lddv + h * HD;
#pragma unroll
      for (int i = 0; i < HD / 8; ++i) {
        *reinterpret_cast<uint32_t*>(pk + i * 8 + 2 * t) = pack2(dkacc[i][2 * r] * scale, dkacc[i][2 * r + 1] * scale);
        *reinterpret_cast<uint32_t*>(pv + i * 8 + 2 * t) = pack2(dvacc[i][2 * r], dvacc[i][2 * r + 1]);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------ dQ kernel
template <int HD>
__global__ void __launch_bounds__(128)
attn_bwd_dq_kernel(const __nv_bfloat16* __restrict__ dout, long long lddo, const __nv_bfloat16* __restrict__ q,
                   long long ldq, const __nv_bfloat16* __restrict__ k, long long ldk,
                   const __nv_bfloat16* __restrict__ v, long long ldv, const float* __restrict__ lse,
                   const float* __restrict__ delta, __nv_bfloat16* __restrict__ dq, long long lddq, int H, int Tq,
                   int Tk, float scale, float scale_log2) {
  constexpr int P = Smem<HD>::kPitch;
  __shared__ __align__(16) __nv_bfloat16 sq[kTile * P];
  __shared__ __align__(16) __nv_bfloat16 sdo[kTile * P];
  extern __shared__ __align__(16) unsigned char smem_dq[];
  __nv_bfloat16* skv = reinterpret_cast<__nv_bfloat16*>(smem_dq);  // [2 buffers][K | V][64 * P]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const int h = blockIdx.y;
  const long long b = blockIdx.z;
  const int q0 = blockIdx.x * kTile;
  const __nv_bfloat16* kg = k + b * Tk * ldk;
  const __nv_bfloat16* vg = v + b * Tk * ldv;

  load_tile_async<HD>(skv, kg, ldk, 0, Tk, h * HD);
  load_tile_async<HD>(skv + kTile * P, vg, ldv, 0, Tk, h * HD);
  cp_async_commit();
  load_tile<HD>(sq, q + b * Tq * ldq, ldq, q0, Tq, h * HD);
  load_tile<HD>(sdo, dout + b * Tq * lddo, lddo, q0, Tq, h * HD);
  __syncthreads();
  uint32_t qa[HD / 16][4], doa[HD / 16][4];
  load_a_frags<HD>(qa, sq, warp * 16, lane);
  load_a_frags<HD>(doa, sdo, warp * 16, lane);
  float lrow[2], drow[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int row = q0 + warp * 16 + g + r * 8;
    lrow[r] = row < Tq ? lse[(b * H + h) * Tq + row] : INFINITY;
    drow[r] = row < Tq ? delta[(b * H + h) * Tq + row] : 0.f;
  }
  float dqacc[HD / 8][4];
#pragma unroll
  for (int i = 0; i < HD / 8; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) dqacc[i][j] = 0.f;

  for (int k0 = 0, it = 0; k0 < Tk; k0 += kTile, ++it) {
    __nv_bfloat16* sk = skv + (it & 1) * (2 * kTile * P);
    __nv_bfloat16* sv = sk + kTile * P;
    if (k0 + kTile < Tk) {
      __nv_bfloat16* nk = skv + ((it + 1) & 1) * (2 * kTile * P);
      load_tile_async<HD>(nk, kg, ldk, k0 + kTile, Tk, h * HD);
      load_tile_async<HD>(nk + kTile * P, vg, ldv, k0 + kTile, Tk, h * HD);
      cp_async_commit();
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    float s[8][4], dp[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) s[i][j] = dp[i][j] = 0.f;
    mma_a_bt<HD>(s, qa, sk, lane);    // S  = Q . K^T
    mma_a_bt<HD>(dp, doa, sv, lane);  // dP = dO . V^T
#pragma unroll
    for (int nt = 0; nt < 8; ++nt)
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int key = k0 + nt * 8 + 2 * t + (j & 1);
        const float p = key < Tk ? exp2f(s[nt][j] * scale_log2 - lrow[j >> 1]) : 0.f;
        s[nt][j] = p * (dp[nt][j] - drow[j >> 1]);
      }
    uint32_t pa[4][4];
    acc_to_afrag(pa, s);
    mma_p_m<HD>(dqacc, pa, sk, lane);  // dQ += dS . K
    __syncthreads();
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int row = q0 + warp * 16 + g + r * 8;
    if (row < Tq) {
      __nv_bfloat16* dst = dq + (b * Tq + row) * lddq + h * HD;
#pragma unroll
      for (int i = 0; i < HD / 8; ++i)
        *reinterpret_cast<uint32_t*>(dst + i * 8 + 2 * t) = pack2(dqacc[i][2 * r] * scale, dqacc[i][2 * r + 1] * scale);
    }
  }
}

// --------------------------------------------------------------------- fused backward, short sequences
// Tq <= 64 and Tk <= KT (64 or 80): one CTA per (sample, head) does the whole backward in a single pass --
// S and dP once (the generic path computes them twice), delta = rowsum(P*dP) on the fly (no delta kernel, no O
// read), dQ straight from registers, and dK / dV from P^T / dS^T read back transposed (ldmatrix.trans) from a
// shared-memory copy.  This is the backbone regime of the benchmark (64 tokens after 75 % masking, 77 caption
// tokens), where the generic kernels are latency- rather than math-bound.
template <int HD, int KT>
__global__ void __launch_bounds__(128)
attn_bwd_small_kernel(const __nv_bfloat16* __restrict__ dout, long long lddo, const __nv_bfloat16* __restrict__ q,
                      long long ldq, const __nv_bfloat16* __restrict__ k, long long ldk,
                      const __nv_bfloat16* __restrict__ v, long long ldv, const float* __restrict__ lse,
                      __nv_bfloat16* __restrict__ dq, long long lddq, __nv_bfloat16* __restrict__ dk, long long lddk,
                      __nv_bfloat16* __restrict__ dv, long long lddv, int H, int Tq, int Tk, float scale,
                      float scale_log2) {
  constexpr int P = Smem<HD>::kPitch;
  constexpr int PP = KT + 8;  // pitch of the P / dS copies ([query][key])
  extern __shared__ __align__(16) unsigned char smem_small[];
  __nv_bfloat16* sq = reinterpret_cast<__nv_bfloat16*>(smem_small);
  __nv_bfloat16* sdo = sq + kTile * P;
  __nv_bfloat16* sk = sdo + kTile * P;
  __nv_bfloat16* sv = sk + KT * P;
  // P and dS copies ([64][PP]) reuse the K and V tiles, which are dead once dQ has been formed: 41 KB instead of
  // 64 KB per CTA -> five CTAs per SM, which is what this latency-bound regime needs.
  static_assert(kTile * (KT + 8) <= KT * Smem<HD>::kPitch || HD == 32, "P copy must fit in the K tile");
  __nv_bfloat16* sp = (HD == 64) ? sk : sv + KT * P;
  __nv_bfloat16* sds = (HD == 64) ? sv : sp + kTile * PP;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const int h = blockIdx.x;
  const long long b = blockIdx.y;

  load_tile<HD>(sq, q + b * Tq * ldq, ldq, 0, Tq, h * HD);
  load_tile<HD>(sdo, dout + b * Tq * lddo, lddo, 0, Tq, h * HD);
  load_tile<HD, KT>(sk, k + b * Tk * ldk, ldk, 0, Tk, h * HD);
  load_tile<HD, KT>(sv, v + b * Tk * ldv, ldv, 0, Tk, h * HD);
  float lrow[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int row = warp * 16 + g + r * 8;
    lrow[r] = row < Tq ? lse[(b * H + h) * Tq + row] : INFINITY;  // +inf -> P = 0 for padded queries
  }
  __syncthreads();

  uint32_t qa[HD / 16][4], doa[HD / 16][4];
  load_a_frags<HD>(qa, sq, warp * 16, lane);
  load_a_frags<HD>(doa, sdo, warp * 16, lane);
  float s[KT / 8][4], dp[KT / 8][4];
#pragma unroll
  for (int i = 0; i < KT / 8; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) s[i][j] = dp[i][j] = 0.f;
  mma_a_bt<HD, KT>(s, qa, sk, lane);    // S  = Q . K^T
  mma_a_bt<HD, KT>(dp, doa, sv, lane);  // dP = dO . V^T
  float dsum[2] = {0.f, 0.f};
#pragma unroll
  for (int nt = 0; nt < KT / 8; ++nt)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int key = nt * 8 + 2 * t + (j & 1);
      const float p = key < Tk ? exp2f(s[nt][j] * scale_log2 - lrow[j >> 1]) : 0.f;
      s[nt][j] = p;
      dsum[j >> 1] += p * dp[nt][j];
    }
#pragma unroll
  for (int r = 0; r < 2; ++r) {  // delta[row] = sum_keys P * dP  (== sum_d dO * O)
    dsum[r] += __shfl_xor_sync(0xffffffffu, dsum[r], 1);
    dsum[r] += __shfl_xor_sync(0xffffffffu, dsum[r], 2);
  }
#pragma unroll
  for (int nt = 0; nt < KT / 8; ++nt)
#pragma unroll
    for (int j = 0; j < 4; ++j) dp[nt][j] = s[nt][j] * (dp[nt][j] - dsum[j >> 1]);  // dS
  // dQ = dS . K  (A straight from the accumulator registers)
  {
    uint32_t pa[KT / 16][4];
    acc_to_afrag<KT / 16>(pa, dp);
    float dqacc[HD / 8][4];
#pragma unroll
    for (int i = 0; i < HD / 8; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) dqacc[i][j] = 0.f;
    mma_p_m<HD, KT>(dqacc, pa, sk, lane);
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int row = warp * 16 + g + r * 8;
      if (row < Tq) {
        __nv_bfloat16* dst = dq + (b * Tq + row) * lddq + h * HD;
#pragma unroll
        for (int i = 0; i < HD / 8; ++i)
          *reinterpret_cast<uint32_t*>(dst + i * 8 + 2 * t) = pack2(dqacc[i][2 * r] * scale, dqacc[i][2 * r + 1] * scale);
      }
    }
  }
  __syncthreads();  // every warp is done reading K / V
  // bf16 copies of P and dS for the transposed contractions
#pragma unroll
  for (int nt = 0; nt < KT / 8; ++nt)
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int row = warp * 16 + g + r * 8;
      *reinterpret_cast<uint32_t*>(sp + row * PP + nt * 8 + 2 * t) = pack2(s[nt][2 * r], s[nt][2 * r + 1]);
      *reinterpret_cast<uint32_t*>(sds + row * PP + nt * 8 + 2 * t) = pack2(dp[nt][2 * r], dp[nt][2 * r + 1]);
    }
  __syncthreads();
  // dV = P^T . dO and dK = dS^T . Q : 16 keys per warp-iteration, reduction over the 64 queries.
  for (int kb = warp; kb < KT / 16; kb += 4) {
    uint32_t pta[4][4], dsta[4][4];
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {  // A[m = key][k = query] = X[query][key]: transposed load
      const int mi = lane >> 3;
      const int rowq = ks * 16 + (lane & 7) + (mi >> 1) * 8;
      const int colk = kb * 16 + (mi & 1) * 8;
      ldsm_x4_t(pta[ks], sp + rowq * PP + colk);
      ldsm_x4_t(dsta[ks], sds + rowq * PP + colk);
    }
    float dvacc[HD / 8][4], dkacc[HD / 8][4];
#pragma unroll
    for (int i = 0; i < HD / 8; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) dvacc[i][j] = dkacc[i][j] = 0.f;
    mma_p_m<HD, 64>(dvacc, pta, sdo, lane);
    mma_p_m<HD, 64>(dkacc, dsta, sq, lane);
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int key = kb * 16 + g + r * 8;
      if (key < Tk) {
        __nv_bfloat16* pk = dk + (b * Tk + key) * lddk + h * HD;
        __nv_bfloat16* pv = dv + (b * Tk + key) * lddv + h * HD;
#pragma unroll
        for (int i = 0; i < HD / 8; ++i) {
          *reinterpret_cast<uint32_t*>(pk + i * 8 + 2 * t) = pack2(dkacc[i][2 * r] * scale, dkacc[i][2 * r + 1] * scale);
          *reinterpret_cast<uint32_t*>(pv + i * 8 + 2 * t) = pack2(dvacc[i][2 * r], dvacc[i][2 * r + 1]);
        }
      }
    }
  }
}

// ---------------------------------------------------------------------- backward, few keys, many queries
// Cross-attention to the caption (Tk <= 80, Tq = 256 / 1024): one CTA per (head, sample) keeps K and V in shared
// memory, streams the 64-query tiles (cp.async double buffer) and carries dK / dV in registers across the tiles, so
// Q / dO / K / V are read exactly once and no partial dK / dV ever leaves the SM.  Warp w owns keys 16w..16w+15; with
// KT = 80 the fifth key block is split by head-dim columns (16 per warp).
template <int HD, int DP>
__device__ __forceinline__ void mma_p_m_slice(float (&out)[2][4], const uint32_t (&pa)[4][4], const __nv_bfloat16* m,
                                              int lane, int dp) {
#pragma unroll
  for (int kt = 0; kt < 4; ++kt) {
    uint32_t b[4];
    const int mi = lane >> 3;
    ldsm_x4_t(b, m + (kt * 16 + (lane & 7) + (mi & 1) * 8) * Smem<HD>::kPitch + dp * 16 + (mi >> 1) * 8);
    mma16816(out[0], pa[kt], b[0], b[1]);
    mma16816(out[1], pa[kt], b[2], b[3]);
  }
}

template <int HD, int KT>
__global__ void __launch_bounds__(128)
attn_bwd_cross_kernel(const __nv_bfloat16* __restrict__ dout, long long lddo, const __nv_bfloat16* __restrict__ q,
                      long long ldq, const __nv_bfloat16* __restrict__ k, long long ldk,
                      const __nv_bfloat16* __restrict__ v, long long ldv, const float* __restrict__ lse,
                      __nv_bfloat16* __restrict__ dq, long long lddq, __nv_bfloat16* __restrict__ dk, long long lddk,
                      __nv_bfloat16* __restrict__ dv, long long lddv, int H, int Tq, int Tk, float scale,
                      float scale_log2) {
  constexpr int P = Smem<HD>::kPitch;
  constexpr int PP = KT + 8;
  constexpr bool kExtra = KT > 64;               // fifth 16-key block (keys 64..79)
  constexpr int kSliceWarps = HD / 16;           // warps that take a 16-column slice of the fifth block
  extern __shared__ __align__(16) unsigned char smem_cross[];
  __nv_bfloat16* sk = reinterpret_cast<__nv_bfloat16*>(smem_cross);
  __nv_bfloat16* sv = sk + KT * P;
  __nv_bfloat16* sqdo = sv + KT * P;             // [2 buffers][Q | dO][64 * P]
  __nv_bfloat16* sp = sqdo + 4 * kTile * P;      // [64][PP]
  __nv_bfloat16* sds = sp + kTile * PP;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const int h = blockIdx.x;
  const long long b = blockIdx.y;
  const __nv_bfloat16* qg = q + b * Tq * ldq;
  const __nv_bfloat16* dog = dout + b * Tq * lddo;
  const float* lseg = lse + (b * H + h) * Tq;

  auto prefetch = [&](int q0, int buf) {
    __nv_bfloat16* dst = sqdo + buf * (2 * kTile * P);
    load_tile_async<HD>(dst, qg, ldq, q0, Tq, h * HD);
    load_tile_async<HD>(dst + kTile * P, dog, lddo, q0, Tq, h * HD);
    cp_async_commit();
  };
  load_tile_async<HD, KT>(sk, k + b * Tk * ldk, ldk, 0, Tk, h * HD);
  load_tile_async<HD, KT>(sv, v + b * Tk * ldv, ldv, 0, Tk, h * HD);
  prefetch(0, 0);  // one group: K, V and the first Q / dO tile

  float dvacc[HD / 8][4], dkacc[HD / 8][4];
  float dvx[2][4], dkx[2][4];
#pragma unroll
  for (int i = 0; i < HD / 8; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) dvacc[i][j] = dkacc[i][j] = 0.f;
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) dvx[i][j] = dkx[i][j] = 0.f;

  for (int q0 = 0, it = 0; q0 < Tq; q0 += kTile, ++it) {
    const __nv_bfloat16* sq = sqdo + (it & 1) * (2 * kTile * P);
    const __nv_bfloat16* sdo = sq + kTile * P;
    float lrow[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int row = q0 + warp * 16 + g + r * 8;
      lrow[r] = row < Tq ? lseg[row] : INFINITY;  // +inf -> P = 0 for padded queries
    }
    if (q0 + kTile < Tq) {
      prefetch(q0 + kTile, (it + 1) & 1);
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();

    uint32_t qa[HD / 16][4], doa[HD / 16][4];
    load_a_frags<HD>(qa, sq, warp * 16, lane);
    load_a_frags<HD>(doa, sdo, warp * 16, lane);
    float s[KT / 8][4], dp[KT / 8][4];
#pragma unroll
    for (int i = 0; i < KT / 8; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) s[i][j] = dp[i][j] = 0.f;
    mma_a_bt<HD, KT>(s, qa, sk, lane);    // S  = Q . K^T
    mma_a_bt<HD, KT>(dp, doa, sv, lane);  // dP = dO . V^T
    float dsum[2] = {0.f, 0.f};
#pragma unroll
    for (int nt = 0; nt < KT / 8; ++nt)
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int key = nt * 8 + 2 * t + (j & 1);
        const float pr = key < Tk ? exp2f(s[nt][j] * scale_log2 - lrow[j >> 1]) : 0.f;
        s[nt][j] = pr;
        dsum[j >> 1] += pr * dp[nt][j];
      }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      dsum[r] += __shfl_xor_sync(0xffffffffu, dsum[r], 1);
      dsum[r] += __shfl_xor_sync(0xffffffffu, dsum[r], 2);
    }
#pragma unroll
    for (int nt = 0; nt < KT / 8; ++nt)
#pragma unroll
      for (int j = 0; j < 4; ++j) dp[nt][j] = s[nt][j] * (dp[nt][j] - dsum[j >> 1]);  // dS
    {
      uint32_t pa[KT / 16][4];
      acc_to_afrag<KT / 16>(pa, dp);
      float dqacc[HD / 8][4];
#pragma unroll
      for (int i = 0; i < HD / 8; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) dqacc[i][j] = 0.f;
      mma_p_m<HD, KT>(dqacc, pa, sk, lane);  // dQ = dS . K
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const int row = q0 + warp * 16 + g + r * 8;
        if (row < Tq) {
          __nv_bfloat16* dst = dq + (b * Tq + row) * lddq + h * HD;
#pragma unroll
          for (int i = 0; i < HD / 8; ++i)
            *reinterpret_cast<uint32_t*>(dst + i * 8 + 2 * t) = pack2(dqacc[i][2 * r] * scale, dqacc[i][2 * r + 1] * scale);
        }
      }
    }
#pragma unroll
    for (int nt = 0; nt < KT / 8; ++nt)
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const int row = warp * 16 + g + r * 8;
        *reinterpret_cast<uint32_t*>(sp + row * PP + nt * 8 + 2 * t) = pack2(s[nt][2 * r], s[nt][2 * r + 1]);
        *reinterpret_cast<uint32_t*>(sds + row * PP + nt * 8 + 2 * t) = pack2(dp[nt][2 * r], dp[nt][2 * r + 1]);
      }
    __syncthreads();
    {  // dV += P^T . dO and dK += dS^T . Q for this warp's 16 keys (reduction over the tile's 64 queries)
      uint32_t pta[4][4], dsta[4][4];
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        const int mi = lane >> 3;
        const int rowq = ks * 16 + (lane & 7) + (mi >> 1) * 8;
        const int colk = warp * 16 + (mi & 1) * 8;
        ldsm_x4_t(pta[ks], sp + rowq * PP + colk);
        ldsm_x4_t(dsta[ks], sds + rowq * PP + colk);
      }
      mma_p_m<HD, 64>(dvacc, pta, sdo, lane);
      mma_p_m<HD, 64>(dkacc, dsta, sq, lane);
      if (kExtra && warp < kSliceWarps) {
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) {
          const int mi = lane >> 3;
          const int rowq = ks * 16 + (lane & 7) + (mi >> 1) * 8;
          const int colk = 64 + (mi & 1) * 8;
          ldsm_x4_t(pta[ks], sp + rowq * PP + colk);
          ldsm_x4_t(dsta[ks], sds + rowq * PP + colk);
        }
        mma_p_m_slice<HD, 0>(dvx, pta, sdo, lane, warp);
        mma_p_m_slice<HD, 0>(dkx, dsta, sq, lane, warp);
      }
    }
    __syncthreads();  // sp / sds / this Q-dO buffer are rewritten by the next iterations
  }

#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int key = warp * 16 + g + r * 8;
    if (key < Tk) {
      __nv_bfloat16* pk = dk + (b * Tk + key) * lddk + h * HD;
      __nv_bfloat16* pv = dv + (b * Tk + key) * lddv + h * HD;
#pragma unroll
      for (int i = 0; i < HD / 8; ++i) {
        *reinterpret_cast<uint32_t*>(pk + i * 8 + 2 * t) = pack2(dkacc[i][2 * r] * scale, dkacc[i][2 * r + 1] * scale);
        *reinterpret_cast<uint32_t*>(pv + i * 8 + 2 * t) = pack2(dvacc[i][2 * r], dvacc[i][2 * r + 1]);
      }
    }
  }
  if (kExtra && warp < kSliceWarps) {
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int key = 64 + g + r * 8;
      if (key < Tk) {
        __nv_bfloat16* pk = dk + (b * Tk + key) * lddk + h * HD + warp * 16;
        __nv_bfloat16* pv = dv + (b * Tk + key) * lddv + h * HD + warp * 16;
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          *reinterpret_cast<uint32_t*>(pk + i * 8 + 2 * t) = pack2(dkx[i][2 * r] * scale, dkx[i][2 * r + 1] * scale);
          *reinterpret_cast<uint32_t*>(pv + i * 8 + 2 * t) = pack2(dvx[i][2 * r], dvx[i][2 * r + 1]);
        }
      }
    }
  }
}

template <int HD, int KT>
static size_t cross_bwd_smem() {
  return sizeof(__nv_bfloat16) * (2 * KT * Smem<HD>::kPitch + 4 * kTile * Smem<HD>::kPitch + 2 * kTile * (KT + 8));
}

template <int HD, int KT>
static size_t small_bwd_smem() {
  const size_t base = 2 * kTile * Smem<HD>::kPitch + 2 * KT * Smem<HD>::kPitch;
  return sizeof(__nv_bfloat16) * (HD == 64 ? base : base + 2 * kTile * (KT + 8));
}

// lds: every row pitch or'ed together; ptrs: every operand address or'ed together.  Each row of a head is read and
// written in 16-byte pieces, so both must keep 16-byte alignment.
static int check_attn(const char* what, int64_t B, int64_t H, int64_t Tq, int64_t Tk, int64_t hd, int64_t lds,
                      uintptr_t ptrs) {
  if (hd != 32 && hd != 64 && hd != 128)
    return md_set_error(MD_ERR_UNSUPPORTED, "attention: head_dim must be 32, 64 or 128");
  if (B < 0 || H <= 0 || Tq <= 0 || Tk <= 0 || H > 65535 || B > 65535)
    return md_set_error(MD_ERR_INVALID, what);
  if (lds % 8 != 0) return md_set_error(MD_ERR_INVALID, "attention: row pitches must be multiples of 8 elements");
  if ((ptrs & 15) != 0) return md_set_error(MD_ERR_INVALID, "attention: operands must be 16-byte aligned");
  return 0;
}

static uintptr_t addr_or(std::initializer_list<const void*> ps) {
  uintptr_t a = 0;
  for (const void* p : ps) a |= reinterpret_cast<uintptr_t>(p);
  return a;
}

}  // namespace md

namespace md {
int attn_bwd_wgmma(const void* dout, int64_t lddo, const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v,
                   int64_t ldv, const float* lse, const float* delta, void* dq, int64_t lddq, void* dk, int64_t lddk,
                   void* dv, int64_t lddv, int64_t B, int64_t H, int64_t Tq, int64_t Tk, cudaStream_t stream);
}
using namespace md;
#define ST(s) reinterpret_cast<cudaStream_t>(s)
#define BF(p) reinterpret_cast<__nv_bfloat16*>(p)
#define CBF(p) reinterpret_cast<const __nv_bfloat16*>(p)

extern "C" int md_attn_fwd(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, void* o,
                           int64_t ldo, float* lse, int64_t B, int64_t H, int64_t Tq, int64_t Tk, int64_t hd,
                           void* stream) {
  if (int rc = check_attn("md_attn_fwd: bad sizes", B, H, Tq, Tk, hd, (ldq | ldk | ldv | ldo), addr_or({q, k, v, o})))
    return rc;
  if (B == 0) return 0;
  if (!q || !k || !v || !o || !lse) return md_set_error(MD_ERR_INVALID, "md_attn_fwd: null pointer");
  // head_dim 64 with all keys in one S tile: the wgmma kernel (attn_wgmma.cu), 1.3-1.5x faster than mma.sync on every
  // forward shape of the res-256 configs on an H100 (B = 256, H = 12 / 16, Tq x Tk = 256 x 256 / 64 x 64 / 64 x 77 / 256 x 77).
  // head_dim 128, any Tk: the chunked wgmma kernel, 1.5-2.5x faster than attn_fwd_kernel<128, .> on every measured shape
  // (res-256 and res-512 MicroDiT_XL_2 widths, 64-1024 queries, 64-1024 keys; DESIGN.md 5.2), so it always takes it.
  if ((hd == 64 && Tk <= 256) || hd == 128)
    return md_attn_fwd_tc(q, ldq, k, ldk, v, ldv, o, ldo, lse, B, H, Tq, Tk, hd, stream);
  return md_attn_fwd_mma(q, ldq, k, ldk, v, ldv, o, ldo, lse, B, H, Tq, Tk, hd, stream);
}

extern "C" int md_attn_fwd_mma(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, void* o,
                               int64_t ldo, float* lse, int64_t B, int64_t H, int64_t Tq, int64_t Tk, int64_t hd,
                               void* stream) {
  if (int rc = check_attn("md_attn_fwd: bad sizes", B, H, Tq, Tk, hd, (ldq | ldk | ldv | ldo), addr_or({q, k, v, o})))
    return rc;
  if (B == 0) return 0;
  if (!q || !k || !v || !o || !lse) return md_set_error(MD_ERR_INVALID, "md_attn_fwd: null pointer");
  const float sl2 = 1.4426950408889634f / sqrtf((float)hd);
  dim3 grid((unsigned)((Tq + kTile - 1) / kTile), (unsigned)H, (unsigned)B);
  const bool kt80 = Tk > 64 && Tk <= 80;  // the 77 caption tokens: one 80-key tile instead of 64 + a 13-key stub
#define FWD(HD_, KT_)                                                                                                \
  do {                                                                                                               \
    static bool attr = false;                                                                                        \
    const size_t sm = (size_t)(kTile + 4 * KT_) * Smem<HD_>::kPitch * sizeof(__nv_bfloat16);                         \
    if (!attr) {                                                                                                     \
      cudaFuncSetAttribute(attn_fwd_kernel<HD_, KT_>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm);        \
      attr = true;                                                                                                   \
    }                                                                                                                \
    attn_fwd_kernel<HD_, KT_><<<grid, 128, sm, ST(stream)>>>(CBF(q), ldq, CBF(k), ldk, CBF(v), ldv, BF(o), ldo, lse, \
                                                             (int)H, (int)Tq, (int)Tk, sl2);                         \
  } while (0)
  if (hd == 128) { if (kt80) FWD(128, 80); else FWD(128, 64); }
  else if (hd == 64) { if (kt80) FWD(64, 80); else FWD(64, 64); }
  else { if (kt80) FWD(32, 80); else FWD(32, 64); }
#undef FWD
  return check_launch("md_attn_fwd");
}

extern "C" int md_attn_bwd(const void* dout, int64_t lddo, const void* q, int64_t ldq, const void* k, int64_t ldk,
                           const void* v, int64_t ldv, const void* o, int64_t ldo, const float* lse, float* delta,
                           void* dq, int64_t lddq, void* dk, int64_t lddk, void* dv, int64_t lddv, int64_t B, int64_t H,
                           int64_t Tq, int64_t Tk, int64_t hd, void* stream) {
  if (int rc = check_attn("md_attn_bwd: bad sizes", B, H, Tq, Tk, hd, (lddo | ldq | ldk | ldv | ldo | lddq | lddk | lddv),
                          addr_or({dout, q, k, v, o, dq, dk, dv})))
    return rc;
  if (B == 0) return 0;
  if (!dout || !q || !k || !v || !o || !lse || !delta || !dq || !dk || !dv)
    return md_set_error(MD_ERR_INVALID, "md_attn_bwd: null pointer");
  // head_dim 64 beyond 128 keys: the wgmma backward (attn_wgmma.cu); up to 128 keys the fused few-key mma.sync kernels
  if (hd == 64 && Tk > 128)
    return md_attn_bwd_tc(dout, lddo, q, ldq, k, ldk, v, ldv, o, ldo, lse, delta, dq, lddq, dk, lddk, dv, lddv, B, H, Tq, Tk,
                          hd, stream);
  return md_attn_bwd_mma(dout, lddo, q, ldq, k, ldk, v, ldv, o, ldo, lse, delta, dq, lddq, dk, lddk, dv, lddv, B, H, Tq, Tk, hd,
                         stream);
}

extern "C" int md_attn_bwd_mma(const void* dout, int64_t lddo, const void* q, int64_t ldq, const void* k, int64_t ldk,
                               const void* v, int64_t ldv, const void* o, int64_t ldo, const float* lse, float* delta,
                               void* dq, int64_t lddq, void* dk, int64_t lddk, void* dv, int64_t lddv, int64_t B, int64_t H,
                               int64_t Tq, int64_t Tk, int64_t hd, void* stream) {
  if (int rc = check_attn("md_attn_bwd: bad sizes", B, H, Tq, Tk, hd, (lddo | ldq | ldk | ldv | ldo | lddq | lddk | lddv),
                          addr_or({dout, q, k, v, o, dq, dk, dv})))
    return rc;
  if (B == 0) return 0;
  if (!dout || !q || !k || !v || !o || !lse || !delta || !dq || !dk || !dv)
    return md_set_error(MD_ERR_INVALID, "md_attn_bwd: null pointer");
  const float scale = 1.f / sqrtf((float)hd);
  const float sl2 = 1.4426950408889634f * scale;
  // head_dim 128 always takes the generic split below: the fused few-key kernels are laid out for <= 64 columns
  if (hd != 128 && Tq <= kTile && Tk <= 80) {  // single-pass fused backward
    dim3 gs((unsigned)H, (unsigned)B);
#define BWD_SMALL(HD_, KT_)                                                                                          \
  do {                                                                                                               \
    static bool attr = false;                                                                                        \
    const size_t sm = small_bwd_smem<HD_, KT_>();                                                                    \
    if (!attr) {                                                                                                     \
      cudaFuncSetAttribute(attn_bwd_small_kernel<HD_, KT_>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm);  \
      attr = true;                                                                                                   \
    }                                                                                                                \
    attn_bwd_small_kernel<HD_, KT_><<<gs, 128, sm, ST(stream)>>>(CBF(dout), lddo, CBF(q), ldq, CBF(k), ldk, CBF(v),  \
                                                                 ldv, lse, BF(dq), lddq, BF(dk), lddk, BF(dv), lddv, \
                                                                 (int)H, (int)Tq, (int)Tk, scale, sl2);              \
  } while (0)
    if (hd == 64) { if (Tk <= 64) BWD_SMALL(64, 64); else BWD_SMALL(64, 80); }
    else { if (Tk <= 64) BWD_SMALL(32, 64); else BWD_SMALL(32, 80); }
#undef BWD_SMALL
    return check_launch("md_attn_bwd");
  }
  if (hd != 128 && Tk <= 80) {  // few keys, many queries (cross-attention at T = 256 / 1024): K / V resident, dK / dV in registers
    dim3 gs((unsigned)H, (unsigned)B);
#define BWD_CROSS(HD_, KT_)                                                                                          \
  do {                                                                                                               \
    static bool attr = false;                                                                                        \
    const size_t sm = cross_bwd_smem<HD_, KT_>();                                                                    \
    if (!attr) {                                                                                                     \
      cudaFuncSetAttribute(attn_bwd_cross_kernel<HD_, KT_>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm);  \
      attr = true;                                                                                                   \
    }                                                                                                                \
    attn_bwd_cross_kernel<HD_, KT_><<<gs, 128, sm, ST(stream)>>>(CBF(dout), lddo, CBF(q), ldq, CBF(k), ldk, CBF(v),  \
                                                                 ldv, lse, BF(dq), lddq, BF(dk), lddk, BF(dv), lddv, \
                                                                 (int)H, (int)Tq, (int)Tk, scale, sl2);              \
  } while (0)
    if (hd == 64) { if (Tk <= 64) BWD_CROSS(64, 64); else BWD_CROSS(64, 80); }
    else { if (Tk <= 64) BWD_CROSS(32, 64); else BWD_CROSS(32, 80); }
#undef BWD_CROSS
    return check_launch("md_attn_bwd");
  }
  // the delta kernel holds a whole token row (all heads) in one warp: H*hd <= 2048, i.e. at most 16 heads at head_dim 128
  if (H * hd > 2048) return md_set_error(MD_ERR_UNSUPPORTED, "md_attn_bwd: H*hd must be <= 2048");
  long long blocks = (B * Tq + 7) / 8;
  if (blocks > 132 * 8) blocks = 132 * 8;
  if (hd == 128)
    attn_delta_kernel<128><<<(unsigned)blocks, 256, 0, ST(stream)>>>(CBF(dout), lddo, CBF(o), ldo, delta, B * Tq, (int)H,
                                                                     (int)Tq);
  else if (hd == 64)
    attn_delta_kernel<64><<<(unsigned)blocks, 256, 0, ST(stream)>>>(CBF(dout), lddo, CBF(o), ldo, delta, B * Tq, (int)H,
                                                                    (int)Tq);
  else
    attn_delta_kernel<32><<<(unsigned)blocks, 256, 0, ST(stream)>>>(CBF(dout), lddo, CBF(o), ldo, delta, B * Tq, (int)H,
                                                                    (int)Tq);
  dim3 gkv((unsigned)((Tk + kTile - 1) / kTile), (unsigned)H, (unsigned)B);
  dim3 gq((unsigned)((Tq + kTile - 1) / kTile), (unsigned)H, (unsigned)B);
#define BWD_GENERIC(HD_)                                                                                             \
  do {                                                                                                               \
    static bool attr = false;                                                                                        \
    const size_t sm_dq = (size_t)4 * kTile * Smem<HD_>::kPitch * sizeof(__nv_bfloat16);                              \
    const size_t sm_kv = sm_dq + 4 * kTile * sizeof(float);                                                          \
    if (!attr) {                                                                                                     \
      cudaFuncSetAttribute(attn_bwd_dkdv_kernel<HD_>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm_kv);     \
      cudaFuncSetAttribute(attn_bwd_dq_kernel<HD_>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm_dq);       \
      attr = true;                                                                                                   \
    }                                                                                                                \
    attn_bwd_dkdv_kernel<HD_><<<gkv, 128, sm_kv, ST(stream)>>>(CBF(dout), lddo, CBF(q), ldq, CBF(k), ldk, CBF(v),    \
                                                               ldv, lse, delta, BF(dk), lddk, BF(dv), lddv, (int)H,  \
                                                               (int)Tq, (int)Tk, scale, sl2);                        \
    attn_bwd_dq_kernel<HD_><<<gq, 128, sm_dq, ST(stream)>>>(CBF(dout), lddo, CBF(q), ldq, CBF(k), ldk, CBF(v), ldv,  \
                                                            lse, delta, BF(dq), lddq, (int)H, (int)Tq, (int)Tk,      \
                                                            scale, sl2);                                             \
  } while (0)
  if (hd == 128) BWD_GENERIC(128); else if (hd == 64) BWD_GENERIC(64); else BWD_GENERIC(32);
#undef BWD_GENERIC
  return check_launch("md_attn_bwd");
}

extern "C" int md_attn_bwd_tc(const void* dout, int64_t lddo, const void* q, int64_t ldq, const void* k, int64_t ldk,
                              const void* v, int64_t ldv, const void* o, int64_t ldo, const float* lse, float* delta,
                              void* dq, int64_t lddq, void* dk, int64_t lddk, void* dv, int64_t lddv, int64_t B, int64_t H,
                              int64_t Tq, int64_t Tk, int64_t hd, void* stream) {
  if (int rc = check_attn("md_attn_bwd_tc: bad sizes", B, H, Tq, Tk, hd, (lddo | ldq | ldk | ldv | ldo | lddq | lddk | lddv),
                          addr_or({dout, q, k, v, o, dq, dk, dv})))
    return rc;
  if (B == 0) return 0;
  if (hd != 64) return md_set_error(MD_ERR_UNSUPPORTED, "md_attn_bwd_tc: needs head_dim 64");
  if (!dout || !q || !k || !v || !o || !lse || !delta || !dq || !dk || !dv)
    return md_set_error(MD_ERR_INVALID, "md_attn_bwd_tc: null pointer");
  // the delta kernel holds a whole token row (all heads) in one warp: H*hd <= 2048, i.e. at most 32 heads of 64
  if (H * hd > 2048) return md_set_error(MD_ERR_UNSUPPORTED, "md_attn_bwd_tc: H*hd must be <= 2048");
  long long blocks = (B * Tq + 7) / 8;
  if (blocks > 132 * 8) blocks = 132 * 8;
  attn_delta_kernel<64><<<(unsigned)blocks, 256, 0, ST(stream)>>>(CBF(dout), lddo, CBF(o), ldo, delta, B * Tq, (int)H, (int)Tq);
  if (int rc = check_launch("md_attn_bwd_tc (delta)")) return rc;
  return attn_bwd_wgmma(dout, lddo, q, ldq, k, ldk, v, ldv, lse, delta, dq, lddq, dk, lddk, dv, lddv, B, H, Tq, Tk, ST(stream));
}
