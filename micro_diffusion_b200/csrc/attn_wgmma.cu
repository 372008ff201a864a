// Attention on the Hopper warpgroup tensor cores (TMA + wgmma): forward for head_dim 64 and Tk <= 256 (below), forward
// for head_dim 128 and any Tk (after it), backward for head_dim 64 and any Tk (further down).
//
// Contract = md_attn_fwd: softmax(Q K^T / sqrt(hd)) V, non-causal (F.scaled_dot_product_attention at reference
// utils.py:188-193 self, 127-132 cross); q / k / v are column slices of the packed projection buffers; lse in the
// log2 domain.  Envelope: all keys of one (sample, head) fit one S tile of <= 256 columns (every sequence of the res-256
// configs: 64, 77, 256).
//
// One CTA = one warpgroup = 64 query rows of one (sample, head).  One TMA transaction brings Q (64 x 64) and the whole K
// and V of the head (keys rounded up to 64, zero-filled past Tk) into 128B-swizzled shared memory.  S = Q K^T runs as
// up to four m64n64k16 wgmma chains (fp32 in registers), the softmax is taken on the whole row in registers (all of S is
// resident: no online rescale; a row lives in the four lanes of a quad), and P goes back into the tensor core straight
// from the registers as the A operand of O = P V (V read through an MN-major descriptor).
#include <cuda.h>

#include "common.cuh"
#include "ptx.cuh"
#include "tensormap.cuh"

namespace md {
namespace attn_wg {

constexpr int kHd = 64;
constexpr int kQ = 64;
constexpr int kMaxKeys = 256;
constexpr int kOffK = kQ * kHd * 2;                 // 8 KB of Q
constexpr int kOffV = kOffK + kMaxKeys * kHd * 2;   // 32 KB of K
constexpr int kOffBar = kOffV + kMaxKeys * kHd * 2; // 32 KB of V
constexpr int kSmemBytes = kOffBar + 64 + 1024;

__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ uint32_t pack2(float a, float b) {
  __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&v);
}

__global__ void __launch_bounds__(128)
attn_fwd_wgmma_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                      const __grid_constant__ CUtensorMap tmV, __nv_bfloat16* __restrict__ o, long long ldo,
                      float* __restrict__ lse, int H, int Tq, int Tk, float sl2) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem + kOffBar);
  const int qb = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int kc = (Tk + 63) >> 6;  // 64-key chunks (1..4)
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmK);
    tma_prefetch_desc(&tmV);
    mbar_init(bar, 1);
    mbar_fence_init();
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    mbar_expect_tx(bar, (kQ + 2 * kc * 64) * kHd * 2);
    tma_load_3d(&tmQ, bar, smem, h * kHd, qb * kQ, b);
    tma_load_3d(&tmK, bar, smem + kOffK, h * kHd, 0, b);
    tma_load_3d(&tmV, bar, smem + kOffV, h * kHd, 0, b);
  }
  mbar_wait(bar, 0);

  // ---- S = Q K^T: Q and K both K-major (head_dim contiguous), 8-row groups 1024 B apart
  float s[4][32];
  const uint64_t dq = wgmma_smem_desc(smem_u32(smem), 16, 1024);
  wgmma_fence();
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    if (c < kc) {
      const uint64_t dk = wgmma_smem_desc(smem_u32(smem + kOffK + c * 64 * 128), 16, 1024);
#pragma unroll
      for (int k = 0; k < kHd / 16; ++k) wgmma_m64n64k16<0, 0>(s[c], dq + 2 * k, dk + 2 * k, k > 0 ? 1u : 0u);
    }
  }
  wgmma_commit();
  wgmma_wait<0>();
#pragma unroll
  for (int c = 0; c < 4; ++c) wgmma_fence_operands(s[c]);

  // ---- whole-row softmax in registers: thread holds rows r0 = 16 warp + lane / 4 and r0 + 8 (i = 0, 1), columns
  // 64 c + 8 j + 2 (lane % 4) + e of s[c][4 j + 2 i + e]
  const int cq = 2 * (lane & 3);
  float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    if (c < kc) {
#pragma unroll
      for (int j = 0; j < 8; ++j)
#pragma unroll
        for (int i = 0; i < 2; ++i)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            float& v = s[c][4 * j + 2 * i + e];
            if (c * 64 + 8 * j + cq + e >= Tk) v = -INFINITY;
            mx[i] = fmaxf(mx[i], v);
          }
    }
  }
  float m2[2], l[2] = {0.f, 0.f};
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    mx[i] = fmaxf(mx[i], __shfl_xor_sync(0xffffffffu, mx[i], 1));
    mx[i] = fmaxf(mx[i], __shfl_xor_sync(0xffffffffu, mx[i], 2));
    m2[i] = mx[i] * sl2;
  }
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    if (c < kc) {
#pragma unroll
      for (int j = 0; j < 8; ++j)
#pragma unroll
        for (int i = 0; i < 2; ++i)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            float& v = s[c][4 * j + 2 * i + e];
            v = ex2_approx(fmaf(v, sl2, -m2[i]));
            l[i] += v;
          }
    }
  }
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    l[i] += __shfl_xor_sync(0xffffffffu, l[i], 1);
    l[i] += __shfl_xor_sync(0xffffffffu, l[i], 2);
  }

  // ---- O = P V: P (bf16) from registers -- the accumulator fragment of 16 keys is the A fragment of one k16 step --,
  // V MN-major (head_dim contiguous), 16-key steps 2048 B apart
  float oacc[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) oacc[i] = 0.f;
  const uint64_t dv = wgmma_smem_desc(smem_u32(smem + kOffV), 64 * 128, 1024);
  uint32_t pa[4][4][4];  // all of P as bf16 A fragments first: the fence below then covers every register-sourced wgmma
#pragma unroll
  for (int c = 0; c < 4; ++c)
#pragma unroll
    for (int t = 0; t < 4; ++t)
#pragma unroll
      for (int r = 0; r < 4; ++r) pa[c][t][r] = pack2(s[c][8 * t + 2 * r], s[c][8 * t + 2 * r + 1]);
  wgmma_fence();
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    if (c < kc) {
#pragma unroll
      for (int t = 0; t < 4; ++t)
        wgmma_m64n64k16_rs<1>(oacc, pa[c][t], dv + static_cast<uint64_t>((c * 4 + t) * 128), (c > 0 || t > 0) ? 1u : 0u);
    }
  }
  wgmma_commit();
  wgmma_wait<0>();
  wgmma_fence_operands(oacc);

#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int row = qb * kQ + warp * 16 + (lane >> 2) + 8 * i;
    if (row < Tq) {
      const float inv = __fdividef(1.f, l[i]);
      __nv_bfloat16* dst = o + (static_cast<long long>(b) * Tq + row) * ldo + h * kHd + cq;
#pragma unroll
      for (int j = 0; j < 8; ++j)
        *reinterpret_cast<uint32_t*>(dst + 8 * j) = pack2(oacc[4 * j + 2 * i] * inv, oacc[4 * j + 2 * i + 1] * inv);
      if ((lane & 3) == 0) lse[(static_cast<long long>(b) * H + h) * Tq + row] = m2[i] + __log2f(l[i]);
    }
  }
}

// ------------------------------------------------------------------------------------------ head_dim 128 forward
// Same contract for head_dim 128 and any Tk.  All keys of a head in one S tile no longer fit next to a 64 x 128 O
// accumulator (a 64 x 256 S tile alone is 128 fp32 registers per thread), so this kernel runs an online softmax over
// 64-key chunks (log2 domain, the running max rescales l and O per chunk, as in the mma.sync kernels).
//
// One CTA = one warpgroup = 64 query rows of one (sample, head).  Every 64-column half of a 128-column row is its own
// 128B-swizzled TMA box (64 rows x 128 B), so Q is two boxes and each key chunk is two K boxes and two V boxes.  K / V
// chunks stream through a two-stage ring: chunk c + 2 is loaded into the stage of chunk c once every warp is done with
// it, so the load of chunk c + 1 overlaps the math of chunk c.  S = Q K^T of a chunk is 8 k16 steps of m64n64k16 (the
// first four in the first column box); O += P V is two m64n64k16 chains (one per 64-column half of O) with P as the
// register A operand, V read MN-major.  126 registers, no spills, 81 KB of shared memory: two CTAs per SM.
constexpr int kHd128 = 128;
constexpr int kBox = 64 * 64 * 2;                       // one 64-row x 64-column bf16 box: 8 KB
constexpr int k128OffKV = 2 * kBox;                     // Q: two boxes
constexpr int k128Stage = 4 * kBox;                     // K (two boxes) | V (two boxes)
constexpr int k128OffBar = k128OffKV + 2 * k128Stage;   // two stages
constexpr int k128SmemBytes = k128OffBar + 64 + 1024;

__global__ void __launch_bounds__(128)
attn_fwd_wgmma128_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                         const __grid_constant__ CUtensorMap tmV, __nv_bfloat16* __restrict__ o, long long ldo,
                         float* __restrict__ lse, int H, int Tq, int Tk, float sl2) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + k128OffBar);  // one barrier per stage
  const int qb = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int nc = (Tk + 63) >> 6;  // 64-key chunks
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int col0 = h * kHd128;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmK);
    tma_prefetch_desc(&tmV);
    mbar_init(&full[0], 1);
    mbar_init(&full[1], 1);
    mbar_fence_init();
  }
  __syncthreads();
  // issued by thread 0: key chunk c (and Q with the first) into stage c & 1, zero-filled past Tq / Tk
  auto load_chunk = [&](int c) {
    uint8_t* st = smem + k128OffKV + (c & 1) * k128Stage;
    uint64_t* bar = &full[c & 1];
    mbar_expect_tx(bar, k128Stage + (c == 0 ? 2 * kBox : 0));
    if (c == 0) {
      tma_load_3d(&tmQ, bar, smem, col0, qb * kQ, b);
      tma_load_3d(&tmQ, bar, smem + kBox, col0 + 64, qb * kQ, b);
    }
    tma_load_3d(&tmK, bar, st, col0, c * 64, b);
    tma_load_3d(&tmK, bar, st + kBox, col0 + 64, c * 64, b);
    tma_load_3d(&tmV, bar, st + 2 * kBox, col0, c * 64, b);
    tma_load_3d(&tmV, bar, st + 3 * kBox, col0 + 64, c * 64, b);
  };
  if (threadIdx.x == 0) {
    load_chunk(0);
    if (nc > 1) load_chunk(1);
  }

  // fragment of thread t: rows r0 = 16 warp + lane / 4 and r0 + 8 (i = 0, 1), columns 8 j + 2 (lane % 4) + e of
  // s[4 j + 2 i + e] (keys of the chunk) and of o[half][4 j + 2 i + e] (head columns 64 half + ...)
  const int cq = 2 * (lane & 3);
  float oacc[2][32];
#pragma unroll
  for (int x = 0; x < 2; ++x)
#pragma unroll
    for (int i = 0; i < 32; ++i) oacc[x][i] = 0.f;
  float m2[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};  // running max (log2 domain) and per-thread partial sum
  const uint32_t sq = smem_u32(smem);

  for (int c = 0; c < nc; ++c) {
    const uint8_t* st = smem + k128OffKV + (c & 1) * k128Stage;
    mbar_wait(&full[c & 1], (c >> 1) & 1);

    // ---- S = Q K^T over the 128 head columns: k16 steps 0..3 in the first column box, 4..7 in the second
    float s[32];
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < kHd128 / 16; ++k) {
      const uint64_t dq = wgmma_smem_desc(sq + (k >> 2) * kBox, 16, 1024) + 2 * (k & 3);
      const uint64_t dk = wgmma_smem_desc(smem_u32(st) + (k >> 2) * kBox, 16, 1024) + 2 * (k & 3);
      wgmma_m64n64k16<0, 0>(s, dq, dk, k > 0 ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_operands(s);

    // ---- online softmax: mask keys past Tk, new running max, rescale of l and O
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          float& v = s[4 * j + 2 * i + e];
          if (c * 64 + 8 * j + cq + e >= Tk) v = -INFINITY;
          mx[i] = fmaxf(mx[i], v);
        }
    float corr[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      mx[i] = fmaxf(mx[i], __shfl_xor_sync(0xffffffffu, mx[i], 1));
      mx[i] = fmaxf(mx[i], __shfl_xor_sync(0xffffffffu, mx[i], 2));
      const float mn = fmaxf(m2[i], mx[i] * sl2);  // every chunk has a valid key: finite
      corr[i] = ex2_approx(m2[i] - mn);             // first chunk: exp2(-inf) = 0
      m2[i] = mn;
      l[i] *= corr[i];
    }
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          float& v = s[4 * j + 2 * i + e];
          v = ex2_approx(fmaf(v, sl2, -m2[i]));
          l[i] += v;
        }
#pragma unroll
    for (int x = 0; x < 2; ++x)
#pragma unroll
      for (int j = 0; j < 8; ++j)
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          oacc[x][4 * j + 2 * i] *= corr[i];
          oacc[x][4 * j + 2 * i + 1] *= corr[i];
        }

    // ---- O += P V: P (bf16) from registers, V MN-major (head columns contiguous), 16-key steps 2048 B apart
    uint32_t pa[4][4];
#pragma unroll
    for (int t = 0; t < 4; ++t)
#pragma unroll
      for (int r = 0; r < 4; ++r) pa[t][r] = pack2(s[8 * t + 2 * r], s[8 * t + 2 * r + 1]);
    const uint64_t dv0 = wgmma_smem_desc(smem_u32(st + 2 * kBox), 64 * 128, 1024);
    const uint64_t dv1 = wgmma_smem_desc(smem_u32(st + 3 * kBox), 64 * 128, 1024);
    wgmma_fence();
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      wgmma_m64n64k16_rs<1>(oacc[0], pa[t], dv0 + static_cast<uint64_t>(t * 128), 1u);
      wgmma_m64n64k16_rs<1>(oacc[1], pa[t], dv1 + static_cast<uint64_t>(t * 128), 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_operands(oacc[0]);
    wgmma_fence_operands(oacc[1]);
    __syncthreads();  // every warp is done with this stage before chunk c + 2 lands in it
    if (threadIdx.x == 0 && c + 2 < nc) load_chunk(c + 2);
  }

#pragma unroll
  for (int i = 0; i < 2; ++i) {
    l[i] += __shfl_xor_sync(0xffffffffu, l[i], 1);
    l[i] += __shfl_xor_sync(0xffffffffu, l[i], 2);
  }
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int row = qb * kQ + warp * 16 + (lane >> 2) + 8 * i;
    if (row < Tq) {
      const float inv = __fdividef(1.f, l[i]);
      __nv_bfloat16* dst = o + (static_cast<long long>(b) * Tq + row) * ldo + col0 + cq;
#pragma unroll
      for (int x = 0; x < 2; ++x)
#pragma unroll
        for (int j = 0; j < 8; ++j)
          *reinterpret_cast<uint32_t*>(dst + 64 * x + 8 * j) =
              pack2(oacc[x][4 * j + 2 * i] * inv, oacc[x][4 * j + 2 * i + 1] * inv);
      if ((lane & 3) == 0) lse[(static_cast<long long>(b) * H + h) * Tq + row] = m2[i] + __log2f(l[i]);
    }
  }
}

// bf16 [batch][rows][cols] view, box = [1][box_rows][64 columns], 128B swizzle.
int make_map(CUtensorMap* map, const void* ptr, long long cols, long long rows, long long batch, long long ld,
             int box_rows) {
  const TmapKey key = make_tmap_key(ptr, cols, rows, batch, ld, rows * ld, 64, box_rows, CU_TENSOR_MAP_SWIZZLE_128B,
                                    CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
  if (cached_tensor_map(map, key) != CUDA_SUCCESS)
    return md_set_error(MD_ERR_CUDA, "attention (wgmma): cuTensorMapEncodeTiled failed");
  return 0;
}

}  // namespace attn_wg
}  // namespace md

extern "C" int md_attn_fwd_tc(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, void* o,
                              int64_t ldo, float* lse, int64_t B, int64_t H, int64_t Tq, int64_t Tk, int64_t hd,
                              void* stream) {
  using namespace md;
  using namespace md::attn_wg;
  if (B <= 0 || H <= 0 || Tq <= 0 || Tk <= 0) return B == 0 ? 0 : md_set_error(MD_ERR_INVALID, "md_attn_fwd_tc: bad sizes");
  if (!(hd == kHd && Tk <= kMaxKeys) && hd != kHd128)
    return md_set_error(MD_ERR_UNSUPPORTED, "md_attn_fwd_tc: needs head_dim 64 with Tk <= 256, or head_dim 128");
  if (!q || !k || !v || !o || !lse) return md_set_error(MD_ERR_INVALID, "md_attn_fwd_tc: null pointer");
  const uintptr_t align = reinterpret_cast<uintptr_t>(q) | reinterpret_cast<uintptr_t>(k) | reinterpret_cast<uintptr_t>(v) |
                          reinterpret_cast<uintptr_t>(o);
  if ((align & 15) != 0 || ((ldq | ldk | ldv | ldo) % 8) != 0)
    return md_set_error(MD_ERR_INVALID, "md_attn_fwd_tc: operands must be 16-byte aligned with pitches % 8 == 0");
  CUtensorMap tmQ, tmK, tmV;
  const dim3 grid(static_cast<unsigned>((Tq + kQ - 1) / kQ), static_cast<unsigned>(H), static_cast<unsigned>(B));
  const float sl2 = 1.4426950408889634f / sqrtf(static_cast<float>(hd));
  if (hd == kHd128) {
    if (int rc = make_map(&tmQ, q, H * hd, Tq, B, ldq, kQ)) return rc;
    if (int rc = make_map(&tmK, k, H * hd, Tk, B, ldk, 64)) return rc;
    if (int rc = make_map(&tmV, v, H * hd, Tk, B, ldv, 64)) return rc;
    static bool attr128 = false;
    if (!attr128) {
      cudaError_t e =
          cudaFuncSetAttribute(attn_fwd_wgmma128_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, k128SmemBytes);
      if (e != cudaSuccess) return md_set_error(MD_ERR_CUDA, cudaGetErrorString(e));
      attr128 = true;
    }
    attn_fwd_wgmma128_kernel<<<grid, 128, k128SmemBytes, reinterpret_cast<cudaStream_t>(stream)>>>(
        tmQ, tmK, tmV, reinterpret_cast<__nv_bfloat16*>(o), ldo, lse, static_cast<int>(H), static_cast<int>(Tq),
        static_cast<int>(Tk), sl2);
    return check_launch("md_attn_fwd_tc");
  }
  const int kbox = static_cast<int>((Tk + 63) / 64 * 64);
  if (int rc = make_map(&tmQ, q, H * hd, Tq, B, ldq, kQ)) return rc;
  if (int rc = make_map(&tmK, k, H * hd, Tk, B, ldk, kbox)) return rc;
  if (int rc = make_map(&tmV, v, H * hd, Tk, B, ldv, kbox)) return rc;
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(attn_fwd_wgmma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes);
    if (e != cudaSuccess) return md_set_error(MD_ERR_CUDA, cudaGetErrorString(e));
    attr = true;
  }
  attn_fwd_wgmma_kernel<<<grid, 128, kSmemBytes, reinterpret_cast<cudaStream_t>(stream)>>>(
      tmQ, tmK, tmV, reinterpret_cast<__nv_bfloat16*>(o), ldo, lse, static_cast<int>(H), static_cast<int>(Tq),
      static_cast<int>(Tk), sl2);
  return check_launch("md_attn_fwd_tc");
}

// ================================================================================================ backward
// dQ, dK, dV of the same attention for head_dim 64, any Tk, as two wgmma kernels (the split of the mma.sync backward:
// no atomics, deterministic).  delta = rowsum(dO * O) comes in precomputed; lse in the log2 domain.
//   dkdv: one warpgroup per (sample, head, 64-key block), looping over 64-query blocks:
//         S^T = K Q^T, dP^T = V dO^T (registers), P^T = exp2(S^T * scale_log2 - lse), dS^T = P^T (dP^T - delta),
//         dV += P^T dO, dK += dS^T Q (A operands from registers, dO / Q read MN-major).
//   dq:   one warpgroup per (sample, head, 64-query block), looping over 64-key blocks:
//         S = Q K^T, dP = dO V^T, P, dS as above, dQ += dS K (K read MN-major).
// Every iteration loads its two 64 x 64 tiles with one TMA transaction (zero-filled past Tq / Tk).
namespace md {
namespace attn_wg {

constexpr int kTileBytes = 64 * kHd * 2;  // 8 KB
// shared memory: [0] fixed tile A, [1] fixed tile B, [2] streamed tile A, [3] streamed tile B, barriers
constexpr int kBwdSmemBytes = 4 * kTileBytes + 64 + 1024;

// acc (64 x 64 fp32 fragment) -> bf16 A fragments of the four k16 steps
__device__ __forceinline__ void to_a_frags(const float (&acc)[32], uint32_t (&a)[4][4]) {
#pragma unroll
  for (int t = 0; t < 4; ++t)
#pragma unroll
    for (int r = 0; r < 4; ++r) a[t][r] = pack2(acc[8 * t + 2 * r], acc[8 * t + 2 * r + 1]);
}

// C (64 x 64) = X Y^T with X, Y 64 x 64 K-major tiles in shared memory
__device__ __forceinline__ void mm_nt(float (&c)[32], const uint8_t* x, const uint8_t* y) {
  const uint64_t dx = wgmma_smem_desc(smem_u32(x), 16, 1024), dy = wgmma_smem_desc(smem_u32(y), 16, 1024);
#pragma unroll
  for (int k = 0; k < kHd / 16; ++k) wgmma_m64n64k16<0, 0>(c, dx + 2 * k, dy + 2 * k, k > 0 ? 1u : 0u);
}
// C (64 x 64) += A Y with A in registers (bf16 fragments) and Y a 64 x 64 tile read MN-major
__device__ __forceinline__ void mm_rs(float (&c)[32], const uint32_t (&a)[4][4], const uint8_t* y) {
  const uint64_t dy = wgmma_smem_desc(smem_u32(y), 64 * 128, 1024);
#pragma unroll
  for (int t = 0; t < 4; ++t) wgmma_m64n64k16_rs<1>(c, a[t], dy + static_cast<uint64_t>(t * 128), 1u);
}

__global__ void __launch_bounds__(128)
attn_bwd_wgmma_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                      const __grid_constant__ CUtensorMap tmV, const __grid_constant__ CUtensorMap tmdO,
                      const float* __restrict__ lse, const float* __restrict__ delta, __nv_bfloat16* __restrict__ dq,
                      long long lddq, __nv_bfloat16* __restrict__ dk, long long lddk, __nv_bfloat16* __restrict__ dv,
                      long long lddv, int H, int Tq, int Tk, float scale, float sl2, int kv_blocks) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem + 4 * kTileBytes);
  uint8_t* f0 = smem;                   // dkdv: K, dq: Q
  uint8_t* f1 = smem + kTileBytes;      // dkdv: V, dq: dO
  uint8_t* s0 = smem + 2 * kTileBytes;  // dkdv: Q, dq: K
  uint8_t* s1 = smem + 3 * kTileBytes;  // dkdv: dO, dq: V
  const bool kv_role = static_cast<int>(blockIdx.x) < kv_blocks;   // dkdv CTA, else dq CTA
  const int blk = kv_role ? blockIdx.x : blockIdx.x - kv_blocks;
  const int h = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int cq = 2 * (lane & 3);
  const int r0 = warp * 16 + (lane >> 2);   // fragment rows r0, r0 + 8
  const long long stat0 = (static_cast<long long>(b) * H + h) * Tq;
  const int n_iter = kv_role ? (Tq + 63) / 64 : (Tk + 63) / 64;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmQ); tma_prefetch_desc(&tmK); tma_prefetch_desc(&tmV); tma_prefetch_desc(&tmdO);
    mbar_init(bar, 1);
    mbar_fence_init();
  }
  __syncthreads();
  float acc0[32], acc1[32];   // dkdv: dV, dK;  dq: dQ
#pragma unroll
  for (int i = 0; i < 32; ++i) acc0[i] = acc1[i] = 0.f;

  for (int it = 0; it < n_iter; ++it) {
    if (threadIdx.x == 0) {
      if (it == 0) {
        mbar_expect_tx(bar, 4 * kTileBytes);
        if (kv_role) {
          tma_load_3d(&tmK, bar, f0, h * kHd, blk * 64, b);
          tma_load_3d(&tmV, bar, f1, h * kHd, blk * 64, b);
        } else {
          tma_load_3d(&tmQ, bar, f0, h * kHd, blk * 64, b);
          tma_load_3d(&tmdO, bar, f1, h * kHd, blk * 64, b);
        }
      } else {
        mbar_expect_tx(bar, 2 * kTileBytes);
      }
      if (kv_role) {
        tma_load_3d(&tmQ, bar, s0, h * kHd, it * 64, b);
        tma_load_3d(&tmdO, bar, s1, h * kHd, it * 64, b);
      } else {
        tma_load_3d(&tmK, bar, s0, h * kHd, it * 64, b);
        tma_load_3d(&tmV, bar, s1, h * kHd, it * 64, b);
      }
    }
    mbar_wait(bar, it & 1);

    float sc[32], dp[32];
    wgmma_fence();
    if (kv_role) {
      mm_nt(sc, f0, s0);   // S^T = K Q^T   [keys][queries]
      mm_nt(dp, f1, s1);   // dP^T = V dO^T
    } else {
      mm_nt(sc, f0, s0);   // S = Q K^T     [queries][keys]
      mm_nt(dp, f1, s1);   // dP = dO V^T
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_operands(sc);
    wgmma_fence_operands(dp);

    // P and dS; query index / key index of fragment element (i, j, e): row r0 + 8 i, column 8 j + cq + e
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      float lrow = 0.f, drow = 0.f;
      if (!kv_role) {
        const int q = blk * 64 + r0 + 8 * i;
        lrow = q < Tq ? lse[stat0 + q] : INFINITY;
        drow = q < Tq ? delta[stat0 + q] : 0.f;
      }
#pragma unroll
      for (int j = 0; j < 8; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int col = it * 64 + 8 * j + cq + e;
          float l2, dl;
          bool valid;
          if (kv_role) {   // column = query
            valid = col < Tq;
            l2 = valid ? lse[stat0 + col] : INFINITY;
            dl = valid ? delta[stat0 + col] : 0.f;
          } else {         // column = key
            valid = col < Tk;
            l2 = lrow;
            dl = drow;
          }
          const int x = 4 * j + 2 * i + e;
          const float p = valid ? ex2_approx(fmaf(sc[x], sl2, -l2)) : 0.f;
          sc[x] = p;
          dp[x] = p * (dp[x] - dl);
        }
    }
    uint32_t pa[4][4], da[4][4];
    to_a_frags(sc, pa);
    to_a_frags(dp, da);
    wgmma_fence();
    if (kv_role) {
      mm_rs(acc0, pa, s1);   // dV += P^T dO
      mm_rs(acc1, da, s0);   // dK += dS^T Q
    } else {
      mm_rs(acc0, da, s0);   // dQ += dS K
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_operands(acc0);
    wgmma_fence_operands(acc1);
    __syncthreads();   // every warp is done with the streamed tiles before the next TMA overwrites them
  }

#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int row = blk * 64 + r0 + 8 * i;
    if (kv_role) {
      if (row < Tk) {
        __nv_bfloat16* pv = dv + (static_cast<long long>(b) * Tk + row) * lddv + h * kHd + cq;
        __nv_bfloat16* pk = dk + (static_cast<long long>(b) * Tk + row) * lddk + h * kHd + cq;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          *reinterpret_cast<uint32_t*>(pv + 8 * j) = pack2(acc0[4 * j + 2 * i], acc0[4 * j + 2 * i + 1]);
          *reinterpret_cast<uint32_t*>(pk + 8 * j) = pack2(acc1[4 * j + 2 * i] * scale, acc1[4 * j + 2 * i + 1] * scale);
        }
      }
    } else if (row < Tq) {
      __nv_bfloat16* pq = dq + (static_cast<long long>(b) * Tq + row) * lddq + h * kHd + cq;
#pragma unroll
      for (int j = 0; j < 8; ++j)
        *reinterpret_cast<uint32_t*>(pq + 8 * j) = pack2(acc0[4 * j + 2 * i] * scale, acc0[4 * j + 2 * i + 1] * scale);
    }
  }
}

}  // namespace attn_wg

// Backward on wgmma (head_dim 64); delta = rowsum(dO * O) precomputed by the caller (attn.cu).
int attn_bwd_wgmma(const void* dout, int64_t lddo, const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v,
                   int64_t ldv, const float* lse, const float* delta, void* dq, int64_t lddq, void* dk, int64_t lddk,
                   void* dv, int64_t lddv, int64_t B, int64_t H, int64_t Tq, int64_t Tk, cudaStream_t stream) {
  using namespace attn_wg;
  CUtensorMap tmQ, tmK, tmV, tmdO;
  if (int rc = make_map(&tmQ, q, H * kHd, Tq, B, ldq, 64)) return rc;
  if (int rc = make_map(&tmK, k, H * kHd, Tk, B, ldk, 64)) return rc;
  if (int rc = make_map(&tmV, v, H * kHd, Tk, B, ldv, 64)) return rc;
  if (int rc = make_map(&tmdO, dout, H * kHd, Tq, B, lddo, 64)) return rc;
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(attn_bwd_wgmma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kBwdSmemBytes);
    if (e != cudaSuccess) return md_set_error(MD_ERR_CUDA, cudaGetErrorString(e));
    attr = true;
  }
  const int kv_blocks = static_cast<int>((Tk + 63) / 64), q_blocks = static_cast<int>((Tq + 63) / 64);
  const dim3 grid(static_cast<unsigned>(kv_blocks + q_blocks), static_cast<unsigned>(H), static_cast<unsigned>(B));
  const float scale = 1.f / sqrtf(static_cast<float>(kHd));
  attn_bwd_wgmma_kernel<<<grid, 128, kBwdSmemBytes, stream>>>(
      tmQ, tmK, tmV, tmdO, lse, delta, reinterpret_cast<__nv_bfloat16*>(dq), lddq, reinterpret_cast<__nv_bfloat16*>(dk),
      lddk, reinterpret_cast<__nv_bfloat16*>(dv), lddv, static_cast<int>(H), static_cast<int>(Tq), static_cast<int>(Tk),
      scale, scale * 1.4426950408889634f, kv_blocks);
  return check_launch("md_attn_bwd_tc");
}

}  // namespace md
