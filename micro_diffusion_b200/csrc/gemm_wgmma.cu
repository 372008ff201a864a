// Persistent warp-specialised bf16 GEMM for sm_90a: TMA -> 128B-swizzled smem ring -> wgmma (fp32 accumulators in
// registers) -> epilogue straight from the accumulator registers with fused element-wise tails.
//
// Replaces, on the MicroDiT training path, every nn.Linear / einsum contraction the reference sends
// to cuBLAS: qkv/proj (reference micro_diffusion/models/utils.py:172-173), cross-attention q/kv/proj
// (utils.py:109-111), SwiGLU w1/w2/w3 (dit.py:84-89), the expert einsums (dit.py:135-137), the
// adaLN / stem / mixer-map / final linears, and all their dgrad / wgrad counterparts.
//
// Two operand layouts (template kMN):
//   kMN=false  "NT":  C[M,N] = sum_k A[M,k] * B[N,k]     A,B row-major with k contiguous (K-major)
//   kMN=true   "TN":  C[P,Q] = sum_r A[r,P] * B[r,Q]     A,B row-major with the reduction index r
//                     strided (MN-major wgmma operands) -- the weight-gradient contraction.
// Tiles of 128 x BLOCK_N (128 or 256), 64-deep k-blocks.  Roles: warpgroup 0 = TMA producer (one thread; it hands its
// registers to the others), warpgroups 1 and 2 = MMA + epilogue, each owning 64 rows of the tile (m64nNk16 wgmma).  The
// producer runs ahead into the next tile while the MMA warpgroups run the epilogue of the current one, so operand loads
// overlap the epilogue.
#include "gemm_wgmma.cuh"

#include <stdio.h>
#include <stdlib.h>

#include <type_traits>

#include "ptx.cuh"
#include "tensormap.cuh"

namespace md {

constexpr int kBlockM = 128;
constexpr int kBlockK = 64;  // 64 bf16 = 128 B = one swizzle row
constexpr int kWgK = 16;
constexpr int kThreads = 384;  // producer warpgroup + two MMA warpgroups

template <int BLOCK_N>
struct GemmCfg {
  static constexpr int kStageBytesA = kBlockM * kBlockK * 2;
  static constexpr int kStageBytesB = BLOCK_N * kBlockK * 2;
  static constexpr int kStageBytes = kStageBytesA + kStageBytesB;
  static constexpr int kStages = (192 * 1024) / kStageBytes;  // 4 (BLOCK_N 256) or 6 (BLOCK_N 128) of the 227 KB
  static constexpr int kSmemBytes = kStages * kStageBytes + 1024 /*align*/ + 256 /*barriers*/;
};

// Cheap activations for the epilogue (it shares 4 issue ports with nothing else but is on the critical path of
// short-K tiles).  erf by Abramowitz-Stegun 7.1.26 (|err| < 1.5e-7, far below bf16 resolution).
__device__ __forceinline__ float gelu_erf_fast(float x) {
  const float z = fabsf(x) * 0.70710678118654752440f;
  const float t = __fdividef(1.0f, fmaf(0.3275911f, z, 1.0f));
  float poly = fmaf(1.061405429f, t, -1.453152027f);
  poly = fmaf(poly, t, 1.421413741f);
  poly = fmaf(poly, t, -0.284496736f);
  poly = fmaf(poly, t, 0.254829592f);
  const float e = 1.0f - poly * t * __expf(-z * z);  // erf(|x|/sqrt2)
  return 0.5f * x * (1.0f + copysignf(e, x));
}
__device__ __forceinline__ float gelu_tanh_fast(float x) {
  const float u = 0.7978845608028654f * fmaf(0.044715f * x, x * x, x);
  const float e = __expf(2.0f * u);                    // tanh(u) = 1 - 2/(e^{2u}+1)
  const float th = 1.0f - __fdividef(2.0f, e + 1.0f);
  return 0.5f * x * (1.0f + th);
}

// d gelu / dx for the activation-gradient tail; shares exp(-x^2/2) between the erf and the density term.
__device__ __forceinline__ float gelu_erf_grad_fast(float x) {
  const float z = fabsf(x) * 0.70710678118654752440f;
  const float t = __fdividef(1.0f, fmaf(0.3275911f, z, 1.0f));
  float poly = fmaf(1.061405429f, t, -1.453152027f);
  poly = fmaf(poly, t, 1.421413741f);
  poly = fmaf(poly, t, -0.284496736f);
  poly = fmaf(poly, t, 0.254829592f);
  const float ez = __expf(-z * z);                     // exp(-x^2 / 2)
  const float e = 1.0f - poly * t * ez;                // erf(|x| / sqrt2)
  const float cdf = 0.5f * (1.0f + copysignf(e, x));
  return fmaf(x * 0.3989422804014327f, ez, cdf);
}
__device__ __forceinline__ float gelu_tanh_grad_fast(float x) {
  const float k0 = 0.7978845608028654f, k1 = 0.044715f;
  const float u = k0 * fmaf(k1 * x, x * x, x);
  const float e = __expf(2.0f * u);
  const float th = 1.0f - __fdividef(2.0f, e + 1.0f);
  return 0.5f * (1.0f + th) + 0.5f * x * (1.0f - th * th) * k0 * fmaf(3.0f * k1 * x, x, 1.0f);
}

// The activation kind is a compile-time parameter of the chunk loops: with a runtime `act ? tanh : erf` per element the
// compiler evaluated BOTH activations and selected (the first fused epilogues spent twice the issue slots they needed).
template <bool kTanh> __device__ __forceinline__ float gelu_fast(float x) {
  if constexpr (kTanh) return gelu_tanh_fast(x);
  else return gelu_erf_fast(x);
}
template <bool kTanh> __device__ __forceinline__ float gelu_grad_fast(float x) {
  if constexpr (kTanh) return gelu_tanh_grad_fast(x);
  else return gelu_erf_grad_fast(x);
}

// Tile order inside one (batch, split) slice: bands of kBand n-blocks, n fastest inside a band, then m, then the
// next band.  Co-resident CTAs share A rows (as before), and a band's B tiles (<= 4 MB) stay in L2 while the sweep
// over m reuses them -- without this a wide-N GEMM (the stacked K/V projection, N = 57k) re-streams B from HBM for
// every row block.
constexpr int kBand = 8;
__device__ __forceinline__ void decode_tile(int r, int m_blocks, int n_blocks, int& mb, int& nb) {
  const int per_band = kBand * m_blocks;
  const int band = r / per_band;
  const int bw = min(kBand, n_blocks - band * kBand);
  const int rr = r - band * per_band;
  mb = rr / bw;
  nb = band * kBand + rr % bw;
}

__device__ __forceinline__ uint32_t pack_bf16(float a, float b) {
  __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&v);
}

// Two adjacent output columns (col, col + 1) per access; `two` = col + 1 is inside the matrix, `vec` = the pair may be
// moved as one 4- / 8-byte word (host-checked alignment of every pointer and pitch).
__device__ __forceinline__ void st_bf16_pair(__nv_bfloat16* dst, float a, float b, bool two, bool vec) {
  if (two && vec) {
    *reinterpret_cast<uint32_t*>(dst) = pack_bf16(a, b);
  } else {
    dst[0] = __float2bfloat16_rn(a);
    if (two) dst[1] = __float2bfloat16_rn(b);
  }
}
__device__ __forceinline__ void st_f32_pair(float* dst, float a, float b, bool two, bool vec) {
  if (two && vec) {
    *reinterpret_cast<float2*>(dst) = make_float2(a, b);
  } else {
    dst[0] = a;
    if (two) dst[1] = b;
  }
}
__device__ __forceinline__ void red_f32_pair(float* dst, float a, float b, bool two, bool vec) {
  if (two && vec) {
    atomicAdd(reinterpret_cast<float2*>(dst), make_float2(a, b));
  } else {
    atomicAdd(dst, a);
    if (two) atomicAdd(dst + 1, b);
  }
}
__device__ __forceinline__ float2 ld_f32_pair(const float* src, bool two, bool vec) {
  if (two && vec) return *reinterpret_cast<const float2*>(src);
  return make_float2(src[0], two ? src[1] : 0.f);
}
__device__ __forceinline__ float2 ld_bf16_pair(const __nv_bfloat16* src, bool two, bool vec) {
  if (two && vec) return __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(src));
  return make_float2(__bfloat162float(src[0]), two ? __bfloat162float(src[1]) : 0.f);
}

// The tails' arithmetic on one column pair, shared by the guarded and the interior epilogue so that both round the
// same way.  Bias, gate and residual are separate roundings (__fadd_rn / __fmul_rn): they are never contracted into an
// FMA with the acc * alpha product, however the code around them is compiled.
__device__ __forceinline__ void add_pair(float& v0, float& v1, float2 b) {
  v0 = __fadd_rn(v0, b.x);
  v1 = __fadd_rn(v1, b.y);
}
// C2 = bf16 copy of v (optional, needed by backward for d(gate)); C = v * g (if gated) + r
__device__ __forceinline__ void resid_tail(float* C, __nv_bfloat16* C2, float v0, float v1, bool gated, float2 g,
                                           float2 r, bool two, bool vec) {
  if (C2 != nullptr) st_bf16_pair(C2, v0, v1, two, vec);
  if (gated) {
    v0 = __fmul_rn(v0, g.x);
    v1 = __fmul_rn(v1, g.y);
  }
  st_f32_pair(C, __fadd_rn(v0, r.x), __fadd_rn(v1, r.y), two, vec);
}
// C = pre-activation (bf16), C2 = act(pre) (bf16); the activation is taken on the bf16-rounded pre-activation so that
// backward (which re-reads C) differentiates the same function
template <bool kTanh>
__device__ __forceinline__ void act_dual_tail(__nv_bfloat16* C, __nv_bfloat16* C2, float v0, float v1, bool two, bool vec) {
  const float x0 = bf16_round(v0), x1 = bf16_round(v1);
  st_bf16_pair(C, x0, x1, two, vec);
  st_bf16_pair(C2, gelu_fast<kTanh>(x0), gelu_fast<kTanh>(x1), two, vec);
}
// C = acc * act'(pre): the dgrad GEMM hands the pre-activation gradient on directly
template <bool kTanh>
__device__ __forceinline__ void act_grad_tail(__nv_bfloat16* C, float v0, float v1, float2 x, bool two, bool vec) {
  st_bf16_pair(C, v0 * gelu_grad_fast<kTanh>(x.x), v1 * gelu_grad_fast<kTanh>(x.y), two, vec);
}
// u1 = (a0, a1), u2 = (b0, b1) (bias included): du = bf16 u at its interleaved columns (u1 at du, u2 at du + 32),
// h = silu(u1) * u2 at the natural column
__device__ __forceinline__ void swiglu_tail(__nv_bfloat16* du, __nv_bfloat16* h, float a0, float a1, float b0, float b1) {
  a0 = bf16_round(a0); a1 = bf16_round(a1);
  b0 = bf16_round(b0); b1 = bf16_round(b1);
  st_bf16_pair(du, a0, a1, true, true);
  st_bf16_pair(du + 32, b0, b1, true, true);
  const float h0 = a0 * __fdividef(1.0f, 1.0f + __expf(-a0)) * b0;
  const float h1 = a1 * __fdividef(1.0f, 1.0f + __expf(-a1)) * b1;
  st_bf16_pair(h, h0, h1, true, true);
}
// d u1 = d h * u2 * silu'(u1) at dst, d u2 = d h * silu(u1) at dst + 32
__device__ __forceinline__ void swiglu_grad_tail(__nv_bfloat16* dst, float d0, float d1, float2 u1, float2 u2) {
  const float s0 = __fdividef(1.0f, 1.0f + __expf(-u1.x)), s1 = __fdividef(1.0f, 1.0f + __expf(-u1.y));
  st_bf16_pair(dst, d0 * u2.x * (s0 * fmaf(u1.x, 1.0f - s0, 1.0f)), d1 * u2.y * (s1 * fmaf(u1.y, 1.0f - s1, 1.0f)),
               true, true);
  st_bf16_pair(dst + 32, d0 * u1.x * s0, d1 * u1.y * s1, true, true);
}

// Epilogue of an interior tile in chunks of CH column groups j (both rows of each).  load(j, side) issues the global
// loads group j needs into `side`; emit(j, side) does its math and stores.  The loads of the next chunk go out before
// the math and stores of the current one, so their latencies overlap instead of being waited out one column pair at a
// time; the first chunk's loads go out before `mma_done` (the wait for the tile's last MMAs: the addresses do not depend
// on the accumulators).  The batching comes from the source order alone: C may alias a side input (the in-place
// residual), and every element is still read before it is written.
template <int NJ, int CH, class Side, class Load, class Emit, class Wait>
__device__ __forceinline__ void chunked_tail(Load&& load, Emit&& emit, Wait&& mma_done) {
  static_assert(NJ % CH == 0, "chunks must tile the column groups");
  Side cur[CH];
#pragma unroll
  for (int jj = 0; jj < CH; ++jj) load(jj, cur[jj]);
  mma_done();
#pragma unroll
  for (int j0 = 0; j0 < NJ; j0 += CH) {
    Side nxt[CH];
    if (j0 + CH < NJ) {
#pragma unroll
      for (int jj = 0; jj < CH; ++jj) load(j0 + CH + jj, nxt[jj]);
    }
#pragma unroll
    for (int jj = 0; jj < CH; ++jj) emit(j0 + jj, cur[jj]);
    if (j0 + CH < NJ) {
#pragma unroll
      for (int jj = 0; jj < CH; ++jj) cur[jj] = nxt[jj];
    }
  }
}

// Side inputs of one column group j (both rows), and how many groups a chunk takes.  Sized so that the 256-wide tile
// compiles without spills: its 128 accumulators are all live while the first chunk loads, two chunks are live while
// the next is in flight, and the compiler runs the unrolled math of a chunk side by side (each element's temporaries
// at once).  Larger chunks for SwiGLU' or GELU' spilled.
struct BiasSide { float2 b; static constexpr int kChunk = 8; };
struct ResidSide { float2 b, g[2], r[2]; static constexpr int kChunk = 2; };
struct SwigluSide { float2 b1, b2; static constexpr int kChunk = 2; };  // groups j % 8 >= 4 load nothing
template <bool kTanh> struct ActGradSide { __nv_bfloat162 x[2]; static constexpr int kChunk = 4; };
struct SwigluGradSide { __nv_bfloat162 u1[2], u2[2]; static constexpr int kChunk = 2; };

// Every tail except the atomic one on a tile whose 128 x BLOCK_N elements are all inside the output, with pair accesses
// allowed everywhere (p.vec2): the same arithmetic as the guarded loops of the kernel, without their per-pair bounds
// checks and scalar fallbacks.  Thread rows r0, r0 + 8 (i), column pairs cb + 8 j (+0, +1); every access is a per-row
// base pointer plus a constant offset of j.
template <int BLOCK_N, class Wait>
__device__ __forceinline__ void interior_epilogue(const GemmDev& p, float (&acc)[BLOCK_N / 2], int bz, int r0, int cb,
                                                  Wait&& mma_done) {
  constexpr int NJ = BLOCK_N / 8;
  const float alpha = p.alpha;
  long long crow[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) crow[i] = 1LL * bz * p.strideC + 1LL * (r0 + 8 * i) * p.ldc;
  auto row_ptr = [&](auto* base, int i) { return base + crow[i] + cb; };
  const float* bias = p.bias != nullptr ? p.bias + 1LL * bz * p.strideBias + cb : nullptr;
  auto v = [&](int j, int i, int e) { return acc[4 * j + 2 * i + e] * alpha; };
  auto ld_bias = [&](int j, BiasSide& s) {
    if (bias != nullptr) s.b = *reinterpret_cast<const float2*>(bias + 8 * j);
  };
  auto with_bias = [&](int j, int i, const BiasSide& s, float& v0, float& v1) {
    v0 = v(j, i, 0);
    v1 = v(j, i, 1);
    if (bias != nullptr) add_pair(v0, v1, s.b);
  };
  auto act_kind = [&](auto&& body) {
    if (p.act) body(std::true_type{});
    else body(std::false_type{});
  };

  switch (p.epi) {
    case EPI_STORE_BF16: {
      __nv_bfloat16* c[2] = {row_ptr(reinterpret_cast<__nv_bfloat16*>(p.C), 0), row_ptr(reinterpret_cast<__nv_bfloat16*>(p.C), 1)};
      chunked_tail<NJ, BiasSide::kChunk, BiasSide>(ld_bias, [&](int j, const BiasSide& s) {
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          float v0, v1;
          with_bias(j, i, s, v0, v1);
          st_bf16_pair(c[i] + 8 * j, v0, v1, true, true);
        }
      }, mma_done);
      break;
    }
    case EPI_STORE_F32: {
      float* c[2] = {row_ptr(reinterpret_cast<float*>(p.C), 0), row_ptr(reinterpret_cast<float*>(p.C), 1)};
      chunked_tail<NJ, BiasSide::kChunk, BiasSide>(ld_bias, [&](int j, const BiasSide& s) {
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          float v0, v1;
          with_bias(j, i, s, v0, v1);
          st_f32_pair(c[i] + 8 * j, v0, v1, true, true);
        }
      }, mma_done);
      break;
    }
    case EPI_RESID_F32: {
      float* c[2] = {row_ptr(reinterpret_cast<float*>(p.C), 0), row_ptr(reinterpret_cast<float*>(p.C), 1)};
      __nv_bfloat16* c2[2] = {nullptr, nullptr};
      const float* res[2];
      const float* gate[2] = {nullptr, nullptr};
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int row = r0 + 8 * i;
        if (p.C2 != nullptr) c2[i] = row_ptr(reinterpret_cast<__nv_bfloat16*>(p.C2), i);
        res[i] = p.res + 1LL * bz * p.strideC + 1LL * (p.res_mod > 0 ? row % p.res_mod : row) * p.ldc + cb;
        if (p.gate != nullptr) gate[i] = p.gate + 1LL * (row / p.rows_per_gate) * p.ldgate + cb;
      }
      // the gate's presence picks the instantiation: a load under a runtime condition would keep a register pair per
      // group alive on both paths
      auto gated_kind = [&](auto&& body) {
        if (p.gate != nullptr) body(std::true_type{});
        else body(std::false_type{});
      };
      gated_kind([&](auto gated_tag) {
        constexpr bool kGated = decltype(gated_tag)::value;
        chunked_tail<NJ, ResidSide::kChunk, ResidSide>(
            [&](int j, ResidSide& s) {
              if (bias != nullptr) s.b = *reinterpret_cast<const float2*>(bias + 8 * j);
#pragma unroll
              for (int i = 0; i < 2; ++i) {
                if constexpr (kGated) s.g[i] = *reinterpret_cast<const float2*>(gate[i] + 8 * j);
                s.r[i] = *reinterpret_cast<const float2*>(res[i] + 8 * j);
              }
            },
            [&](int j, const ResidSide& s) {
#pragma unroll
              for (int i = 0; i < 2; ++i) {
                float v0 = v(j, i, 0), v1 = v(j, i, 1);
                if (bias != nullptr) add_pair(v0, v1, s.b);
                resid_tail(c[i] + 8 * j, c2[i] != nullptr ? c2[i] + 8 * j : nullptr, v0, v1, kGated, s.g[i], s.r[i], true,
                           true);
              }
            },
            mma_done);
      });
      break;
    }
    case EPI_ACT_DUAL: {
      __nv_bfloat16* c[2] = {row_ptr(reinterpret_cast<__nv_bfloat16*>(p.C), 0), row_ptr(reinterpret_cast<__nv_bfloat16*>(p.C), 1)};
      __nv_bfloat16* c2[2] = {row_ptr(reinterpret_cast<__nv_bfloat16*>(p.C2), 0), row_ptr(reinterpret_cast<__nv_bfloat16*>(p.C2), 1)};
      act_kind([&](auto tanh_tag) {
        constexpr bool kTanh = decltype(tanh_tag)::value;
        chunked_tail<NJ, BiasSide::kChunk, BiasSide>(ld_bias, [&](int j, const BiasSide& s) {
#pragma unroll
          for (int i = 0; i < 2; ++i) {
            float v0, v1;
            with_bias(j, i, s, v0, v1);
            act_dual_tail<kTanh>(c[i] + 8 * j, c2[i] + 8 * j, v0, v1, true, true);
          }
        }, mma_done);
      });
      break;
    }
    case EPI_ACT_GRAD: {
      __nv_bfloat16* c[2] = {row_ptr(reinterpret_cast<__nv_bfloat16*>(p.C), 0), row_ptr(reinterpret_cast<__nv_bfloat16*>(p.C), 1)};
      const __nv_bfloat16* x[2] = {row_ptr(reinterpret_cast<const __nv_bfloat16*>(p.aux), 0),
                                   row_ptr(reinterpret_cast<const __nv_bfloat16*>(p.aux), 1)};
      act_kind([&](auto tanh_tag) {
        constexpr bool kTanh = decltype(tanh_tag)::value;
        chunked_tail<NJ, ActGradSide<kTanh>::kChunk, ActGradSide<kTanh>>(
            [&](int j, ActGradSide<kTanh>& s) {
#pragma unroll
              for (int i = 0; i < 2; ++i) s.x[i] = *reinterpret_cast<const __nv_bfloat162*>(x[i] + 8 * j);
            },
            [&](int j, const ActGradSide<kTanh>& s) {
#pragma unroll
              for (int i = 0; i < 2; ++i)
                act_grad_tail<kTanh>(c[i] + 8 * j, v(j, i, 0), v(j, i, 1), __bfloat1622float2(s.x[i]), true, true);
            },
            mma_done);
      });
      break;
    }
    case EPI_SWIGLU: {
      // groups j and j + 4 of every 8 hold u1 and u2 of the same columns (see the guarded loop); cb % 64 < 8, so group j
      // (j % 8 < 4) is column cb + 8 j of u, natural column cb + 8 j - 32 (j / 8) of h and of the bias halves
      __nv_bfloat16* c[2] = {row_ptr(reinterpret_cast<__nv_bfloat16*>(p.C), 0), row_ptr(reinterpret_cast<__nv_bfloat16*>(p.C), 1)};
      __nv_bfloat16* h[2];
#pragma unroll
      for (int i = 0; i < 2; ++i)
        h[i] = reinterpret_cast<__nv_bfloat16*>(p.C2) + 1LL * bz * p.strideC2 + 1LL * (r0 + 8 * i) * p.ldc2 +
               (cb >> 6) * 32 + (cb & 63);
      const float* b1 = p.bias != nullptr ? p.bias + 1LL * bz * p.strideBias + (cb >> 6) * 32 + (cb & 63) : nullptr;
      chunked_tail<NJ, SwigluSide::kChunk, SwigluSide>(
          [&](int j, SwigluSide& s) {
            if ((j & 7) >= 4 || b1 == nullptr) return;
            s.b1 = *reinterpret_cast<const float2*>(b1 + 8 * j - 32 * (j >> 3));
            s.b2 = *reinterpret_cast<const float2*>(b1 + 8 * j - 32 * (j >> 3) + (p.N >> 1));
          },
          [&](int j, const SwigluSide& s) {
            if ((j & 7) >= 4) return;
#pragma unroll
            for (int i = 0; i < 2; ++i) {
              float a0 = v(j, i, 0), a1 = v(j, i, 1);
              float bb0 = v(j + 4, i, 0), bb1 = v(j + 4, i, 1);
              if (b1 != nullptr) {
                add_pair(a0, a1, s.b1);
                add_pair(bb0, bb1, s.b2);
              }
              swiglu_tail(c[i] + 8 * j, h[i] + 8 * j - 32 * (j >> 3), a0, a1, bb0, bb1);
            }
          },
          mma_done);
      break;
    }
    case EPI_SWIGLU_GRAD: {
      // dh column n sits at 64 (n / 32) + n % 32 of u and du; cb % 32 < 8, so group j is 64 (j / 4) + 8 (j % 4) further
      __nv_bfloat16* c[2];
      const __nv_bfloat16* u[2];
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const long long o = crow[i] + 64 * (cb >> 5) + (cb & 31);
        c[i] = reinterpret_cast<__nv_bfloat16*>(p.C) + o;
        u[i] = reinterpret_cast<const __nv_bfloat16*>(p.aux) + o;
      }
      auto off = [](int j) { return 64 * (j >> 2) + 8 * (j & 3); };
      chunked_tail<NJ, SwigluGradSide::kChunk, SwigluGradSide>(
          [&](int j, SwigluGradSide& s) {
#pragma unroll
            for (int i = 0; i < 2; ++i) {
              s.u1[i] = *reinterpret_cast<const __nv_bfloat162*>(u[i] + off(j));
              s.u2[i] = *reinterpret_cast<const __nv_bfloat162*>(u[i] + off(j) + 32);
            }
          },
          [&](int j, const SwigluGradSide& s) {
#pragma unroll
            for (int i = 0; i < 2; ++i)
              swiglu_grad_tail(c[i] + off(j), v(j, i, 0), v(j, i, 1), __bfloat1622float2(s.u1[i]),
                               __bfloat1622float2(s.u2[i]));
          },
          mma_done);
      break;
    }
    default:
      mma_done();
      break;
  }
}

template <int BLOCK_N, bool kMN>
__device__ __forceinline__ void wgmma_k16(float (&acc)[BLOCK_N / 2], uint64_t da, uint64_t db, uint32_t accumulate) {
  if constexpr (BLOCK_N == 256) wgmma_m64n256k16<kMN ? 1 : 0, kMN ? 1 : 0>(acc, da, db, accumulate);
  else wgmma_m64n128k16<kMN ? 1 : 0, kMN ? 1 : 0>(acc, da, db, accumulate);
}

template <int BLOCK_N, bool kMN>
__global__ void __launch_bounds__(kThreads, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GemmDev p) {
  using Cfg = GemmCfg<BLOCK_N>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + Cfg::kStages * Cfg::kStageBytes);
  uint64_t* empty_bar = full_bar + Cfg::kStages;

  const int wg = threadIdx.x >> 7;
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int i = 0; i < Cfg::kStages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 8);  // one arrive per MMA warp
    }
    mbar_fence_init();
  }
  __syncthreads();

  const int m_blocks = (p.M + kBlockM - 1) / kBlockM;
  const int n_blocks = (p.N + BLOCK_N - 1) / BLOCK_N;
  const int kb_total = (p.K + kBlockK - 1) / kBlockK;
  const int kb_per_split = (kb_total + p.splits - 1) / p.splits;
  const long long mn = 1LL * n_blocks * m_blocks;
  const long long tiles = 1LL * p.batch * p.splits * mn;

  if (wg == 0) {
    // ================================ TMA producer ================================
    warpgroup_reg_dealloc<40>();
    if (threadIdx.x == 0) {
      uint32_t it = 0;
      for (long long tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
        long long t = tile;
        int mb, nb;
        decode_tile(static_cast<int>(t % mn), m_blocks, n_blocks, mb, nb);
        t /= mn;
        const int sp = t % p.splits; t /= p.splits;
        const int bz = static_cast<int>(t);
        const int kb0 = sp * kb_per_split;
        const int kb1 = min(kb_total, kb0 + kb_per_split);
        for (int kb = kb0; kb < kb1; ++kb, ++it) {
          const int s = it % Cfg::kStages;
          const uint32_t ph = (it / Cfg::kStages) & 1;
          mbar_wait(&empty_bar[s], ph ^ 1);
          uint8_t* sa = smem + s * Cfg::kStageBytes;
          uint8_t* sb = sa + Cfg::kStageBytesA;
          mbar_expect_tx(&full_bar[s], Cfg::kStageBytes);
          if constexpr (!kMN) {
            tma_load_3d(&tmA, &full_bar[s], sa, kb * kBlockK, mb * kBlockM, bz);
            tma_load_3d(&tmB, &full_bar[s], sb, kb * kBlockK, nb * BLOCK_N, bz);
          } else {
            // boxes of 64 (MN, contiguous) x 64 (reduction rows); one box per 64 MN elements
#pragma unroll
            for (int j = 0; j < kBlockM / 64; ++j)
              tma_load_3d(&tmA, &full_bar[s], sa + j * (kBlockK * 128), mb * kBlockM + j * 64, kb * kBlockK, bz);
#pragma unroll
            for (int j = 0; j < BLOCK_N / 64; ++j)
              tma_load_3d(&tmB, &full_bar[s], sb + j * (kBlockK * 128), nb * BLOCK_N + j * 64, kb * kBlockK, bz);
          }
        }
      }
    }
    return;
  }

  // ================================ MMA + epilogue (warpgroups 1, 2: rows 0-63 / 64-127 of the tile) ================
  warpgroup_reg_alloc<232>();
  const int half = wg - 1;
  const int wq = warp & 3;  // warp inside the warpgroup: accumulator rows 16 wq .. 16 wq + 15
  // K-major: 8-row groups 1024 B apart (SBO), LBO unused.  MN-major: 64-element MN atoms one whole box apart (LBO = 64
  // rows * 128 B), 8-deep reduction groups 1024 B apart (SBO).  Either way the warpgroup's 64 rows start 8 KB in.
  constexpr uint32_t lbo = kMN ? (kBlockK * 128) : 16;
  constexpr uint32_t sbo = 1024;
  constexpr uint32_t kstep = (kMN ? (kWgK * 128) : (kWgK * 2)) >> 4;  // descriptor advance per 16-deep MMA
  float acc[BLOCK_N / 2];
#pragma unroll
  for (int i = 0; i < BLOCK_N / 2; ++i) acc[i] = 0.f;
  const bool vec = p.vec2 != 0;
  const float alpha = p.alpha;

  uint32_t it = 0;
  for (long long tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    long long t = tile;
    int mb, nb;
    decode_tile(static_cast<int>(t % mn), m_blocks, n_blocks, mb, nb);
    t /= mn;
    const int sp = t % p.splits; t /= p.splits;
    const int bz = static_cast<int>(t);
    const int kb0 = sp * kb_per_split;
    const int kb1 = min(kb_total, kb0 + kb_per_split);
    const bool has_k = kb0 < kb_total;  // empty split (possible when splits does not divide)

    for (int kb = kb0; kb < kb1; ++kb, ++it) {
      const int s = it % Cfg::kStages;
      mbar_wait(&full_bar[s], (it / Cfg::kStages) & 1);
      const uint32_t sa = smem_u32(smem + s * Cfg::kStageBytes) + half * (64 * 128);
      const uint32_t sb = smem_u32(smem + s * Cfg::kStageBytes + Cfg::kStageBytesA);
      const uint64_t da0 = wgmma_smem_desc(sa, lbo, sbo);
      const uint64_t db0 = wgmma_smem_desc(sb, lbo, sbo);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < kBlockK / kWgK; ++k)
        wgmma_k16<BLOCK_N, kMN>(acc, da0 + k * kstep, db0 + k * kstep, (kb > kb0 || k > 0) ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<1>();  // the previous k-block's MMAs have retired: its stage may be refilled
      if (kb > kb0) {
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[(it - 1) % Cfg::kStages]);
      }
    }
    auto mma_done = [&]() {
      wgmma_wait<0>();
      wgmma_fence_operands(acc);
      if (kb1 > kb0) {
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[(it - 1) % Cfg::kStages]);
      }
    };

    // ---------------------------------------------------------------- epilogue, straight from the registers
    // thread owns rows r0, r0 + 8 and column pairs cb + 8 j (+0, +1), j < BLOCK_N / 8
    const int r0 = mb * kBlockM + half * 64 + wq * 16 + (lane >> 2);
    const int cb = nb * BLOCK_N + 2 * (lane & 3);
    if (vec && p.epi != EPI_ATOMIC_F32 && (mb + 1) * kBlockM <= p.M && (nb + 1) * BLOCK_N <= p.N) {
      interior_epilogue<BLOCK_N>(p, acc, bz, r0, cb, mma_done);
      continue;
    }
    // edge tiles, unaligned pitches and the atomic tail: every pair checks its bounds and falls back to scalar accesses
    mma_done();
    // f(row, crow, i, j, col, v0, v1, two) for every in-bounds pair; crow = offset of the output row
    auto for_each_pair = [&](auto&& f) {
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int row = r0 + 8 * i;
        if (row >= p.M) continue;
        int row_out = row;
        // weight gradient of a 32-row-interleaved stack (the fused-SwiGLU w1 | w2 layout): tile row -> parameter row
        if (p.row_interleave > 0) {
          const int blk = row >> 6, in = row & 63;
          row_out = (in < 32 ? 0 : p.row_interleave) + 32 * blk + (in & 31);
        }
        const long long crow = 1LL * bz * p.strideC + 1LL * row_out * p.ldc;
#pragma unroll
        for (int j = 0; j < BLOCK_N / 8; ++j) {
          const int col = cb + 8 * j;
          if (col < p.N) f(row, crow, i, j, col, acc[4 * j + 2 * i] * alpha, acc[4 * j + 2 * i + 1] * alpha, col + 1 < p.N);
        }
      }
    };
    auto add_bias = [&](int col, float& v0, float& v1, bool two) {
      if (p.bias != nullptr) add_pair(v0, v1, ld_f32_pair(p.bias + 1LL * bz * p.strideBias + col, two, vec));
    };

    switch (p.epi) {
      case EPI_STORE_BF16:
        for_each_pair([&](int, long long crow, int, int, int col, float v0, float v1, bool two) {
          add_bias(col, v0, v1, two);
          st_bf16_pair(reinterpret_cast<__nv_bfloat16*>(p.C) + crow + col, v0, v1, two, vec);
        });
        break;
      case EPI_STORE_F32:
        for_each_pair([&](int, long long crow, int, int, int col, float v0, float v1, bool two) {
          add_bias(col, v0, v1, two);
          st_f32_pair(reinterpret_cast<float*>(p.C) + crow + col, v0, v1, two, vec);
        });
        break;
      case EPI_RESID_F32:
        for_each_pair([&](int row, long long crow, int, int, int col, float v0, float v1, bool two) {
          add_bias(col, v0, v1, two);
          float2 g = make_float2(0.f, 0.f);
          if (p.gate != nullptr) g = ld_f32_pair(p.gate + 1LL * (row / p.rows_per_gate) * p.ldgate + col, two, vec);
          const long long rrow = 1LL * bz * p.strideC + 1LL * (p.res_mod > 0 ? row % p.res_mod : row) * p.ldc;
          const float2 r = ld_f32_pair(p.res + rrow + col, two, vec);
          resid_tail(reinterpret_cast<float*>(p.C) + crow + col,
                     p.C2 != nullptr ? reinterpret_cast<__nv_bfloat16*>(p.C2) + crow + col : nullptr, v0, v1,
                     p.gate != nullptr, g, r, two, vec);
        });
        break;
      case EPI_ATOMIC_F32:
        if (p.split_ws != nullptr) {
          // deterministic split-K: this split's partial tile goes to the workspace [split][batch][M][N] with plain stores
          // (zeros for an empty split); splitk_reduce_kernel adds the splits up in a fixed order
          for_each_pair([&](int row, long long, int, int, int col, float v0, float v1, bool two) {
            float* dst = p.split_ws + ((1LL * sp * p.batch + bz) * p.M + row) * p.N + col;
            st_f32_pair(dst, has_k ? v0 : 0.f, has_k ? v1 : 0.f, two, vec);
          });
        } else if (has_k) {
          for_each_pair([&](int, long long crow, int, int, int col, float v0, float v1, bool two) {
            add_bias(col, v0, v1, two);
            red_f32_pair(reinterpret_cast<float*>(p.C) + crow + col, v0, v1, two, vec);
          });
        }
        break;
      case EPI_ACT_DUAL: {
        auto dual = [&](auto tanh_tag) {
          constexpr bool kTanh = decltype(tanh_tag)::value;
          for_each_pair([&](int, long long crow, int, int, int col, float v0, float v1, bool two) {
            add_bias(col, v0, v1, two);
            act_dual_tail<kTanh>(reinterpret_cast<__nv_bfloat16*>(p.C) + crow + col,
                                 reinterpret_cast<__nv_bfloat16*>(p.C2) + crow + col, v0, v1, two, vec);
          });
        };
        if (p.act) dual(std::true_type{});
        else dual(std::false_type{});
        break;
      }
      case EPI_ACT_GRAD: {
        auto grad = [&](auto tanh_tag) {
          constexpr bool kTanh = decltype(tanh_tag)::value;
          for_each_pair([&](int, long long crow, int, int, int col, float v0, float v1, bool two) {
            const float2 x = ld_bf16_pair(reinterpret_cast<const __nv_bfloat16*>(p.aux) + crow + col, two, vec);
            act_grad_tail<kTanh>(reinterpret_cast<__nv_bfloat16*>(p.C) + crow + col, v0, v1, x, two, vec);
          });
        };
        if (p.act) grad(std::true_type{});
        else grad(std::false_type{});
        break;
      }
      case EPI_SWIGLU:
        // SwiGLU (dit.py:88-89) in the epilogue of the stacked w1 | w2 GEMM.  The weight stack is interleaved in blocks of
        // 32 rows (w1 block j, w2 block j, ...), so column c < 32 of every 64-column group holds u1 and column c + 32 the
        // matching u2 -- register pairs j and j + 4 of the same thread: C = u (bf16, the interleaved layout backward reads
        // again), C2 = silu(u1) * u2 (bf16, natural layout).  N % 64 == 0 and 32-byte aligned outputs (host-checked).
        // The optional bias is the natural-order [b1 | b2] fp32 vector: u1 column col (col % 64 < 32) takes
        // b1[32 (col / 64) + col % 64], its u2 partner b2 at the same index; u = acc + b is what C keeps for backward.
        for_each_pair([&](int row, long long crow, int i, int j, int col, float, float, bool) {
          if ((j & 7) >= 4) return;
          float a0 = acc[4 * j + 2 * i] * alpha, a1 = acc[4 * j + 2 * i + 1] * alpha;
          float b0 = acc[4 * (j + 4) + 2 * i] * alpha, b1 = acc[4 * (j + 4) + 2 * i + 1] * alpha;
          if (p.bias != nullptr) {
            const float* bb = p.bias + 1LL * bz * p.strideBias + 32 * (col >> 6) + (col & 63);
            add_pair(a0, a1, ld_f32_pair(bb, true, vec));
            add_pair(b0, b1, ld_f32_pair(bb + (p.N >> 1), true, vec));
          }
          swiglu_tail(reinterpret_cast<__nv_bfloat16*>(p.C) + crow + col,
                      reinterpret_cast<__nv_bfloat16*>(p.C2) + 1LL * bz * p.strideC2 + 1LL * row * p.ldc2 +
                          (col >> 6) * 32 + (col & 63),
                      a0, a1, b0, b1);
        });
        break;
      case EPI_SWIGLU_GRAD:
        // backward of the above inside the w3 dgrad GEMM: acc = d h (never stored); with the saved u1 | u2 of column n (aux,
        // interleaved layout: u1 at 64 (n / 32) + n % 32, u2 32 further) the pair leaves as d u1 = d h * u2 * silu'(u1),
        // d u2 = d h * silu(u1), at the same interleaved positions of C.
        for_each_pair([&](int, long long crow, int, int, int col, float d0, float d1, bool) {
          const long long off = crow + 64 * (col >> 5) + (col & 31);
          const float2 u1 = ld_bf16_pair(reinterpret_cast<const __nv_bfloat16*>(p.aux) + off, true, true);
          const float2 u2 = ld_bf16_pair(reinterpret_cast<const __nv_bfloat16*>(p.aux) + off + 32, true, true);
          swiglu_grad_tail(reinterpret_cast<__nv_bfloat16*>(p.C) + off, d0, d1, u1, u2);
        });
        break;
      default:
        break;
    }
  }
}

// C[b][rowmap(m)][n] += sum_sp ws[sp][b][m][n], sp = 0, 1, ... (deterministic split-K, second pass)
__global__ void __launch_bounds__(256)
splitk_reduce_kernel(const float* __restrict__ ws, float* __restrict__ C, int splits, int batch, int M, int N,
                     long long ldc, long long strideC, int row_interleave) {
  const long long total = 1LL * batch * M * N;
  for (long long i = 1LL * blockIdx.x * blockDim.x + threadIdx.x; i < total; i += 1LL * gridDim.x * blockDim.x) {
    const int n = static_cast<int>(i % N);
    const long long bm = i / N;
    const int m = static_cast<int>(bm % M);
    const int b = static_cast<int>(bm / M);
    float s = 0.f;
    for (int sp = 0; sp < splits; ++sp) s += ws[1LL * sp * total + i];
    int row = m;
    if (row_interleave > 0) {
      const int blk = m >> 6, in = m & 63;
      row = (in < 32 ? 0 : row_interleave) + 32 * blk + (in & 31);
    }
    C[1LL * b * strideC + 1LL * row * ldc + n] += s;
  }
}

// ---------------------------------------------------------------------------------------------- host

// bf16 tensor viewed as [batch][rows][cols] (cols contiguous), box = [1][box_rows][64], 128B swizzle.
static int make_map(CUtensorMap* map, const void* ptr, long long cols, long long rows, long long batch,
                    long long ld, long long batch_stride, int box_rows) {
  if ((reinterpret_cast<uintptr_t>(ptr) & 15) != 0 || (ld % 8) != 0 || (batch > 1 && (batch_stride % 8) != 0))
    return md_set_error(MD_ERR_INVALID, "gemm operand must be 16-byte aligned with ld %% 8 == 0");
  const TmapKey key = make_tmap_key(ptr, cols, rows, batch, ld, batch > 1 ? batch_stride : rows * ld, 64, box_rows,
                                    CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
  CUresult r = cached_tensor_map(map, key);
  if (r != CUDA_SUCCESS) {
    char msg[160];
    snprintf(msg, sizeof(msg), "cuTensorMapEncodeTiled failed (%d) cols=%lld rows=%lld ld=%lld", (int)r, cols,
             rows, ld);
    return md_set_error(MD_ERR_CUDA, msg);
  }
  return 0;
}

template <int BLOCK_N, bool kMN>
static int launch(const md_gemm_args* a, const GemmDev& dev, int sm_count, cudaStream_t stream) {
  using Cfg = GemmCfg<BLOCK_N>;
  CUtensorMap tmA, tmB;
  int rc;
  if (!kMN) {
    rc = make_map(&tmA, a->A, a->K, a->M, a->batch, a->lda, a->strideA, kBlockM);
    if (rc) return rc;
    rc = make_map(&tmB, a->B, a->K, a->N, a->batch, a->ldb, a->strideB, BLOCK_N);
    if (rc) return rc;
  } else {
    rc = make_map(&tmA, a->A, a->M, a->K, a->batch, a->lda, a->strideA, kBlockK);
    if (rc) return rc;
    rc = make_map(&tmB, a->B, a->N, a->K, a->batch, a->ldb, a->strideB, kBlockK);
    if (rc) return rc;
  }
  auto kern = gemm_wgmma_kernel<BLOCK_N, kMN>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes);
    if (e != cudaSuccess) return md_set_error(MD_ERR_CUDA, cudaGetErrorString(e));
    attr_set = true;
  }
  const long long m_blocks = (a->M + kBlockM - 1) / kBlockM;
  const long long n_blocks = (a->N + BLOCK_N - 1) / BLOCK_N;
  const long long tiles = a->batch * dev.splits * m_blocks * n_blocks;
  const int grid = static_cast<int>(tiles < sm_count ? tiles : sm_count);
  kern<<<grid, kThreads, Cfg::kSmemBytes, stream>>>(tmA, tmB, dev);
  return check_launch("md_gemm_bf16");
}

}  // namespace md

extern "C" int md_gemm_bf16(const md_gemm_args* a, void* stream_) {
  using namespace md;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (a == nullptr || a->A == nullptr || a->B == nullptr || a->C == nullptr)
    return md_set_error(MD_ERR_INVALID, "md_gemm_bf16: null operand");
  if (a->M <= 0 || a->N <= 0 || a->K <= 0 || a->batch <= 0) return 0;  // empty problem: nothing to do
  if (a->epilogue < 0 || a->epilogue >= EPI_COUNT) return md_set_error(MD_ERR_INVALID, "md_gemm_bf16: bad epilogue");
  if (a->epilogue == EPI_RESID_F32 && a->res == nullptr)
    return md_set_error(MD_ERR_INVALID, "md_gemm_bf16: residual epilogue needs res");
  if (a->epilogue == EPI_ACT_DUAL && a->C2 == nullptr)
    return md_set_error(MD_ERR_INVALID, "md_gemm_bf16: activation epilogue needs C2");
  if (a->epilogue == EPI_ACT_GRAD && a->aux == nullptr)
    return md_set_error(MD_ERR_INVALID, "md_gemm_bf16: activation-gradient epilogue needs aux (the saved pre-activation)");
  if (a->epilogue == EPI_ACT_GRAD && a->bias != nullptr)
    return md_set_error(MD_ERR_INVALID, "md_gemm_bf16: the activation-gradient epilogue takes no bias");
  // every split would add it once (and the deterministic partials not at all): C += alpha*acc has no bias term
  if (a->epilogue == EPI_ATOMIC_F32 && a->bias != nullptr)
    return md_set_error(MD_ERR_INVALID, "md_gemm_bf16: the accumulate epilogue takes no bias");
  if (a->epilogue == EPI_SWIGLU || a->epilogue == EPI_SWIGLU_GRAD) {
    const bool fwd = a->epilogue == EPI_SWIGLU;
    const void* second = fwd ? a->C2 : a->aux;
    const int64_t ld2 = fwd ? (a->ldc2 > 0 ? a->ldc2 : a->N / 2) : a->ldc;
    if (second == nullptr || (!fwd && a->bias != nullptr) || a->layout != MD_GEMM_NT || a->splits > 1)
      return md_set_error(MD_ERR_INVALID,
                          "md_gemm_bf16: SwiGLU epilogues need C2 (forward) / aux (backward), NT layout, no bias on the backward");
    if (a->N % (fwd ? 64 : 32) != 0 || (a->ldc % 16) != 0 || (ld2 % 16) != 0 ||
        ((reinterpret_cast<uintptr_t>(a->C) | reinterpret_cast<uintptr_t>(second)) & 31) != 0 ||
        (a->batch > 1 && ((a->strideC % 16) != 0 || (fwd && (a->strideC2 % 16) != 0))))
      return md_set_error(MD_ERR_UNSUPPORTED,
                          "md_gemm_bf16: SwiGLU epilogues need 32-byte aligned outputs, pitches % 16 == 0 and whole 32-column blocks");
  }
  if (a->row_interleave != 0 && (a->epilogue != EPI_ATOMIC_F32 || a->row_interleave % 32 != 0 || a->M != 2 * a->row_interleave))
    return md_set_error(MD_ERR_INVALID, "md_gemm_bf16: row_interleave = f needs the atomic epilogue, f % 32 == 0 and M == 2 f");
  if (a->gate != nullptr && a->rows_per_gate <= 0)
    return md_set_error(MD_ERR_INVALID, "md_gemm_bf16: gate needs rows_per_gate > 0");
  int splits = a->splits > 0 ? a->splits : 1;
  if (splits > 1 && a->epilogue != EPI_ATOMIC_F32)
    return md_set_error(MD_ERR_INVALID, "md_gemm_bf16: split-K needs the atomic epilogue");

  int dev_id = 0, sm_count = 0;
  cudaError_t e = cudaGetDevice(&dev_id);
  if (e != cudaSuccess) return md_set_error(MD_ERR_CUDA, cudaGetErrorString(e));
  static int cached_sm[64] = {0};
  if (dev_id < 64 && cached_sm[dev_id] > 0) sm_count = cached_sm[dev_id];
  else {
    int major = 0;
    cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, dev_id);
    cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev_id);
    if (major != 9) return md_set_error(MD_ERR_UNSUPPORTED, "md_gemm_bf16: requires an sm_90a device (H100)");
    if (dev_id < 64) cached_sm[dev_id] = sm_count;
  }

  if (a->sm_limit > 0 && a->sm_limit < sm_count) sm_count = a->sm_limit;

  GemmDev dev;
  dev.C = a->C; dev.C2 = a->C2;
  dev.bias = reinterpret_cast<const float*>(a->bias);
  dev.res = reinterpret_cast<const float*>(a->res);
  dev.gate = reinterpret_cast<const float*>(a->gate);
  dev.aux = a->aux;
  dev.ldc2 = a->ldc2 > 0 ? a->ldc2 : a->N / 2;
  dev.strideC2 = a->strideC2;
  dev.row_interleave = static_cast<int>(a->row_interleave);
  dev.split_ws = nullptr;
  dev.M = static_cast<int>(a->M); dev.N = static_cast<int>(a->N); dev.K = static_cast<int>(a->K);
  dev.batch = static_cast<int>(a->batch); dev.splits = splits;
  dev.ldc = a->ldc; dev.strideC = a->strideC; dev.strideBias = a->strideBias;
  dev.ldgate = a->ldgate; dev.rows_per_gate = static_cast<int>(a->rows_per_gate > 0 ? a->rows_per_gate : 1);
  dev.epi = a->epilogue;
  dev.res_mod = static_cast<int>(a->res_mod);
  dev.act = a->act;
  dev.alpha = a->alpha == 0.0f ? 1.0f : a->alpha;
  {  // pair accesses (4 / 8 bytes at even columns) need 8-byte aligned bases and even pitches everywhere
    const uintptr_t ptrs = reinterpret_cast<uintptr_t>(a->C) | reinterpret_cast<uintptr_t>(a->C2) |
                           reinterpret_cast<uintptr_t>(a->bias) | reinterpret_cast<uintptr_t>(a->res) |
                           reinterpret_cast<uintptr_t>(a->gate) | reinterpret_cast<uintptr_t>(a->aux);
    const long long pitches = a->N | a->ldc | a->strideC | dev.ldc2 | a->strideC2 | a->strideBias | a->ldgate;
    dev.vec2 = ((ptrs & 7) == 0 && (pitches & 1) == 0) ? 1 : 0;
  }

  const bool mn = a->layout == MD_GEMM_TN;
  const long long m_blocks = (a->M + kBlockM - 1) / kBlockM;
  const long long kb_total = (a->K + kBlockK - 1) / kBlockK;
  auto tiles_for = [&](int bn) { return a->batch * m_blocks * ((a->N + bn - 1) / bn); };
  // Tile-N: 256 halves the shared-memory traffic of the A operand per MMA, so prefer it whenever the padding waste is
  // small (<= 20 % padded columns: N = 640 / 896, the 0.625 / 0.875 attention widths of MicroDiT_XL_2, still qualify) and
  // there is enough work to spread over the SMs.
  const long long n256 = (a->N + 255) / 256 * 256;
  bool use256 = (a->N >= 256) && (n256 - a->N) * 5 <= a->N;
  if (a->splits == 0 && a->epilogue == EPI_ATOMIC_F32) {
    // auto split of the reduction: minimise  waves * (k-blocks per split + fixed per-tile cost)
    const long long t = tiles_for(use256 ? 256 : 128);
    const long long smax = kb_total / 8 > 0 ? (kb_total / 8 < 64 ? kb_total / 8 : 64) : 1;
    double best = 1e30;
    for (long long sp = 1; sp <= smax; ++sp) {
      const long long units = t * sp;
      const long long waves = (units + sm_count - 1) / sm_count;
      const double cost = static_cast<double>(waves) * (static_cast<double>((kb_total + sp - 1) / sp) + 10.0);
      if (cost < best - 1e-9) { best = cost; splits = static_cast<int>(sp); }
    }
    dev.splits = splits;
  } else if (use256 && tiles_for(256) * splits < sm_count && tiles_for(128) * splits > tiles_for(256) * splits) {
    use256 = false;  // too few 256-wide tiles to occupy the machine: smaller tiles win
  }
  const bool math_tail = a->epilogue == EPI_SWIGLU || a->epilogue == EPI_SWIGLU_GRAD || a->epilogue == EPI_ACT_DUAL ||
                         a->epilogue == EPI_ACT_GRAD;
  if (math_tail && mn) return md_set_error(MD_ERR_UNSUPPORTED, "md_gemm_bf16: the activation / SwiGLU epilogues need the NT layout");
  // deterministic mode: a split reduction goes through per-split partial tiles in the workspace and a fixed-order second
  // pass; if the workspace cannot hold them the reduction is not split (one writer per element: deterministic, slower)
  if (det_enabled() && a->epilogue == EPI_ATOMIC_F32 && dev.splits > 1) {
    dev.split_ws = det_workspace(sizeof(float) * static_cast<size_t>(dev.splits) * a->batch * a->M * a->N);
    if (dev.split_ws == nullptr) dev.splits = 1;
  }
  auto run = [&]() -> int {
    if (mn) return use256 ? launch<256, true>(a, dev, sm_count, stream) : launch<128, true>(a, dev, sm_count, stream);
    return use256 ? launch<256, false>(a, dev, sm_count, stream) : launch<128, false>(a, dev, sm_count, stream);
  };
  if (int rc = run()) return rc;
  if (dev.split_ws != nullptr) {
    const long long total = 1LL * a->batch * a->M * a->N;
    const int blocks = static_cast<int>(total / 256 + 1 < 16LL * sm_count ? total / 256 + 1 : 16LL * sm_count);
    splitk_reduce_kernel<<<blocks, 256, 0, stream>>>(dev.split_ws, reinterpret_cast<float*>(a->C), dev.splits, dev.batch, dev.M,
                                                     dev.N, dev.ldc, dev.strideC, dev.row_interleave);
    return check_launch("md_gemm_bf16 (deterministic split-K reduction)");
  }
  return 0;
}
