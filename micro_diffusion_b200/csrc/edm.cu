// EDM noise / preconditioning / loss step and random patch masking of the MicroDiT training path.
// Reference: LatentDiffusion.edm_loss + model_forward_wrapper (model.py:144-210), get_mask /
// mask_out_token / unmask_tokens (utils.py:382-426), DiT.unpatchify (dit.py:566-575).
// HBM-bound; masked patches are never materialised on the training path (mask_token is a zero buffer
// and masked patches carry zero loss weight, model.py:206-209).
#include <cuda_fp16.h>

#include "act.cuh"

namespace md {

__device__ __forceinline__ float load_lat(const void* lat, int f16, long long i) {
  return f16 ? __half2float(reinterpret_cast<const __half*>(lat)[i]) : reinterpret_cast<const float*>(lat)[i];
}

// coef layout: [0]=sigma [1]=c_skip [2]=c_out [3]=c_in [4]=c_noise [5]=weight, each [B]
__global__ void edm_coef_kernel(const float* __restrict__ rnd, const float* __restrict__ sigma_in, float p_mean,
                                float p_std, float sd, float* __restrict__ coef, int B) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const float sigma = sigma_in ? sigma_in[b] : expf(rnd[b] * p_std + p_mean);
  const float s2 = sigma * sigma, d2 = sd * sd;
  coef[0 * B + b] = sigma;
  coef[1 * B + b] = d2 / (s2 + d2);
  coef[2 * B + b] = sigma * sd / sqrtf(s2 + d2);
  coef[3 * B + b] = 1.f / sqrtf(d2 + s2);
  coef[4 * B + b] = logf(sigma) * 0.25f;
  coef[5 * B + b] = (s2 + d2) / ((sigma * sd) * (sigma * sd));
}

// one thread per (sample, patch, channel, patch-row): p consecutive pixels (coalesced across patches)
template <typename AT>
__global__ void edm_prepare_kernel(const void* __restrict__ lat, int lat_f16, const float* __restrict__ eps,
                                   const float* __restrict__ coef, float* __restrict__ xn, AT* __restrict__ patches,
                                   int B, int C, int H, int W, int p) {
  const int gw = W / p, gh = H / p;
  const long long total = 1LL * B * C * H * gw;  // (b, c, y, patch-col)
  const int Kp = C * p * p;
  for (long long i = 1LL * blockIdx.x * blockDim.x + threadIdx.x; i < total; i += 1LL * gridDim.x * blockDim.x) {
    const int pw = static_cast<int>(i % gw);
    long long r = i / gw;
    const int y = static_cast<int>(r % H); r /= H;
    const int c = static_cast<int>(r % C);
    const int b = static_cast<int>(r / C);
    const float sigma = coef[b], c_in = coef[3 * B + b];
    const int ph = y / p, ii = y % p;
    const long long tok = 1LL * b * gh * gw + 1LL * ph * gw + pw;
    for (int j = 0; j < p; ++j) {
      const long long src = ((1LL * b * C + c) * H + y) * W + pw * p + j;
      const float v = load_lat(lat, lat_f16, src) + sigma * eps[src];
      xn[src] = v;
      st1a(patches + tok * Kp + (c * p + ii) * p + j, c_in * v);
    }
  }
}

template <typename AT>
__global__ void patchify_kernel(const float* __restrict__ x, const float* __restrict__ scale, AT* __restrict__ patches,
                                int B, int C, int H, int W, int p) {
  const int gw = W / p, gh = H / p;
  const long long total = 1LL * B * C * H * gw;
  const int Kp = C * p * p;
  for (long long i = 1LL * blockIdx.x * blockDim.x + threadIdx.x; i < total; i += 1LL * gridDim.x * blockDim.x) {
    const int pw = static_cast<int>(i % gw);
    long long r = i / gw;
    const int y = static_cast<int>(r % H); r /= H;
    const int c = static_cast<int>(r % C);
    const int b = static_cast<int>(r / C);
    const float sc = scale ? scale[b] : 1.f;
    const long long tok = 1LL * b * gh * gw + 1LL * (y / p) * gw + pw;
    for (int j = 0; j < p; ++j)
      st1a(patches + tok * Kp + (c * p + y % p) * p + j, sc * x[((1LL * b * C + c) * H + y) * W + pw * p + j]);
  }
}

// Per-sample masked, weighted MSE.  One block per sample; thread per kept token.
// ftok column for pixel (c, i, j) of a patch is (i*p + j)*C + c (unpatchify 'nhwpqc->nchpwq').
template <bool kBackward, typename AT>
__global__ void __launch_bounds__(256)
edm_loss_kernel(const float* __restrict__ ftok, const int32_t* __restrict__ keep_tok, const void* __restrict__ lat,
                int lat_f16, const float* __restrict__ xn, const float* __restrict__ coef,
                float* __restrict__ per_sample, float* __restrict__ loss, const float* __restrict__ gscale,
                AT* __restrict__ dftok, int B, int C, int H, int W, int p, int Tk, float* __restrict__ det_ws) {
  const int b = blockIdx.x;
  const int gw = W / p;
  const int T = gw * (H / p);
  const int Nf = p * p * C;
  const float c_skip = coef[1 * B + b], c_out = coef[2 * B + b], wgt = coef[5 * B + b];
  const float inv = 1.f / (static_cast<float>(C) * p * p);
  float acc = 0.f;
  float gs = 0.f;
  if (kBackward) gs = gscale[0] * (1.f / B) * (1.f / Tk) * inv * wgt * 2.f * c_out;
  for (int j = threadIdx.x; j < Tk; j += blockDim.x) {
    const int tok = keep_tok ? keep_tok[1LL * b * Tk + j] % T : j;  // keep_tok holds global rows b*T + token
    const int ph = tok / gw, pw = tok % gw;
    const float* f = ftok + (1LL * b * Tk + j) * Nf;
    for (int c = 0; c < C; ++c)
      for (int ii = 0; ii < p; ++ii)
        for (int jj = 0; jj < p; ++jj) {
          const long long src = ((1LL * b * C + c) * H + ph * p + ii) * W + pw * p + jj;
          const float xv = load_lat(lat, lat_f16, src);
          const float d = c_skip * xn[src] + c_out * f[(ii * p + jj) * C + c] - xv;
          if (kBackward)
            st1a(dftok + (1LL * b * Tk + j) * Nf + (ii * p + jj) * C + c, gs * d);
          else
            acc += wgt * d * d;
        }
  }
  if (kBackward) return;
  acc = warp_sum(acc);
  __shared__ float part[8];
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int w = 0; w < (blockDim.x >> 5); ++w) s += part[w];
    s = s * inv / Tk;
    per_sample[b] = s;
    if (det_ws != nullptr) det_ws[b] = s / B;   // deterministic mode: summed over samples in a fixed order afterwards
    else atomicAdd(loss, s / B);
  }
}

__global__ void edm_output_kernel(const float* __restrict__ ftok, const int32_t* __restrict__ ids_restore,
                                  const float* __restrict__ mask_token, const float* __restrict__ xn,
                                  const float* __restrict__ coef, float* __restrict__ fx, float* __restrict__ dx,
                                  int B, int C, int H, int W, int p, int Tk) {
  const int gw = W / p, gh = H / p, T = gw * gh, Nf = p * p * C;
  const long long total = 1LL * B * C * H * W;
  for (long long i = 1LL * blockIdx.x * blockDim.x + threadIdx.x; i < total; i += 1LL * gridDim.x * blockDim.x) {
    const int x = static_cast<int>(i % W);
    long long r = i / W;
    const int y = static_cast<int>(r % H); r /= H;
    const int c = static_cast<int>(r % C);
    const int b = static_cast<int>(r / C);
    const int tok = (y / p) * gw + x / p;
    const int col = ((y % p) * p + (x % p)) * C + c;
    const int pos = ids_restore ? ids_restore[1LL * b * T + tok] : tok;
    const float f = pos < Tk ? ftok[(1LL * b * Tk + pos) * Nf + col] : (mask_token ? mask_token[col] : 0.f);
    if (fx) fx[i] = f;
    if (dx) dx[i] = coef[1 * B + b] * xn[i] + coef[2 * B + b] * f;
  }
}

// ------------------------------------------------------------------------------------- adjoints (DiT VJP)
// Adjoint of the un-mask + unpatchify of edm_output_kernel for the raw output F: one thread per element of dftok
// [B*Tk, p*p*C] (column (i*p+j)*C+c, coalesced writes).  Masked tokens show the non-trainable mask_token buffer, so only
// the kept tokens have a gradient.
template <typename AT>
__global__ void unpatchify_bwd_kernel(const float* __restrict__ dF, const int32_t* __restrict__ keep_rows,
                                      AT* __restrict__ dftok, int B, int C, int H, int W, int p, int Tk) {
  const int gw = W / p, T = gw * (H / p), Nf = p * p * C;
  const long long total = 1LL * B * Tk * Nf;
  for (long long i = 1LL * blockIdx.x * blockDim.x + threadIdx.x; i < total; i += 1LL * gridDim.x * blockDim.x) {
    const int col = static_cast<int>(i % Nf);
    const long long row = i / Nf;  // b * Tk + j
    const int b = static_cast<int>(row / Tk);
    const int tok = keep_rows ? keep_rows[row] % T : static_cast<int>(row % Tk);  // keep_rows holds b*T + token
    const int c = col % C, q = col / C;
    const long long src = ((1LL * b * C + c) * H + (tok / gw) * p + q / p) * W + (tok % gw) * p + q % p;
    st1a(dftok + i, dF[src]);
  }
}

// Adjoint of patchify_kernel (col2im of the stride-p patch-embed conv, column (c*p+i)*p+j): the patches do not overlap,
// so every pixel reads exactly one element.  One thread per pixel of dx (coalesced writes).
__global__ void patchify_bwd_kernel(const float* __restrict__ dpatches, const float* __restrict__ scale,
                                    float* __restrict__ dx, int B, int C, int H, int W, int p) {
  const int gw = W / p, gh = H / p, Kp = C * p * p;
  const long long total = 1LL * B * C * H * W;
  for (long long i = 1LL * blockIdx.x * blockDim.x + threadIdx.x; i < total; i += 1LL * gridDim.x * blockDim.x) {
    const int x = static_cast<int>(i % W);
    long long r = i / W;
    const int y = static_cast<int>(r % H); r /= H;
    const int c = static_cast<int>(r % C);
    const int b = static_cast<int>(r / C);
    const long long tok = 1LL * b * gh * gw + 1LL * (y / p) * gw + x / p;
    const float v = dpatches[tok * Kp + (c * p + y % p) * p + x % p];
    dx[i] = scale ? scale[b] * v : v;
  }
}

// Adjoint of timestep_embed_kernel: dt[b] = sum_i f_i * (dfreq[b, half+i] cos(t f_i) - dfreq[b, i] sin(t f_i)).  One
// block per sample; every thread sums a fixed stride of frequencies, then a fixed-order warp / block reduction, so the
// result does not depend on scheduling (no atomics).
__global__ void __launch_bounds__(256)
timestep_embed_bwd_kernel(const float* __restrict__ dfreq, const float* __restrict__ t, float* __restrict__ dt, int dim) {
  const long long b = blockIdx.x;
  const int half = dim / 2;
  const float tv = t[b];
  float acc = 0.f;
  for (int i = threadIdx.x; i < half; i += blockDim.x) {
    const float freq = expf(-9.210340371976184f * static_cast<float>(i) / static_cast<float>(half));
    const float a = tv * freq;
    acc += freq * (dfreq[b * dim + half + i] * cosf(a) - dfreq[b * dim + i] * sinf(a));
  }
  acc = warp_sum(acc);
  __shared__ float part[8];
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int w = 0; w < (blockDim.x >> 5); ++w) s += part[w];
    dt[b] = s;
  }
}

// ------------------------------------------------------------------------------------- mask_sort
// One block per sample: bitonic sort of (noise, index) ascending in shared memory (n = next pow2 >= T).
__global__ void __launch_bounds__(1024)
mask_sort_kernel(const float* __restrict__ noise, int32_t* __restrict__ ids_shuffle, int32_t* __restrict__ ids_restore,
                 float* __restrict__ mask, int32_t* __restrict__ keep_rows, int T, int keep, int n) {
  extern __shared__ unsigned long long keys[];  // (orderable float bits << 32) | index
  const long long b = blockIdx.x;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    unsigned long long k = ~0ULL;
    if (i < T) {
      unsigned int u = __float_as_uint(noise[b * T + i]);
      u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);  // total order on floats
      k = (static_cast<unsigned long long>(u) << 32) | static_cast<unsigned int>(i);
    }
    keys[i] = k;
  }
  __syncthreads();
  for (int size = 2; size <= n; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int i = threadIdx.x; i < (n >> 1); i += blockDim.x) {
        const int lo = 2 * i - (i & (stride - 1));
        const int hi = lo + stride;
        const bool up = ((lo & size) == 0);
        const unsigned long long a = keys[lo], c = keys[hi];
        if ((a > c) == up) {
          keys[lo] = c;
          keys[hi] = a;
        }
      }
      __syncthreads();
    }
  }
  for (int j = threadIdx.x; j < T; j += blockDim.x) {
    const int idx = static_cast<int>(keys[j] & 0xffffffffu);
    if (ids_shuffle) ids_shuffle[b * T + j] = idx;
    if (ids_restore) ids_restore[b * T + idx] = j;
    if (mask) mask[b * T + idx] = j < keep ? 0.f : 1.f;
    if (keep_rows && j < keep) keep_rows[b * keep + j] = static_cast<int32_t>(b * T + idx);
  }
}

__global__ void gather_rows_kernel(const float* __restrict__ x, const int32_t* __restrict__ src_rows,
                                   float* __restrict__ y, long long rows, int D, int scatter_add) {
  const int dv = D >> 2;
  const long long total = rows * dv;
  for (long long i = 1LL * blockIdx.x * blockDim.x + threadIdx.x; i < total; i += 1LL * gridDim.x * blockDim.x) {
    const long long r = i / dv;
    const int c = static_cast<int>(i % dv) * 4;
    const long long s = src_rows[r];
    if (!scatter_add) {
      *reinterpret_cast<float4*>(y + r * D + c) = *reinterpret_cast<const float4*>(x + s * D + c);
    } else {  // y[s] += x[r]; source rows are unique, so no atomics are needed
      float4 a = *reinterpret_cast<float4*>(y + s * D + c);
      const float4 v = *reinterpret_cast<const float4*>(x + r * D + c);
      a.x += v.x; a.y += v.y; a.z += v.z; a.w += v.w;
      *reinterpret_cast<float4*>(y + s * D + c) = a;
    }
  }
}

// ------------------------------------------------------------------------------------- EDM Heun sampler
// The fp64 state update of LatentDiffusion._heun (model.py:260-276), one launch per stage, so that one captured CUDA graph
// serves every step: the per-step times come from a device table and a device step index that the graph advances itself.
// table f64 [2*max_steps + 1] = [t_steps[0..max_steps] | t_hat[0..max_steps)].  Every operation is an explicitly rounded
// intrinsic in the association order of the torch expressions, so nothing is contracted into an FMA and the state is
// bit-identical to the eager loop's.
enum { HEUN_IN = 0, HEUN_EULER = 1, HEUN_CORRECT = 2, HEUN_NEXT = 3 };

__global__ void edm_heun_kernel(int stage, double* __restrict__ x, double* __restrict__ x_hat, double* __restrict__ d_cur,
                                const float* __restrict__ den, const double* __restrict__ noise, float* __restrict__ xin,
                                float* __restrict__ sigma, const double* __restrict__ table,
                                const int32_t* __restrict__ step, int max_steps, long long n, int B, int copies,
                                double s_noise) {
  const int k = *step;
  const bool ok = k >= 0 && k < max_steps;  // an index outside the table poisons the outputs instead of reading past it
  const double nan = __longlong_as_double(0x7ff8000000000000LL);
  const double t_cur = ok ? table[k] : nan, t_next = ok ? table[k + 1] : nan, t_hat = ok ? table[max_steps + 1 + k] : nan;
  const long long tid = 1LL * blockIdx.x * blockDim.x + threadIdx.x;
  if (stage != HEUN_CORRECT && tid < 1LL * copies * B)
    sigma[tid] = __double2float_rn(stage == HEUN_IN ? t_hat : t_next);  // t_hat / t_next .to(float32), per sample
  // (t_hat ** 2 - t_cur ** 2).sqrt() * S_noise and t_next - t_hat: 0-dim tensors in the eager loop
  const double c_noise = __dmul_rn(__dsqrt_rn(__dsub_rn(__dmul_rn(t_hat, t_hat), __dmul_rn(t_cur, t_cur))), s_noise);
  const double dt = __dsub_rn(t_next, t_hat);
  for (long long i = tid; i < n; i += 1LL * gridDim.x * blockDim.x) {
    double out;
    if (stage == HEUN_IN) {  // x_hat = x_cur + c * n_k
      out = __dadd_rn(x[i], __dmul_rn(c_noise, ok ? noise[1LL * k * n + i] : nan));
      x_hat[i] = out;
    } else if (stage == HEUN_EULER) {  // d_cur = (x_hat - D) / t_hat; x_next = x_hat + (t_next - t_hat) * d_cur
      const double xh = x_hat[i];
      const double d = __ddiv_rn(__dsub_rn(xh, static_cast<double>(den[i])), t_hat);
      d_cur[i] = d;
      out = __dadd_rn(xh, __dmul_rn(dt, d));
      x[i] = out;
    } else {  // d' = (x_next - D) / t_next; x_next = x_hat + (t_next - t_hat) * (0.5 * d_cur + 0.5 * d')
      const double dp = __ddiv_rn(__dsub_rn(x[i], static_cast<double>(den[i])), t_next);
      x[i] = __dadd_rn(x_hat[i], __dmul_rn(dt, __dadd_rn(__dmul_rn(0.5, d_cur[i]), __dmul_rn(0.5, dp))));
      continue;
    }
    const float f = __double2float_rn(out);  // the next denoiser input, in both halves of a CFG batch
    xin[i] = f;
    if (copies == 2) xin[n + i] = f;
  }
}

__global__ void edm_heun_next_kernel(int32_t* step) { *step += 1; }

// Classifier-free guidance + preconditioning for the doubled batch (model.py:197-201): ftok holds the cond samples
// [0, B) then the uncond samples [B, 2B).  D = c_skip * x + c_out * (unc + cfg * (cond - unc)) with the rounding of the
// torch expression: c_skip = reciprocal(sg*sg + sd2) * sd2 (a Python float over a tensor is a reciprocal and a product),
// c_out = (sg * sd) / sqrt(sg*sg + sd2), every product and sum rounded on its own.
__global__ void edm_output_cfg_kernel(const float* __restrict__ ftok, const float* __restrict__ x,
                                      const float* __restrict__ sigma, const float* __restrict__ cfg,
                                      float* __restrict__ dx, float sd, float sd2, int B, int C, int H, int W, int p) {
  const int gw = W / p, T = gw * (H / p), Nf = p * p * C;
  const long long total = 1LL * B * C * H * W;
  const float g = *cfg;
  for (long long i = 1LL * blockIdx.x * blockDim.x + threadIdx.x; i < total; i += 1LL * gridDim.x * blockDim.x) {
    const int xx = static_cast<int>(i % W);
    long long r = i / W;
    const int y = static_cast<int>(r % H); r /= H;
    const int c = static_cast<int>(r % C);
    const int b = static_cast<int>(r / C);
    const long long col = ((y % p) * p + (xx % p)) * C + c, tok = (y / p) * gw + xx / p;
    const float cond = ftok[(1LL * b * T + tok) * Nf + col], unc = ftok[(1LL * (B + b) * T + tok) * Nf + col];
    const float f = __fadd_rn(unc, __fmul_rn(g, __fsub_rn(cond, unc)));
    const float sg = sigma[b];
    const float den = __fadd_rn(__fmul_rn(sg, sg), sd2);
    const float c_skip = __fmul_rn(__frcp_rn(den), sd2);
    const float c_out = __fdiv_rn(__fmul_rn(sg, sd), __fsqrt_rn(den));
    dx[i] = __fadd_rn(__fmul_rn(c_skip, x[i]), __fmul_rn(c_out, f));
  }
}

static int grid_for(long long items, int threads) {
  long long blocks = (items + threads - 1) / threads;
  if (blocks > 132LL * 16) blocks = 132LL * 16;
  if (blocks < 1) blocks = 1;
  return static_cast<int>(blocks);
}

}  // namespace md

using namespace md;
#define ST(s) reinterpret_cast<cudaStream_t>(s)

extern "C" int md_edm_prepare(const void* lat, int lat_f16, const float* eps, const float* rnd, const float* sigma_in,
                              float p_mean, float p_std, float sigma_data, float* xn, void* patches, float* coef,
                              int64_t B, int64_t C, int64_t H, int64_t W, int64_t p, int prec, void* stream) {
  if (B == 0) return 0;
  if (!lat || !eps || (!rnd && !sigma_in) || !xn || !patches || !coef)
    return md_set_error(MD_ERR_INVALID, "md_edm_prepare: null pointer");
  if (p <= 0 || H % p != 0 || W % p != 0) return md_set_error(MD_ERR_INVALID, "md_edm_prepare: H, W must be multiples of p");
  edm_coef_kernel<<<(unsigned)((B + 127) / 128), 128, 0, ST(stream)>>>(rnd, sigma_in, p_mean, p_std, sigma_data, coef,
                                                                      (int)B);
  MD_WITH_ACT(prec, edm_prepare_kernel<AT><<<grid_for(B * C * H * (W / p), 256), 256, 0, ST(stream)>>>(
                        lat, lat_f16, eps, coef, xn, AP(AT, patches), (int)B, (int)C, (int)H, (int)W, (int)p));
  return check_launch("md_edm_prepare");
}

extern "C" int md_patchify(const float* x, const float* scale, void* patches, int64_t B, int64_t C, int64_t H,
                           int64_t W, int64_t p, int prec, void* stream) {
  if (B == 0) return 0;
  if (!x || !patches) return md_set_error(MD_ERR_INVALID, "md_patchify: null pointer");
  if (p <= 0 || H % p != 0 || W % p != 0) return md_set_error(MD_ERR_INVALID, "md_patchify: H, W must be multiples of p");
  MD_WITH_ACT(prec, patchify_kernel<AT><<<grid_for(B * C * H * (W / p), 256), 256, 0, ST(stream)>>>(
                        x, scale, AP(AT, patches), (int)B, (int)C, (int)H, (int)W, (int)p));
  return check_launch("md_patchify");
}

extern "C" int md_edm_loss_fwd(const float* ftok, const int32_t* keep_tok, const void* lat, int lat_f16,
                               const float* xn, const float* coef, float* per_sample, float* loss, int64_t B,
                               int64_t C, int64_t H, int64_t W, int64_t p, int64_t Tk, void* stream) {
  if (B == 0) return 0;
  if (!ftok || !lat || !xn || !coef || !per_sample || !loss)
    return md_set_error(MD_ERR_INVALID, "md_edm_loss_fwd: null pointer");
  float* ws = nullptr;
  if (det_enabled()) {  // B > 262144 samples overflow the 1 MiB minimum workspace: refuse rather than take the atomics
    ws = det_workspace(static_cast<size_t>(B) * sizeof(float));
    if (ws == nullptr) return md_set_error(MD_ERR_INVALID, "md_edm_loss_fwd: deterministic workspace too small");
  }
  edm_loss_kernel<false, float><<<(unsigned)B, 256, 0, ST(stream)>>>(ftok, keep_tok, lat, lat_f16, xn, coef, per_sample,
                                                                     loss, nullptr, nullptr, (int)B, (int)C, (int)H,
                                                                     (int)W, (int)p, (int)Tk, ws);
  if (int rc = check_launch("md_edm_loss_fwd")) return rc;
  return ws ? det_reduce(ws, loss, B, 1, 1, ST(stream)) : 0;
}

extern "C" int md_edm_loss_bwd(const float* ftok, const int32_t* keep_tok, const void* lat, int lat_f16,
                               const float* xn, const float* coef, const float* gscale, void* dftok, int64_t B,
                               int64_t C, int64_t H, int64_t W, int64_t p, int64_t Tk, int prec, void* stream) {
  if (B == 0) return 0;
  if (!ftok || !lat || !xn || !coef || !gscale || !dftok)
    return md_set_error(MD_ERR_INVALID, "md_edm_loss_bwd: null pointer");
  MD_WITH_ACT(prec, edm_loss_kernel<true, AT><<<(unsigned)B, 256, 0, ST(stream)>>>(
                        ftok, keep_tok, lat, lat_f16, xn, coef, nullptr, nullptr, gscale, AP(AT, dftok), (int)B, (int)C,
                        (int)H, (int)W, (int)p, (int)Tk, nullptr));
  return check_launch("md_edm_loss_bwd");
}

extern "C" int md_edm_output(const float* ftok, const int32_t* ids_restore, const float* mask_token, const float* xn,
                             const float* coef, float* fx, float* dx, int64_t B, int64_t C, int64_t H, int64_t W,
                             int64_t p, int64_t Tk, void* stream) {
  if (B == 0) return 0;
  if (!ftok || (dx && (!xn || !coef))) return md_set_error(MD_ERR_INVALID, "md_edm_output: null pointer");
  edm_output_kernel<<<grid_for(B * C * H * W, 256), 256, 0, ST(stream)>>>(ftok, ids_restore, mask_token, xn, coef, fx,
                                                                          dx, (int)B, (int)C, (int)H, (int)W, (int)p,
                                                                          (int)Tk);
  return check_launch("md_edm_output");
}

extern "C" int md_unpatchify_bwd(const float* dF, const int32_t* keep_rows, void* dftok, int64_t B, int64_t C, int64_t H,
                                 int64_t W, int64_t p, int64_t Tk, int prec, void* stream) {
  if (B == 0) return 0;
  if (!dF || !dftok) return md_set_error(MD_ERR_INVALID, "md_unpatchify_bwd: null pointer");
  if (p <= 0 || H % p != 0 || W % p != 0)
    return md_set_error(MD_ERR_INVALID, "md_unpatchify_bwd: H, W must be multiples of p");
  if (Tk < 1 || Tk > (H / p) * (W / p) || (!keep_rows && Tk != (H / p) * (W / p)))
    return md_set_error(MD_ERR_INVALID, "md_unpatchify_bwd: Tk must be in [1, T] (T without keep_rows)");
  if (prec != 0 && prec != 1) return md_set_error(MD_ERR_INVALID, "md_unpatchify_bwd: prec must be 0 or 1");
  MD_WITH_ACT(prec, unpatchify_bwd_kernel<AT><<<grid_for(B * Tk * C * p * p, 256), 256, 0, ST(stream)>>>(
                        dF, keep_rows, AP(AT, dftok), (int)B, (int)C, (int)H, (int)W, (int)p, (int)Tk));
  return check_launch("md_unpatchify_bwd");
}

extern "C" int md_patchify_bwd(const float* dpatches, const float* scale, float* dx, int64_t B, int64_t C, int64_t H,
                               int64_t W, int64_t p, int prec, void* stream) {
  if (B == 0) return 0;
  if (!dpatches || !dx) return md_set_error(MD_ERR_INVALID, "md_patchify_bwd: null pointer");
  if (p <= 0 || H % p != 0 || W % p != 0)
    return md_set_error(MD_ERR_INVALID, "md_patchify_bwd: H, W must be multiples of p");
  if (prec != 0 && prec != 1) return md_set_error(MD_ERR_INVALID, "md_patchify_bwd: prec must be 0 or 1");
  patchify_bwd_kernel<<<grid_for(B * C * H * W, 256), 256, 0, ST(stream)>>>(dpatches, scale, dx, (int)B, (int)C, (int)H,
                                                                           (int)W, (int)p);
  return check_launch("md_patchify_bwd");
}

extern "C" int md_timestep_embed_bwd(const float* dfreq, const float* t, float* dt, int64_t B, int64_t dim, int prec,
                                     void* stream) {
  if (B == 0) return 0;
  if (!dfreq || !t || !dt) return md_set_error(MD_ERR_INVALID, "md_timestep_embed_bwd: null pointer");
  if (dim < 2) return md_set_error(MD_ERR_INVALID, "md_timestep_embed_bwd: dim must be >= 2");
  if (prec != 0 && prec != 1) return md_set_error(MD_ERR_INVALID, "md_timestep_embed_bwd: prec must be 0 or 1");
  timestep_embed_bwd_kernel<<<(unsigned)B, 256, 0, ST(stream)>>>(dfreq, t, dt, (int)dim);
  return check_launch("md_timestep_embed_bwd");
}

extern "C" int md_mask_sort(const float* noise, int32_t* ids_shuffle, int32_t* ids_restore, float* mask,
                            int32_t* keep_rows, int64_t B, int64_t T, int64_t keep, void* stream) {
  if (B == 0) return 0;
  if (!noise) return md_set_error(MD_ERR_INVALID, "md_mask_sort: null pointer");
  if (T > 4096 || T < 1) return md_set_error(MD_ERR_UNSUPPORTED, "md_mask_sort: T must be in [1, 4096]");
  int n = 1;
  while (n < T) n <<= 1;
  if (n < 2) n = 2;
  const int threads = n / 2 < 32 ? 32 : (n / 2 > 1024 ? 1024 : n / 2);
  mask_sort_kernel<<<(unsigned)B, threads, n * sizeof(unsigned long long), ST(stream)>>>(
      noise, ids_shuffle, ids_restore, mask, keep_rows, (int)T, (int)keep, n);
  return check_launch("md_mask_sort");
}

extern "C" int md_gather_rows_f32(const float* x, const int32_t* src_rows, float* y, int64_t rows, int64_t D,
                                  void* stream) {
  if (rows == 0) return 0;
  if (!x || !src_rows || !y || D % 4 != 0) return md_set_error(MD_ERR_INVALID, "md_gather_rows_f32: bad argument");
  gather_rows_kernel<<<grid_for(rows * (D / 4), 256), 256, 0, ST(stream)>>>(x, src_rows, y, rows, (int)D, 0);
  return check_launch("md_gather_rows_f32");
}
extern "C" int md_scatter_rows_f32(const float* dy, const int32_t* src_rows, float* dx, int64_t rows, int64_t D,
                                   void* stream) {
  if (rows == 0) return 0;
  if (!dy || !src_rows || !dx || D % 4 != 0) return md_set_error(MD_ERR_INVALID, "md_scatter_rows_f32: bad argument");
  gather_rows_kernel<<<grid_for(rows * (D / 4), 256), 256, 0, ST(stream)>>>(dy, src_rows, dx, rows, (int)D, 1);
  return check_launch("md_scatter_rows_f32");
}

extern "C" int md_edm_heun(int stage, double* x, double* x_hat, double* d_cur, const float* den, const double* noise,
                           float* xin, float* sigma, const double* table, int32_t* step, int64_t max_steps, int64_t B,
                           int64_t sample_numel, int64_t copies, double s_noise, void* stream) {
  if (stage < HEUN_IN || stage > HEUN_NEXT) return md_set_error(MD_ERR_INVALID, "md_edm_heun: stage must be 0..3");
  if (!step) return md_set_error(MD_ERR_INVALID, "md_edm_heun: null pointer");
  if (stage == HEUN_NEXT) {
    edm_heun_next_kernel<<<1, 1, 0, ST(stream)>>>(step);
    return check_launch("md_edm_heun");
  }
  if (max_steps < 1 || max_steps > (1 << 20)) return md_set_error(MD_ERR_INVALID, "md_edm_heun: max_steps out of range");
  if (B < 1 || sample_numel < 1 || (copies != 1 && copies != 2))
    return md_set_error(MD_ERR_INVALID, "md_edm_heun: B and sample_numel must be >= 1, copies 1 or 2");
  if (!table || !x || !x_hat) return md_set_error(MD_ERR_INVALID, "md_edm_heun: null pointer");
  if (stage == HEUN_IN && (!noise || !xin || !sigma)) return md_set_error(MD_ERR_INVALID, "md_edm_heun: null pointer");
  if (stage == HEUN_EULER && (!d_cur || !den || !xin || !sigma))
    return md_set_error(MD_ERR_INVALID, "md_edm_heun: null pointer");
  if (stage == HEUN_CORRECT && (!d_cur || !den)) return md_set_error(MD_ERR_INVALID, "md_edm_heun: null pointer");
  const long long n = B * sample_numel;
  edm_heun_kernel<<<grid_for(n, 256), 256, 0, ST(stream)>>>(stage, x, x_hat, d_cur, den, noise, xin, sigma, table, step,
                                                            (int)max_steps, n, (int)B, (int)copies, s_noise);
  return check_launch("md_edm_heun");
}

extern "C" int md_edm_output_cfg(const float* ftok, const float* x, const float* sigma, const float* cfg, float* dx,
                                 float sigma_data, float sigma_data_sq, int64_t B, int64_t C, int64_t H, int64_t W,
                                 int64_t p, void* stream) {
  if (B == 0) return 0;
  if (!ftok || !x || !sigma || !cfg || !dx) return md_set_error(MD_ERR_INVALID, "md_edm_output_cfg: null pointer");
  if (B < 0 || C < 1 || p <= 0 || H % p != 0 || W % p != 0)
    return md_set_error(MD_ERR_INVALID, "md_edm_output_cfg: bad shape (H, W must be multiples of p)");
  edm_output_cfg_kernel<<<grid_for(B * C * H * W, 256), 256, 0, ST(stream)>>>(ftok, x, sigma, cfg, dx, sigma_data,
                                                                             sigma_data_sq, (int)B, (int)C, (int)H,
                                                                             (int)W, (int)p);
  return check_launch("md_edm_output_cfg");
}
