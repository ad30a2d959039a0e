// Surface (2-D) and edge (1-D) VAE decoders: latents -> 32x32 / 32-point control grids.
//
// Reference: AutoencoderKLFastDecode.forward network.py:1013-1040 (diffusers 0.27 `Decoder`, cfg
// sample.py:72-82) and AutoencoderKL1DFastDecode.forward network.py:846-858 (Decoder1D :188-299, UNetMidBlock1D :51-83,
// UpBlock1D :30-48, cfg sample.py:86-97); layer-by-layer arithmetic: SURVEY.md Appendix A.1 / A.2.
//
// Layout: activations are channels-last ([sample][position][channel]), fp32 for the residual stream and fp16 for GEMM
// operands.  Convolutions are IMPLICIT GEMMs on the wgmma GEMM kernel (gemm.cu, ConvGeom): the A tile of
// k-block (term, tap, 64-channel chunk) is a TMA box of the channels-last image shifted by the tap's offset, out-of-range
// coordinates zero-filled = the padding, so the im2col matrix only ever exists as shared-memory tiles (round 1 / early
// round 2 materialised it in HBM: ~9x the activation traffic and ~40 % of the decode time).  The few shapes a box cannot
// express (3 input channels, 3 x 3 / 24 x 24 extents, stride-2 encoder convolutions) keep the explicit gather.  The GEMM
// epilogue adds bias and the residual; GroupNorm + SiLU/GELU (+ residual) is one CTA-per-sample kernel; nearest-2x
// upsampling is one gather into the next convolution's input; the tiny attentions run on CUDA cores.
#include <algorithm>
#include <string>
#include <type_traits>
#include <utility>

#include "../../include/brepgen_b200.h"
#include "bg_internal.h"

#include <stdlib.h>

namespace bg {
namespace {

inline int round64(int k) { return (k + 63) / 64 * 64; }

// ------------------------------------------------------------------------------------------------ kernels
// Compensated fp16 products.  Every GEMM of the decoders computes  A_hi W_hi + A_lo W_hi + A_hi W_lo  (hi = fp16(v),
// lo = fp16(v - hi); only the ~2^-22 lo*lo term is dropped) as ONE GEMM over a 3x longer K: activations are stored as
// [hi | lo] pairs (pitch 2C), weights as [W_hi | W_hi | W_lo], and the A tile wraps around after 2K columns (a_kwrap).
// ~30 chained convolutions otherwise accumulate 1.9e-3 of fp16 rounding; decode is 0.13 % of the cascade's FLOPs.
// weights [Cout][Cin][taps] fp32 -> [Cout_pad][3 * Kpad] fp16 with k = tap * Cin + cin (zero padded)
__global__ void pack_conv_kernel(const float* __restrict__ w, __half* __restrict__ dst, int Cout, int Cin, int taps, int Kpad,
                                 int Cout_pad, int terms) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)Cout_pad * Kpad) return;
  const int co = (int)(i / Kpad), k = (int)(i % Kpad);
  float v = 0.f;
  if (co < Cout && k < taps * Cin) {
    const int tap = k / Cin, ci = k % Cin;
    v = w[((size_t)co * Cin + ci) * taps + tap];
  }
  const __half hi = __float2half_rn(v), lo = __float2half_rn(v - __half2float(hi));
  dst[(size_t)co * 3 * Kpad + k] = hi;                                  // 3 terms: [W_hi | W_hi | W_lo]
  dst[(size_t)co * 3 * Kpad + Kpad + k] = terms == 3 ? hi : lo;         // 2 terms: [W_hi | W_lo | (unused)]
  dst[(size_t)co * 3 * Kpad + 2 * Kpad + k] = lo;
}
__device__ __forceinline__ void store_hl(__half* dst, int lo_off, float v) {
  const __half hi = __float2half_rn(v);
  dst[0] = hi;
  dst[lo_off] = __float2half_rn(v - __half2float(hi));
}
// x fp32 [rows][C] -> [rows][2C] fp16 hi|lo
__global__ void cast_split_kernel(const float* __restrict__ x, __half* __restrict__ y, int C, size_t total) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const size_t row = i / C;
    const int c = (int)(i % C);
    store_hl(y + row * 2 * C + c, C, x[i]);
  }
}

// nearest-2x upsampling into the [hi | lo] fp16 input of the following convolution: x fp32 (N, H, W, C) -> y (N, 2H, 2W, 2C)
__global__ void upsample2x_split_kernel(const float* __restrict__ x, __half* __restrict__ y, int H, int W, int C, size_t total) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    size_t pix = i / C;                                   // output pixel (n, yo, xo)
    const int xo = (int)(pix % (2 * W)), yo = (int)((pix / (2 * W)) % (2 * H));
    const size_t n = pix / ((size_t)4 * W * H);
    store_hl(y + pix * 2 * C + c, C, x[((n * H + (yo >> 1)) * W + (xo >> 1)) * C + c]);
  }
}

// z (N, 3, P) fp32 -> y (N, P, [3 hi | 3 lo]) fp16, y = W z + b  (post_quant_conv, 1x1)
__global__ void postquant_kernel(const float* __restrict__ z, const float* __restrict__ w, const float* __restrict__ b,
                                 __half* __restrict__ y, int N, int P) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N * P) return;
  const int n = i / P, p = i % P;
  const float z0 = z[((size_t)n * 3 + 0) * P + p], z1 = z[((size_t)n * 3 + 1) * P + p], z2 = z[((size_t)n * 3 + 2) * P + p];
#pragma unroll
  for (int co = 0; co < 3; ++co)
    store_hl(y + (size_t)i * 6 + co, 3, b[co] + w[co * 3] * z0 + w[co * 3 + 1] * z1 + w[co * 3 + 2] * z2);
}

// in (N, H, W, C) fp16 (pitch ldin per pixel) -> A (N*Ho*Wo, Kpad) fp16 with k = tap * C + c, tap = ky * kw + kx, zero
// padded; a 1-D convolution is the case H = 1, kh = 1.  Ho x Wo = (H / stride) x (W / stride); `pad` zero rows / columns
// precede the image along each axis the kernel extends over.  stride 1, pad = k / 2: the "same" convolution; stride 2,
// pad 0: diffusers Downsample2D(padding=0), i.e. zero padding on the right / bottom only.  VEC channels per access (8:
// 16-byte loads and stores, needs C % 8 == 0).
template <int VEC>
__global__ void im2col_kernel(const __half* __restrict__ in, int ldin, __half* __restrict__ A, int ldA, int H, int W, int C,
                              int kh, int kw, int stride, int pad, int Kpad, size_t total_vec) {
  using V = typename std::conditional<VEC == 8, uint4, __half>::type;
  const int Ho = H / stride, Wo = W / stride;
  const int pad_y = kh > 1 ? pad : 0, pad_x = kw > 1 ? pad : 0;
  const int kvec = Kpad / VEC;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total_vec; i += (size_t)gridDim.x * blockDim.x) {
    const size_t row = i / kvec;
    const int k = (int)(i % kvec) * VEC;
    const int x = (int)(row % Wo), y = (int)((row / Wo) % Ho);
    const size_t n = row / ((size_t)Wo * Ho);
    V v{};
    if (k < kh * kw * C) {
      const int tap = k / C, c = k % C;
      const int yy = y * stride + tap / kw - pad_y, xx = x * stride + tap % kw - pad_x;
      if (yy >= 0 && yy < H && xx >= 0 && xx < W) v = *reinterpret_cast<const V*>(in + ((n * H + yy) * W + xx) * ldin + c);
    }
    *reinterpret_cast<V*>(A + row * ldA + k) = v;
  }
}

__device__ __forceinline__ float act_fn(float y, int act) {
  if (act == 1) return y / (1.f + __expf(-y));                       // SiLU
  if (act == 2) return 0.5f * y * (1.f + erff(y * 0.70710678118f));   // exact (erf) GELU
  return y;
}

// GroupNorm helpers: one CTA per sample, blockDim == C, thread <-> channel, cpg = C / G channels per group.
// Sum of v over all threads of this thread's group (lane / warp: of this thread); s_part: 32 floats of shared memory.
__device__ __forceinline__ float group_reduce(float v, int cpg, float* s_part, int lane, int warp) {
  if (cpg <= 32) {
    for (int o = cpg >> 1; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
  }
  // G == 1 (or groups spanning several warps with G small): block-wide reduction, groups are warp aligned
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  if (lane == 0) s_part[warp] = v;
  __syncthreads();
  const int wpg = cpg >> 5;                      // warps per group
  float t = 0.f;
  const int w0 = (warp / wpg) * wpg;
  for (int w = 0; w < wpg; ++w) t += s_part[w0 + w];
  return t;
}
// output of channel c at position `row` (= n * P + p): act(v * ga + be) (+ resid) as fp32 and / or [hi | lo] fp16
__device__ __forceinline__ void gn_store(float v, float ga, float be, int act, const float* resid, float* out32,
                                         __half* out16, size_t row, int C, int c) {
  float y = act_fn(v * ga + be, act);
  const size_t o = row * C + c;
  if (resid) y += resid[o];
  if (out32) out32[o] = y;
  if (out16) store_hl(out16 + row * 2 * C + c, C, y);
}

// GroupNorm over (P positions x C/G channels) per sample and group, then activation, then optional residual add.
// x (N, P, C) fp32 (pitch ldx per position).
__global__ void groupnorm_kernel(const float* __restrict__ x, int ldx, int P, int C, int G, float eps,
                                 const float* __restrict__ gamma, const float* __restrict__ beta, int act,
                                 const float* __restrict__ resid, float* __restrict__ out32, __half* __restrict__ out16) {
  __shared__ float s_part[32];
  const int n = blockIdx.x, c = threadIdx.x, lane = c & 31, warp = c >> 5;
  const int cpg = C / G;
  const float* xs = x + (size_t)n * P * ldx;
  const float cnt = (float)P * cpg;
  float s = 0.f;
  for (int p = 0; p < P; ++p) s += xs[(size_t)p * ldx + c];
  const float mean = group_reduce(s, cpg, s_part, lane, warp) / cnt;
  float q = 0.f;
  for (int p = 0; p < P; ++p) {
    const float d = xs[(size_t)p * ldx + c] - mean;
    q += d * d;
  }
  const float rstd = rsqrtf(group_reduce(q, cpg, s_part, lane, warp) / cnt + eps);
  const float ga = gamma[c] * rstd, be = beta[c] - mean * gamma[c] * rstd;
  for (int p = 0; p < P; ++p) gn_store(xs[(size_t)p * ldx + c], ga, be, act, resid, out32, out16, (size_t)n * P + p, C, c);
}

// Same for P <= 64 positions (every 1-D stage, the 4x4 / 8x8 2-D stages): the thread's P values stay in registers, so the
// activation is read once instead of three times (this kernel was 30 % of the edge decoder).
template <int P>
__global__ void groupnorm_regs_kernel(const float* __restrict__ x, int ldx, int C, int G, float eps,
                                      const float* __restrict__ gamma, const float* __restrict__ beta, int act,
                                      const float* __restrict__ resid, float* __restrict__ out32, __half* __restrict__ out16) {
  __shared__ float s_part[32];
  const int n = blockIdx.x, c = threadIdx.x, lane = c & 31, warp = c >> 5;
  const int cpg = C / G;
  const float* xs = x + (size_t)n * P * ldx;
  const float cnt = (float)P * cpg;
  float v[P];
  float s = 0.f;
#pragma unroll
  for (int p = 0; p < P; ++p) {
    v[p] = xs[(size_t)p * ldx + c];
    s += v[p];
  }
  const float mean = group_reduce(s, cpg, s_part, lane, warp) / cnt;
  float q = 0.f;
#pragma unroll
  for (int p = 0; p < P; ++p) {
    const float d = v[p] - mean;
    q += d * d;
  }
  const float rstd = rsqrtf(group_reduce(q, cpg, s_part, lane, warp) / cnt + eps);
  const float ga = gamma[c] * rstd, be = beta[c] - mean * gamma[c] * rstd;
#pragma unroll
  for (int p = 0; p < P; ++p) gn_store(v[p], ga, be, act, resid, out32, out16, (size_t)n * P + p, C, c);
}

// small multi-head attention: qkv (N*T, 3*C) fp16 [q | k | v], out (N*T, C) fp16; heads Hh x dh = C; T*T*Hh <= 256
__global__ void __launch_bounds__(256) small_attention_kernel(const __half* __restrict__ qkv, __half* __restrict__ out, int T,
                                                              int Hh, int dh, float scale) {
  extern __shared__ float sm[];          // q,k,v: 3 * T * C floats, then scores Hh*T*T
  const int C = Hh * dh, n = blockIdx.x;
  float* sq = sm;
  float* sk = sq + T * C;
  float* sv = sk + T * C;
  float* sp = sv + T * C;
  for (int i = threadIdx.x; i < T * 3 * C; i += blockDim.x) {
    const int t = i / (3 * C), j = i % (3 * C);
    const float v = __half2float(qkv[((size_t)n * T + t) * 3 * C + j]);
    (j < C ? sq : j < 2 * C ? sk : sv)[t * C + (j % C)] = v;
  }
  __syncthreads();
  const int ns = Hh * T * T;
  if ((int)threadIdx.x < ns) {
    const int h = threadIdx.x / (T * T), i = (threadIdx.x / T) % T, j = threadIdx.x % T;
    float acc = 0.f;
    for (int d = 0; d < dh; ++d) acc = fmaf(sq[i * C + h * dh + d], sk[j * C + h * dh + d], acc);
    sp[threadIdx.x] = acc * scale;
  }
  __syncthreads();
  if ((int)threadIdx.x < Hh * T) {       // softmax over j for row (h, i)
    float* row = sp + threadIdx.x * T;
    float m = row[0];
    for (int j = 1; j < T; ++j) m = fmaxf(m, row[j]);
    float s = 0.f;
    for (int j = 0; j < T; ++j) { row[j] = __expf(row[j] - m); s += row[j]; }
    const float inv = 1.f / s;
    for (int j = 0; j < T; ++j) row[j] *= inv;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < T * C; i += blockDim.x) {
    const int t = i / C, c = i % C, h = c / dh;
    float acc = 0.f;
    for (int j = 0; j < T; ++j) acc = fmaf(sp[(h * T + t) * T + j], sv[j * C + c], acc);
    store_hl(out + ((size_t)n * T + t) * 2 * C + c, C, acc);
  }
}

// diffusers Upsample1d("cubic"): reflect pad 2, depthwise conv_transpose1d(stride 2, padding 7).  x (N,L,C) -> (N,2L,C)
__global__ void cubic_up1d_kernel(const float* __restrict__ x, float* __restrict__ y, int L, int C, const float* __restrict__ kern,
                                  size_t total) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const int o = (int)((i / C) % (2 * L));
    const size_t n = i / ((size_t)C * 2 * L);
    float acc = 0.f;
    // y[o] = sum_i xp[i] * k[o + 7 - 2 i],  xp = reflect-padded x (length L + 4)
    for (int ii = 0; ii < L + 4; ++ii) {
      const int kk = o + 7 - 2 * ii;
      if (kk < 0 || kk >= 8) continue;
      int src = ii - 2;
      if (src < 0) src = -src;
      if (src >= L) src = 2 * (L - 1) - src;
      acc = fmaf(x[(n * L + src) * C + c], kern[kk], acc);
    }
    y[i] = acc;
  }
}

// diffusers Downsample1d("cubic"): reflect pad 3, depthwise conv1d stride 2.  x (N,L,C) -> (N,L/2,C)
__global__ void cubic_down1d_kernel(const float* __restrict__ x, float* __restrict__ y, int L, int C, const float* __restrict__ kern,
                                    size_t total) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const int o = (int)((i / C) % (L / 2));
    const size_t n = i / ((size_t)C * (L / 2));
    float acc = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      int src = 2 * o + k - 3;
      if (src < 0) src = -src;
      if (src >= L) src = 2 * (L - 1) - src;
      acc = fmaf(x[(n * L + src) * C + c], kern[k], acc);
    }
    y[i] = acc;
  }
}

// encoder tail: h (N*P, ld) fp32 holds the 6 moment channels of conv_out; mode = first 3 channels of quant_conv(h).
// out (N, 3, P) fp32
__global__ void quant_mode_kernel(const float* __restrict__ h, int ld, const float* __restrict__ wq, const float* __restrict__ bq,
                                  float* __restrict__ out, int N, int P) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N * 3 * P) return;
  const int p = i % P, co = (i / P) % 3, n = i / (3 * P);
  const float* hr = h + ((size_t)n * P + p) * ld;
  float acc = bq[co];
#pragma unroll
  for (int ci = 0; ci < 6; ++ci) acc = fmaf(wq[co * 6 + ci], hr[ci], acc);
  out[i] = acc;
}

// Posterior of the encoders' latent: diffusers DiagonalGaussianDistribution over quant_conv(encoder(x)).  One warp per
// sample, lane <-> latent position (p = lane, lane + 32, ...).  The six moment channels are computed here from the conv_out
// rows h (N*P, pitch ld) by quant_conv when wq != null -- the fmaf order of quant_mode_kernel, so the mean half is
// bit-identical to the mode bg_vae_encode writes -- or read from mom_in (N, 6, P).  Outputs, each optional:
//   moments (N, 6, P) raw, diffusers' channel order: mean = channels 0-2, logvar = 3-5
//   z (N, 3, P) = mean + exp(0.5 clamp(logvar, -30, 20)) * noise, noise (N, 3, P); noise == null: z = mean
//   kl (N) = 0.5 sum_{c,p} (mean^2 + var - 1 - logvar), var = exp(clamped logvar): lane partials, then a fixed xor tree
// deterministic != 0: std = var = 0, so z = mean and kl = 0 (diffusers' kl() returns 0 for a deterministic posterior).
__global__ void posterior_kernel(const float* __restrict__ h, int ld, const float* __restrict__ wq, const float* __restrict__ bq,
                                 const float* __restrict__ mom_in, const float* __restrict__ noise, int N, int P,
                                 int deterministic, float* __restrict__ moments, float* __restrict__ z, float* __restrict__ kl) {
  const int n = (int)((blockIdx.x * (size_t)blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (n >= N) return;                      // whole warps: blockDim is a multiple of 32
  float part = 0.f;
  for (int p = lane; p < P; p += 32) {
    float m[6];
    if (wq) {
      const float* hr = h + ((size_t)n * P + p) * ld;
#pragma unroll
      for (int co = 0; co < 6; ++co) {
        float acc = bq[co];
#pragma unroll
        for (int ci = 0; ci < 6; ++ci) acc = fmaf(wq[co * 6 + ci], hr[ci], acc);
        m[co] = acc;
      }
    } else {
#pragma unroll
      for (int co = 0; co < 6; ++co) m[co] = mom_in[((size_t)n * 6 + co) * P + p];
    }
    if (moments) {
#pragma unroll
      for (int co = 0; co < 6; ++co) moments[((size_t)n * 6 + co) * P + p] = m[co];
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float logvar = fminf(fmaxf(m[3 + c], -30.f), 20.f);
      const float sd = deterministic ? 0.f : expf(0.5f * logvar), var = deterministic ? 0.f : expf(logvar);
      const size_t o = ((size_t)n * 3 + c) * P + p;
      if (z) z[o] = noise ? fmaf(sd, noise[o], m[c]) : m[c];
      part += m[c] * m[c] + var - 1.f - logvar;
    }
  }
  if (!kl) return;
  for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
  if (lane == 0) kl[n] = deterministic ? 0.f : 0.5f * part;
}

// per-sample reconstruction error: mse[n] = mean over the cnt values of sample n of (a - b)^2.  One 256-thread CTA per
// sample: strided fp32 partial sums, a fixed shuffle tree per warp, then the 8 warp sums in order (no atomics).
__global__ void __launch_bounds__(256) sample_mse_kernel(const float* __restrict__ a, const float* __restrict__ b, int cnt,
                                                         float* __restrict__ mse) {
  __shared__ float s_part[8];
  const size_t base = (size_t)blockIdx.x * cnt;
  float s = 0.f;
  for (int i = threadIdx.x; i < cnt; i += 256) {
    const float d = a[base + i] - b[base + i];
    s = fmaf(d, d, s);
  }
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) s_part[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int w = 0; w < 8; ++w) t += s_part[w];
    mse[blockIdx.x] = t / (float)cnt;
  }
}

// conv_out result (N*P, ld) fp32 -> out (N, 3, P) fp32 (first three channels)
__global__ void slice_out_kernel(const float* __restrict__ h, int ld, float* __restrict__ out, int N, int P) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N * 3 * P) return;
  const int p = i % P, co = (i / P) % 3, n = i / (3 * P);
  out[i] = h[((size_t)n * P + p) * ld + co];
}

inline unsigned grid_for(size_t work, int bs = 256) {
  size_t blocks = (work + bs - 1) / bs;
  const size_t cap = (size_t)num_sms() * 32;
  return (unsigned)(blocks < 1 ? 1 : (blocks > cap ? cap : blocks));
}

struct Conv {      // packed convolution / linear:  out[rows, cout_pad] = A[rows, kpad] * w^T + bias
  __half* w = nullptr;
  float* bias = nullptr;
  int cin = 0, cout = 0, taps = 1, kpad = 0, cout_pad = 0;
};
struct Norm {
  float *g = nullptr, *b = nullptr;
};
struct Res2d {
  Norm n1, n2;
  Conv c1, c2, sc;
  bool has_sc = false;
};
struct Res1d {
  Conv c1, c2, skip;
  Norm n1, n2;
  bool has_skip = false;
};
struct Attn {
  Norm gn;
  Conv qkv, proj;
};

}  // namespace
}  // namespace bg

using namespace bg;

struct BgVae {
  int kind = 0;                 // 0 surface decoder, 1 edge decoder, 2 surface encoder, 3 edge encoder
  int terms = 3;                // product terms of the compensated GEMMs (bg_vae_create)
  int implicit = 1;             // convolutions as implicit GEMMs; BREPGEN_B200_VAE_IM2COL=1 at creation: explicit gather (A/B)
  char* arena = nullptr;
  size_t arena_bytes = 0;
  float *pq_w = nullptr, *pq_b = nullptr, *up_kernel = nullptr;
  Conv conv_in, conv_out;
  Norm norm_out;
  // surface
  Res2d s_mid[2];
  Attn s_attn;
  Res2d s_up[4][3];
  Conv s_upconv[3];
  // edge
  Res1d e_mid[6];
  Attn e_attn[6];
  Res1d e_up[3][3];
  // encoders (kind 2 surface, 3 edge): conv_in / conv_out / norm_out / mid blocks reuse the members above
  Res2d s_down[4][2];
  Conv s_downconv[3];
  Res1d e_down[3][3];
  float *q_w = nullptr, *q_b = nullptr, *down_kernel = nullptr;
};

namespace {

struct VPacker : Packer {
  int terms;
  VPacker(const BgNamedTensor* weights, int n, void* stream, int terms_) : Packer(weights, n, stream), terms(terms_) {}

  Norm norm(const std::string& name, int c) {
    Norm n;
    n.g = copy_f32(name + ".weight", c);
    n.b = copy_f32(name + ".bias", c);
    return n;
  }
  // weights [cout][cin][taps] fp32 at w -> the [cout_pad][3 * kpad] operand at dst
  void pack(const float* w, __half* dst, int cout, int cin, int taps, int kpad, int cout_pad) {
    if (dry || !w || err) return;
    const size_t tot = (size_t)cout_pad * kpad;
    pack_conv_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, st>>>(w, dst, cout, cin, taps, kpad, cout_pad, terms);
    err = check_launch("pack_conv_kernel launch");
  }
  Conv conv(const std::string& name, int cout, int cin, int taps, bool bias = true, int cout_pad = 0) {
    Conv c;
    c.cin = cin; c.cout = cout; c.taps = taps;
    c.kpad = round64(cin * taps);
    c.cout_pad = cout_pad ? cout_pad : cout;
    const float* w = find(name + ".weight", (int64_t)cout * cin * taps);
    c.w = take<__half>((size_t)c.cout_pad * 3 * c.kpad);
    pack(w, c.w, cout, cin, taps, c.kpad, c.cout_pad);
    if (bias) {
      if (c.cout_pad == cout) {
        c.bias = copy_f32(name + ".bias", cout);
      } else {
        const float* b = find(name + ".bias", cout);
        c.bias = zeros(c.cout_pad);
        if (!dry && b && !err) err = check_cuda(cudaMemcpyAsync(c.bias, b, cout * 4, cudaMemcpyDeviceToDevice, st), "copy");
      }
    }
    return c;
  }
  // diffusers ResnetBlock2D without time embedding
  Res2d res2d(const std::string& n, int cin, int cout) {
    Res2d r;
    r.n1 = norm(n + ".norm1", cin);
    r.c1 = conv(n + ".conv1", cout, cin, 9);
    r.n2 = norm(n + ".norm2", cout);
    r.c2 = conv(n + ".conv2", cout, cout, 9);
    r.has_sc = cin != cout;
    if (r.has_sc) r.sc = conv(n + ".conv_shortcut", cout, cin, 1);
    return r;
  }
  // diffusers ResConvBlock (1-D)
  Res1d res1d(const std::string& n, int cin, int cmid, int cout) {
    Res1d r;
    r.has_skip = cin != cout;
    if (r.has_skip) r.skip = conv(n + ".conv_skip", cout, cin, 1, false);
    r.c1 = conv(n + ".conv_1", cmid, cin, 5);
    r.n1 = norm(n + ".group_norm_1", cmid);
    r.c2 = conv(n + ".conv_2", cout, cmid, 5);
    r.n2 = norm(n + ".group_norm_2", cout);
    return r;
  }
  // attention block over 512 channels: group norm, then q | k | v (C -> C linears) as rows [0, C), [C, 2C), [2C, 3C) of
  // one [3C][C] operand, then the output projection.  2-D: diffusers Attention (to_q / to_k / to_v / to_out.0); 1-D: the
  // mid block's SelfAttention1d (query / key / value / proj_attn)
  Attn attn_block(const std::string& a, bool two_d) {
    static const char* const names_2d[4] = {"to_q", "to_k", "to_v", "to_out.0"};
    static const char* const names_1d[4] = {"query", "key", "value", "proj_attn"};
    const char* const* names = two_d ? names_2d : names_1d;
    const int C = 512;
    Attn r;
    r.gn = norm(a + ".group_norm", C);
    Conv& c = r.qkv;
    c.cin = C; c.cout = 3 * C; c.taps = 1; c.kpad = C; c.cout_pad = 3 * C;
    c.w = take<__half>((size_t)3 * C * 3 * C);
    c.bias = take<float>(3 * C);
    for (int i = 0; i < 3; ++i) {
      const float* w = find(a + "." + names[i] + ".weight", (int64_t)C * C);
      const float* b = find(a + "." + names[i] + ".bias", C);
      pack(w, c.w + (size_t)i * C * 3 * C, C, C, 1, C, C);
      if (!dry && b && !err) err = check_cuda(cudaMemcpyAsync(c.bias + i * C, b, C * 4, cudaMemcpyDeviceToDevice, st), "copy");
    }
    r.proj = conv(a + "." + names[3], C, C, 1);
    return r;
  }
};

// UNetMidBlock2D (resnet, attention, resnet) or UNetMidBlock1D (6 resnets, 6 attentions) under prefix p
void pack_mid(BgVae* m, VPacker& pk, const std::string& p, bool two_d) {
  if (two_d) {
    m->s_mid[0] = pk.res2d(p + "mid_block.resnets.0", 512, 512);
    m->s_attn = pk.attn_block(p + "mid_block.attentions.0", true);
    m->s_mid[1] = pk.res2d(p + "mid_block.resnets.1", 512, 512);
    return;
  }
  for (int i = 0; i < 6; ++i) m->e_mid[i] = pk.res1d(p + "mid_block.resnets." + std::to_string(i), 512, 512, 512);
  for (int i = 0; i < 6; ++i) m->e_attn[i] = pk.attn_block(p + "mid_block.attentions." + std::to_string(i), false);
}

int pack_decoder(BgVae* m, VPacker& pk) {
  const std::string d = "decoder.";
  const bool surf = m->kind == 0;
  m->pq_w = pk.copy_f32("post_quant_conv.weight", 9);
  m->pq_b = pk.copy_f32("post_quant_conv.bias", 3);
  m->conv_in = pk.conv(d + "conv_in", 512, 3, surf ? 9 : 3);
  pack_mid(m, pk, d, surf);
  if (surf) {
    const int chans[4][2] = {{512, 512}, {512, 512}, {512, 256}, {256, 128}};
    for (int i = 0; i < 4; ++i) {
      for (int j = 0; j < 3; ++j)
        m->s_up[i][j] = pk.res2d(d + "up_blocks." + std::to_string(i) + ".resnets." + std::to_string(j),
                                 j == 0 ? chans[i][0] : chans[i][1], chans[i][1]);
      if (i < 3) m->s_upconv[i] = pk.conv(d + "up_blocks." + std::to_string(i) + ".upsamplers.0.conv", chans[i][1], chans[i][1], 9);
    }
  } else {
    const int chans[3][2] = {{512, 512}, {512, 256}, {256, 128}};
    for (int i = 0; i < 3; ++i) {
      const std::string b = d + "up_blocks." + std::to_string(i);
      m->e_up[i][0] = pk.res1d(b + ".resnets.0", chans[i][0], chans[i][0], chans[i][0]);
      m->e_up[i][1] = pk.res1d(b + ".resnets.1", chans[i][0], chans[i][0], chans[i][0]);
      m->e_up[i][2] = pk.res1d(b + ".resnets.2", chans[i][0], chans[i][0], chans[i][1]);
    }
    m->up_kernel = pk.copy_f32(d + "up_blocks.0.up.kernel", 8);   // the same fixed 8-tap buffer in all three blocks
  }
  m->norm_out = pk.norm(d + "conv_norm_out", 128);
  m->conv_out = pk.conv(d + "conv_out", 3, 128, surf ? 9 : 3, true, 128);
  return pk.err;
}

int pack_encoder(BgVae* m, VPacker& pk) {
  const std::string e = "encoder.";
  const bool surf = m->kind == 2;
  // the "post-quant" slot holds the identity: the input image goes through the same fp32 -> [hi | lo] fp16 kernel
  m->pq_w = pk.zeros(9);
  m->pq_b = pk.zeros(3);
  if (!pk.dry && !pk.err) {
    const float ident[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
    pk.err = check_cuda(cudaMemcpyAsync(m->pq_w, ident, sizeof(ident), cudaMemcpyHostToDevice, pk.st), "copy identity");
    if (!pk.err) pk.err = check_cuda(cudaStreamSynchronize(pk.st), "sync");   // `ident` lives on this stack frame
  }
  m->conv_in = pk.conv(e + "conv_in", 128, 3, surf ? 9 : 3);
  if (surf) {
    const int chans[4][2] = {{128, 128}, {128, 256}, {256, 512}, {512, 512}};
    for (int i = 0; i < 4; ++i) {
      for (int j = 0; j < 2; ++j)
        m->s_down[i][j] = pk.res2d(e + "down_blocks." + std::to_string(i) + ".resnets." + std::to_string(j),
                                   j == 0 ? chans[i][0] : chans[i][1], chans[i][1]);
      if (i < 3) m->s_downconv[i] = pk.conv(e + "down_blocks." + std::to_string(i) + ".downsamplers.0.conv", chans[i][1], chans[i][1], 9);
    }
  } else {
    const int chans[3][2] = {{128, 128}, {128, 256}, {256, 512}};
    for (int i = 0; i < 3; ++i) {
      const std::string b = e + "down_blocks." + std::to_string(i);
      m->e_down[i][0] = pk.res1d(b + ".resnets.0", chans[i][0], chans[i][1], chans[i][1]);
      m->e_down[i][1] = pk.res1d(b + ".resnets.1", chans[i][1], chans[i][1], chans[i][1]);
      m->e_down[i][2] = pk.res1d(b + ".resnets.2", chans[i][1], chans[i][1], chans[i][1]);
    }
    m->down_kernel = pk.copy_f32(e + "down_blocks.0.down.kernel", 8);
  }
  pack_mid(m, pk, e, surf);
  m->norm_out = pk.norm(e + "conv_norm_out", 512);
  m->conv_out = pk.conv(e + "conv_out", 6, 512, surf ? 9 : 3, true, 128);
  m->q_w = pk.copy_f32("quant_conv.weight", 36);
  m->q_b = pk.copy_f32("quant_conv.bias", 6);
  return pk.err;
}

// per-sample buffer sizes (elements)
struct VaeWs {
  float *X, *H, *S;        // fp32 activations
  __half *T, *A, *Q;       // fp16: normalised / cast activations, im2col matrix, qkv + attention output
  size_t bytes;
};
VaeWs carve_vae(char* base, int kind, size_t N) {
  // maxima over the layer list (positions x channels per sample) at the largest supported extent (32 x 32 / 32 points)
  const bool two_d = (kind & 1) == 0;
  const size_t act = two_d ? 32 * 32 * 256 : 32 * 256;                    // largest activation (elements)
  const size_t col = two_d ? (size_t)32 * 32 * 9 * 256 : (size_t)16 * 5 * 512;   // largest im2col row block
  const size_t qkv = two_d ? 16 * 2560 : 4 * 2560;                        // qkv (3C) + attention out (2C, hi | lo)
  size_t off = 0;
  auto take = [&](size_t bytes) {
    char* p = base ? base + off : nullptr;
    off += align_up(bytes, 1024);
    return p;
  };
  VaeWs w;
  w.X = reinterpret_cast<float*>(take(N * act * 4));
  w.H = reinterpret_cast<float*>(take(N * act * 4));
  w.S = reinterpret_cast<float*>(take(N * act * 4));
  w.T = reinterpret_cast<__half*>(take(N * act * 2 * 2));       // [hi | lo]
  w.A = reinterpret_cast<__half*>(take(N * col * 2 * 2));       // [A_hi | A_lo]
  w.Q = reinterpret_cast<__half*>(take(N * qkv * 2));
  w.bytes = off;
  return w;
}

// the encoders' posterior tail (bg_vae_encode_moments / bg_vae_reconstruct): posterior_kernel's inputs and outputs, written
// in place of the mode
struct Tail {
  const float* noise = nullptr;
  float *moments = nullptr, *z = nullptr, *kl = nullptr;
};

struct Ctx {
  cudaStream_t st;
  size_t N;
  VaeWs w;
  int terms = 3;
  int implicit = 1;
  const Tail* tail = nullptr;   // encoders: the posterior tail instead of the mode
};

// out = A * cv^T + bias (+ resid).  A is [rows][2 * cv.kpad] fp16 = [A_hi | A_lo] read cyclically along K:
//   3 terms: [A_hi | A_lo | A_hi] x [W_hi | W_hi | W_lo];  2 terms: [A_hi | A_hi] x [W_hi | W_lo] (the lo plane of A is not read)
// or, with geom.taps > 0, the [hi | lo] image (pitch 2 * cv.cin) of an implicit convolution.
int gemm(const Ctx& c, const __half* A, const Conv& cv, size_t rows, float* out32, __half* out16, const float* resid,
         const ConvGeom& geom = ConvGeom()) {
  GemmEpilogue ep;
  ep.out = out16 ? (void*)out16 : (void*)out32;
  ep.out_f16 = out16 ? 1 : 0;
  ep.ldo = cv.cout_pad;
  ep.bias = cv.bias;
  ep.resid = resid;
  ep.ldr = cv.cout_pad;
  ep.conv = geom;
  int lda = 2 * cv.cin;
  if (!geom.taps) {
    lda = 2 * cv.kpad;
    ep.a_kwrap = (c.terms - 1) * cv.kpad;
  }
  return launch_gemm_f16(c.st, A, lda, cv.w, 3 * cv.kpad, (int)rows, cv.cout_pad, c.terms * cv.kpad, ep);
}
// shapes the implicit convolution covers: a 128-row tile of output pixels must be a box {W, box_h, box_n} of whole image rows
bool conv_implicit_ok(int H, int W, int C) {
  const int hw = H * W;
  return C % 64 == 0 && W <= 128 && 128 % W == 0 && (hw % 128 == 0 || 128 % hw == 0);
}
// explicit gather of one fp16 plane (pitch ldin) of N images into the kh x kw im2col matrix A (pitch ldA, Kpad columns)
int im2col(const Ctx& c, const __half* in, int ldin, __half* A, int ldA, int H, int W, int C, int kh, int kw, int stride,
           int Kpad) {
  const size_t rows = c.N * (size_t)(H / stride) * (W / stride);
  const bool v8 = C % 8 == 0;
  const auto kernel = v8 ? im2col_kernel<8> : im2col_kernel<1>;
  const size_t tot = rows * (Kpad / (v8 ? 8 : 1));
  kernel<<<grid_for(tot), 256, 0, c.st>>>(in, ldin, A, ldA, H, W, C, kh, kw, stride, stride == 1 ? kw / 2 : 0, Kpad, tot);
  return check_launch("im2col_kernel launch");
}
// kh x kw convolution (kh * kw = cv.taps; 1-D: H = 1, kh = 1) of the [hi | lo] fp16 image `in` (N, H, W, 2 * cv.cin) into
// fp32 (N, H / stride, W / stride, cv.cout_pad).  stride 1: "same" zero padding, an implicit GEMM where the shape allows;
// stride 2: diffusers Downsample2D(padding=0).  Otherwise the explicit im2col gather into the workspace, then a GEMM.
int conv(const Ctx& c, const __half* in, int H, int W, int kw, int stride, const Conv& cv, float* out32, const float* resid) {
  const size_t rows = c.N * (size_t)(H / stride) * (W / stride);
  if (c.implicit && stride == 1 && conv_implicit_ok(H, W, cv.cin)) {
    ConvGeom g;
    g.taps = cv.taps; g.kw = kw; g.C = cv.cin; g.W = W; g.H = H; g.N = (int)c.N;
    g.lo_plane = 1; g.terms = c.terms;
    return gemm(c, in, cv, rows, out32, nullptr, resid, g);
  }
  for (int part = 0; part < c.terms - 1; ++part)     // hi plane, then (3-term mode) lo plane of the [hi | lo] activation
    BG_TRY(im2col(c, in + part * cv.cin, 2 * cv.cin, c.w.A + part * cv.kpad, 2 * cv.kpad, H, W, cv.cin, cv.taps / kw, kw,
                  stride, cv.kpad));
  return gemm(c, c.w.A, cv, rows, out32, nullptr, resid);
}
int groupnorm(const Ctx& c, const float* x, int P, int C, int G, float eps, const Norm& n, int act, const float* resid,
              float* out32, __half* out16) {
  switch (P) {
#define BG_GN_CASE(PP)                                                                                                   \
    case PP:                                                                                                             \
      groupnorm_regs_kernel<PP><<<(unsigned)c.N, C, 0, c.st>>>(x, C, C, G, eps, n.g, n.b, act, resid, out32, out16);     \
      break;
    BG_GN_CASE(4) BG_GN_CASE(8) BG_GN_CASE(16) BG_GN_CASE(32) BG_GN_CASE(64)
#undef BG_GN_CASE
    default:
      groupnorm_kernel<<<(unsigned)c.N, C, 0, c.st>>>(x, C, P, C, G, eps, n.g, n.b, act, resid, out32, out16);
  }
  return check_launch("groupnorm_kernel launch");
}
int cast_split(const Ctx& c, const float* x, __half* y, int C, size_t rows) {
  const size_t tot = rows * C;
  cast_split_kernel<<<grid_for(tot), 256, 0, c.st>>>(x, y, C, tot);
  return check_launch("cast_split_kernel launch");
}
// softmax(q k^T * scale) v over the T positions of each sample, 512 channels in Hh heads: qkv (N*T, 3C) fp16 ->
// out (N*T, [C hi | C lo]) fp16
int small_attention(const Ctx& c, const __half* qkv, __half* out, int T, int Hh, float scale) {
  const int C = 512, dh = C / Hh;
  const size_t smem = (size_t)(3 * T * C + Hh * T * T) * 4;
  BG_TRY(ensure_dynamic_smem(reinterpret_cast<const void*>(&small_attention_kernel), 112 * 1024));
  small_attention_kernel<<<(unsigned)c.N, 256, smem, c.st>>>(qkv, out, T, Hh, dh, scale);
  return check_launch("small_attention_kernel launch");
}
// attention block with residual over the T positions of each sample, 512 channels in Hh heads:
// x += proj(attention(qkv(GroupNorm(x))))
int attention(const Ctx& c, const Attn& a, float* x, int T, int G, float eps, int Hh, float scale) {
  const int C = 512;
  BG_TRY(groupnorm(c, x, T, C, G, eps, a.gn, 0, nullptr, nullptr, c.w.T));
  BG_TRY(gemm(c, c.w.T, a.qkv, c.N * T, nullptr, c.w.Q, nullptr));
  __half* o = c.w.Q + c.N * (size_t)T * 3 * C;   // [N*T][2C]
  BG_TRY(small_attention(c, c.w.Q, o, T, Hh, scale));
  return gemm(c, o, a.proj, c.N * T, x, nullptr, x);
}
// nearest-2x upsampling of x (N, H, W, C) fp32 into the [hi | lo] fp16 image y (N, 2H, 2W, 2C)
int upsample2x_split(const Ctx& c, const float* x, __half* y, int H, int W, int C) {
  const size_t tot = c.N * (size_t)4 * H * W * C;
  upsample2x_split_kernel<<<grid_for(tot), 256, 0, c.st>>>(x, y, H, W, C, tot);
  return check_launch("upsample2x_split_kernel launch");
}
// cubic 2x resampling along L of x (N, L, C) fp32: up -> y (N, 2L, C), else -> y (N, L / 2, C)
int cubic1d(const Ctx& c, const float* x, float* y, int L, int C, const float* kern, bool up) {
  if (up) {
    const size_t tot = c.N * (size_t)2 * L * C;
    cubic_up1d_kernel<<<grid_for(tot), 256, 0, c.st>>>(x, y, L, C, kern, tot);
    return check_launch("cubic_up1d_kernel launch");
  }
  const size_t tot = c.N * (size_t)(L / 2) * C;
  cubic_down1d_kernel<<<grid_for(tot), 256, 0, c.st>>>(x, y, L, C, kern, tot);
  return check_launch("cubic_down1d_kernel launch");
}
// z (N, 3, P) fp32 -> y (N, P, [3 hi | 3 lo]) fp16, y = W z + b (post_quant_conv; the identity for the encoders)
int postquant(const Ctx& c, const float* z, const float* w, const float* b, __half* y, int P) {
  const int N = (int)c.N;
  postquant_kernel<<<(N * P + 255) / 256, 256, 0, c.st>>>(z, w, b, y, N, P);
  return check_launch("postquant_kernel launch");
}

// x (in place, fp32 [N, H*H, Cout] in *px): diffusers ResnetBlock2D without time embedding
int resnet2d(const Ctx& c, const Res2d& r, float** px, float** pfree, int H) {
  const int cin = r.c1.cin, cout = r.c1.cout, HW = H * H;
  float* x = *px;
  BG_TRY(groupnorm(c, x, HW, cin, 32, 1e-6f, r.n1, 1, nullptr, nullptr, c.w.T));
  BG_TRY(conv(c, c.w.T, H, H, 3, 1, r.c1, c.w.H, nullptr));
  if (!r.has_sc) {
    BG_TRY(groupnorm(c, c.w.H, HW, cout, 32, 1e-6f, r.n2, 1, nullptr, nullptr, c.w.T));
    return conv(c, c.w.T, H, H, 3, 1, r.c2, x, x);
  }
  // 1x1 shortcut on the raw input (T is free between the two convolutions), then conv2 accumulates onto it
  float* s = *pfree;
  BG_TRY(cast_split(c, x, c.w.T, cin, c.N * (size_t)HW));
  BG_TRY(gemm(c, c.w.T, r.sc, c.N * HW, s, nullptr, nullptr));
  BG_TRY(groupnorm(c, c.w.H, HW, cout, 32, 1e-6f, r.n2, 1, nullptr, nullptr, c.w.T));
  BG_TRY(conv(c, c.w.T, H, H, 3, 1, r.c2, s, s));
  *px = s;
  *pfree = x;
  return BG_OK;
}

int resconv1d(const Ctx& c, const Res1d& r, float** px, float** pfree, int L) {
  const int cin = r.c1.cin, cmid = r.c1.cout, cout = r.c2.cout;
  float* x = *px;
  BG_TRY(cast_split(c, x, c.w.T, cin, c.N * (size_t)L));
  const float* res = x;
  float* out = x;
  if (r.has_skip) {
    BG_TRY(gemm(c, c.w.T, r.skip, c.N * L, *pfree, nullptr, nullptr));
    res = *pfree;
    out = *pfree;
  }
  BG_TRY(conv(c, c.w.T, 1, L, 5, 1, r.c1, c.w.H, nullptr));
  BG_TRY(groupnorm(c, c.w.H, L, cmid, 1, 1e-5f, r.n1, 2, nullptr, nullptr, c.w.T));
  BG_TRY(conv(c, c.w.T, 1, L, 5, 1, r.c2, c.w.H, nullptr));
  BG_TRY(groupnorm(c, c.w.H, L, cout, 1, 1e-5f, r.n2, 2, res, out, nullptr));
  if (r.has_skip) {
    *px = out;
    *pfree = x;
  }
  return BG_OK;
}

// UNetMidBlock2D at H x H: resnet, single-head attention (legacy diffusers attention block), resnet
int mid2d(const Ctx& c, const BgVae* m, float** px, float** pfree, int H) {
  BG_TRY(resnet2d(c, m->s_mid[0], px, pfree, H));
  BG_TRY(attention(c, m->s_attn, *px, H * H, 32, 1e-6f, 1, 0.044194173824159216f));   // 1 / sqrt(512)
  return resnet2d(c, m->s_mid[1], px, pfree, H);
}
// UNetMidBlock1D at 4 positions: 6 x (ResConvBlock, 16-head attention)
int mid1d(const Ctx& c, const BgVae* m, float** px, float** pfree) {
  for (int i = 0; i < 6; ++i) {
    BG_TRY(resconv1d(c, m->e_mid[i], px, pfree, 4));
    BG_TRY(attention(c, m->e_attn[i], *px, 4, 1, 1e-5f, 16, 0.17677669529663687f));   // (1/sqrt(sqrt(32)))^2
  }
  return BG_OK;
}

// in (N, 3, H*W) fp32 -> 1x1 post_quant_conv (the identity for the encoders) into [hi | lo] fp16 -> conv_in -> x
int stem(const Ctx& c, const BgVae* m, const float* in, int H, int W, float* x) {
  BG_TRY(postquant(c, in, m->pq_w, m->pq_b, c.w.T, H * W));
  return conv(c, c.w.T, H, W, 3, 1, m->conv_in, x, nullptr);
}
// posterior_kernel over the N samples of c: moments from quant_conv(h) (wq != null) or from mom_in (N, 6, P)
int posterior(const Ctx& c, const float* h, int ld, const float* wq, const float* bq, const float* mom_in, const Tail& t,
              int P, int deterministic) {
  posterior_kernel<<<(unsigned)((c.N * 32 + 255) / 256), 256, 0, c.st>>>(h, ld, wq, bq, mom_in, t.noise, (int)c.N, P,
                                                                        deterministic, t.moments, t.z, t.kl);
  return check_launch("posterior_kernel launch");
}
int sample_mse(const Ctx& c, const float* a, const float* b, int cnt, float* mse) {
  sample_mse_kernel<<<(unsigned)c.N, 256, 0, c.st>>>(a, b, cnt, mse);
  return check_launch("sample_mse_kernel launch");
}

// x -> GroupNorm + SiLU -> conv_out -> out (N, 3, H*W) fp32: the first three channels (decoders) or the mode of
// quant_conv over the six moment channels (encoders; with c.tail, the posterior tail instead and `out` is not written)
int head(const Ctx& c, const BgVae* m, const float* x, int H, int W, float* out) {
  const int N = (int)c.N, P = H * W, ld = m->conv_out.cout_pad;
  BG_TRY(groupnorm(c, x, P, m->conv_out.cin, 32, 1e-6f, m->norm_out, 1, nullptr, nullptr, c.w.T));
  BG_TRY(conv(c, c.w.T, H, W, 3, 1, m->conv_out, c.w.H, nullptr));
  if (m->kind >= 2 && c.tail) return posterior(c, c.w.H, ld, m->q_w, m->q_b, nullptr, *c.tail, P, 0);
  if (m->kind >= 2) {
    quant_mode_kernel<<<(N * 3 * P + 255) / 256, 256, 0, c.st>>>(c.w.H, ld, m->q_w, m->q_b, out, N, P);
    return check_launch("quant_mode_kernel launch");
  }
  slice_out_kernel<<<(N * 3 * P + 255) / 256, 256, 0, c.st>>>(c.w.H, ld, out, N, P);
  return check_launch("slice_out_kernel launch");
}

// the whole network of handle m on N inputs of extent hw (latent side for the decoders, image side for the encoders)
int run_vae(const BgVae* m, const float* in, int N, int hw, float* out, void* workspace, size_t workspace_bytes,
            void* stream, const char* what, const Tail* tail = nullptr) {
  Ctx c;
  c.st = reinterpret_cast<cudaStream_t>(stream);
  c.N = (size_t)N;
  c.terms = m->terms;
  c.implicit = m->implicit;
  c.tail = tail;
  char* base;
  BG_TRY(align_workspace(workspace, workspace_bytes, carve_vae(nullptr, m->kind, c.N).bytes, what, &base));
  c.w = carve_vae(base, m->kind, c.N);
  float* x = c.w.X;
  float* spare = c.w.S;
  int H = hw, L = hw;

  switch (m->kind) {
    case 0:   // surface decoder
      BG_TRY(stem(c, m, in, H, H, x));
      BG_TRY(mid2d(c, m, &x, &spare, H));
      for (int i = 0; i < 4; ++i) {
        for (int j = 0; j < 3; ++j) BG_TRY(resnet2d(c, m->s_up[i][j], &x, &spare, H));
        if (i < 3) {   // nearest 2x into the [hi | lo] input of the upsampler's convolution
          const Conv& uc = m->s_upconv[i];
          BG_TRY(upsample2x_split(c, x, c.w.T, H, H, uc.cin));
          H *= 2;
          BG_TRY(conv(c, c.w.T, H, H, 3, 1, uc, spare, nullptr));
          std::swap(x, spare);
        }
      }
      return head(c, m, x, H, H, out);
    case 1:   // edge decoder
      BG_TRY(stem(c, m, in, 1, L, x));
      BG_TRY(mid1d(c, m, &x, &spare));
      for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j) BG_TRY(resconv1d(c, m->e_up[i][j], &x, &spare, L));
        BG_TRY(cubic1d(c, x, spare, L, m->e_up[i][2].c2.cout, m->up_kernel, true));
        std::swap(x, spare);
        L *= 2;
      }
      return head(c, m, x, 1, L, out);
    case 2:   // surface encoder
      BG_TRY(stem(c, m, in, H, H, x));
      for (int i = 0; i < 4; ++i) {
        for (int j = 0; j < 2; ++j) BG_TRY(resnet2d(c, m->s_down[i][j], &x, &spare, H));
        if (i < 3) {
          const Conv& dc = m->s_downconv[i];
          BG_TRY(cast_split(c, x, c.w.T, dc.cin, c.N * (size_t)H * H));
          BG_TRY(conv(c, c.w.T, H, H, 3, 2, dc, spare, nullptr));
          H /= 2;
          std::swap(x, spare);
        }
      }
      BG_TRY(mid2d(c, m, &x, &spare, H));
      return head(c, m, x, H, H, out);
    default:  // edge encoder
      BG_TRY(stem(c, m, in, 1, L, x));
      for (int i = 0; i < 3; ++i) {
        BG_TRY(cubic1d(c, x, spare, L, m->e_down[i][0].c1.cin, m->down_kernel, false));
        std::swap(x, spare);
        L /= 2;
        for (int j = 0; j < 3; ++j) BG_TRY(resconv1d(c, m->e_down[i][j], &x, &spare, L));
      }
      BG_TRY(mid1d(c, m, &x, &spare));
      return head(c, m, x, 1, L, out);
  }
}

// stream and sample count of a unit-level entry point (no workspace)
Ctx op_ctx(int N, void* stream) {
  Ctx c{};
  c.st = reinterpret_cast<cudaStream_t>(stream);
  c.N = (size_t)N;
  return c;
}

}  // namespace

extern "C" {

int bg_vae_create(int kind, const BgNamedTensor* weights, int n_weights, void* stream, BgVae** out) {
  return bg_vae_create_ex(kind, 0, weights, n_weights, stream, out);
}

int bg_vae_create_ex(int kind, int terms, const BgNamedTensor* weights, int n_weights, void* stream, BgVae** out) {
  BG_REQUIRE(kind >= 0 && kind <= 3 && (terms == 0 || terms == 2 || terms == 3) && weights && n_weights > 0 && out,
             "vae_create: bad arguments");
  BG_TRY(bg_check_device());
  BgVae* m = new BgVae();
  m->kind = kind;
  // Product terms of the compensated GEMMs:
  //   3: A_hi W_hi + A_lo W_hi + A_hi W_lo   (activations AND weights split)
  //   2: A_hi W_hi + A_hi W_lo               (weights split only: the systematic part of the fp16 error) -- 1/3 less GEMM work
  //                                           and no lo plane in the im2col matrices
  // Relative L2 errors against the fp32 oracle (bar 1e-3), measured on an H100 with 3 / 2 terms: surface decoder 9.4e-5 /
  // 1.3e-3, edge decoder 3.6e-5 / 4.1-4.3e-4, encoders <= 1.1e-4 / 6.4-9.0e-4.  So the edge decoder uses 2 terms (a third
  // less GEMM work); the surface decoder, over the bar with 2, and the encoders, close to it, keep 3.  terms != 0 overrides
  // the default: the full auto-encoders' edge decoder takes 3, since the two-term error depends on the weights and reaches
  // 1.1e-3 on some draws.
  m->terms = terms ? terms : (kind == 1 ? 2 : 3);
  if (const char* e = getenv("BREPGEN_B200_VAE_IM2COL")) m->implicit = atoi(e) ? 0 : 1;
  VPacker pk(weights, n_weights, stream, m->terms);
  const int s = pack_arena(pk, [&] { return kind >= 2 ? pack_encoder(m, pk) : pack_decoder(m, pk); }, &m->arena,
                           &m->arena_bytes);
  if (s != 0) {
    bg_vae_destroy(m);
    return s;
  }
  *out = m;
  return BG_OK;
}

void bg_vae_destroy(BgVae* m) {
  if (!m) return;
  if (m->arena) cudaFree(m->arena);
  delete m;
}

size_t bg_vae_workspace_bytes(const BgVae* m, int N) {
  if (!m || N <= 0) return 0;
  return carve_vae(nullptr, m->kind, (size_t)N).bytes + 1024;
}

int bg_vae_decode(BgVae* m, const float* z, int N, float* out, void* workspace, size_t workspace_bytes, void* stream) {
  return bg_vae_decode_hw(m, z, N, 4, out, workspace, workspace_bytes, stream);
}

int bg_vae_decode_hw(BgVae* m, const float* z, int N, int hw, float* out, void* workspace, size_t workspace_bytes, void* stream) {
  BG_REQUIRE(m && z && out && workspace && N > 0, "vae_decode: bad arguments");
  BG_REQUIRE(m->kind == 0 || m->kind == 1, "vae_decode: handle is not a decoder");
  BG_REQUIRE(m->kind == 0 ? (hw >= 1 && hw <= 4) : hw == 4, "vae_decode: latent extent must be 1..4 (surface) or 4 (edge)");
  return run_vae(m, z, N, hw, out, workspace, workspace_bytes, stream, "vae_decode");
}

int bg_vae_encode(BgVae* m, const float* xin, int N, int hw, float* out, void* workspace, size_t workspace_bytes, void* stream) {
  BG_REQUIRE(m && xin && out && workspace && N > 0, "vae_encode: bad arguments");
  BG_REQUIRE(m->kind == 2 || m->kind == 3, "vae_encode: handle is not an encoder");
  BG_REQUIRE(m->kind == 2 ? (hw == 8 || hw == 16 || hw == 24 || hw == 32) : hw == 32,
             "vae_encode: input extent must be 8/16/24/32 (surface) or 32 (edge)");
  return run_vae(m, xin, N, hw, out, workspace, workspace_bytes, stream, "vae_encode");
}

int bg_vae_encode_moments(BgVae* m, const float* xin, int N, int hw, float* moments, void* workspace, size_t workspace_bytes,
                          void* stream) {
  BG_REQUIRE(m && xin && moments && workspace && N > 0, "vae_encode_moments: bad arguments");
  BG_REQUIRE(m->kind == 2 || m->kind == 3, "vae_encode_moments: handle is not an encoder");
  BG_REQUIRE(m->kind == 2 ? (hw == 8 || hw == 16 || hw == 24 || hw == 32) : hw == 32,
             "vae_encode_moments: input extent must be 8/16/24/32 (surface) or 32 (edge)");
  Tail t;
  t.moments = moments;
  return run_vae(m, xin, N, hw, nullptr, workspace, workspace_bytes, stream, "vae_encode_moments", &t);
}

int bg_vae_posterior(const float* moments, const float* noise, int N, int P, int deterministic, float* z, float* kl,
                     void* stream) {
  BG_TRY(bg_check_device());
  BG_REQUIRE(moments && N > 0 && P > 0, "vae_posterior: bad arguments");
  Tail t;
  t.noise = noise;
  t.z = z;
  t.kl = kl;
  return posterior(op_ctx(N, stream), nullptr, 0, nullptr, nullptr, moments, t, P, deterministic);
}

// The round trip shares one carve between the encoder and then the decoder; z follows it, outside the carve.
static size_t recon_carve_bytes(const BgVae* enc, const BgVae* dec, size_t N) {
  return std::max(carve_vae(nullptr, enc->kind, N).bytes, carve_vae(nullptr, dec->kind, N).bytes);
}

size_t bg_vae_reconstruct_workspace_bytes(const BgVae* enc, const BgVae* dec, int N) {
  if (!enc || !dec || N <= 0) return 0;
  const size_t max_p = enc->kind == 2 ? 16 : 4;      // latent positions at the largest extent (32 x 32 / 32 points)
  return recon_carve_bytes(enc, dec, (size_t)N) + align_up((size_t)N * 3 * max_p * 4, 1024) + 1024;
}

int bg_vae_reconstruct(BgVae* enc, BgVae* dec, const float* x, int N, int hw, const float* noise, float* moments, float* z,
                       float* kl, float* dec_out, float* mse, void* workspace, size_t workspace_bytes, void* stream) {
  BG_REQUIRE(enc && dec && x && dec_out && workspace && N > 0, "vae_reconstruct: bad arguments");
  BG_REQUIRE((enc->kind == 2 || enc->kind == 3) && dec->kind == enc->kind - 2,
             "vae_reconstruct: needs an encoder handle and the decoder handle of the same family");
  BG_REQUIRE(enc->kind == 2 ? (hw == 8 || hw == 16 || hw == 24 || hw == 32) : hw == 32,
             "vae_reconstruct: input extent must be 8/16/24/32 (surface) or 32 (edge)");
  const int lat = hw / 8, P = enc->kind == 2 ? lat * lat : lat, vals = 3 * hw * (enc->kind == 2 ? hw : 1);
  const size_t carve = recon_carve_bytes(enc, dec, (size_t)N);
  char* base;
  BG_TRY(align_workspace(workspace, workspace_bytes, carve + align_up((size_t)N * 3 * P * 4, 1024), "vae_reconstruct", &base));
  Tail t;
  t.noise = noise;
  t.moments = moments;
  t.kl = kl;
  t.z = z ? z : reinterpret_cast<float*>(base + carve);
  BG_TRY(run_vae(enc, x, N, hw, nullptr, base, carve, stream, "vae_reconstruct", &t));
  BG_TRY(run_vae(dec, t.z, N, lat, dec_out, base, carve, stream, "vae_reconstruct"));
  return mse ? sample_mse(op_ctx(N, stream), dec_out, x, vals, mse) : BG_OK;
}

// ---- unit-level entry points: the networks' own launch code on caller-owned buffers
int bg_op_groupnorm(const float* x, int N, int P, int C, int G, float eps, const float* gamma, const float* beta, int act,
                    const float* resid, float* out32, void* out16, void* stream) {
  BG_TRY(bg_check_device());
  const int cpg = G > 0 ? C / G : 0;
  BG_REQUIRE(x && gamma && beta && (out32 || out16) && N > 0 && P > 0 && C > 0 && C <= 1024 && C % 32 == 0 && cpg > 0 &&
                 C % G == 0 && (cpg > 32 ? cpg % 32 == 0 : 32 % cpg == 0) && act >= 0 && act <= 2,
             "groupnorm: bad arguments");
  Norm n;
  n.g = const_cast<float*>(gamma);
  n.b = const_cast<float*>(beta);
  return groupnorm(op_ctx(N, stream), x, P, C, G, eps, n, act, resid, out32, reinterpret_cast<__half*>(out16));
}

int bg_op_vae_attention(const void* qkv, void* out, int N, int T, int Hh, float scale, void* stream) {
  BG_TRY(bg_check_device());
  BG_REQUIRE(qkv && out && N > 0 && T > 0 && Hh > 0 && 512 % Hh == 0 && T * T * Hh <= 256, "vae_attention: bad arguments");
  return small_attention(op_ctx(N, stream), reinterpret_cast<const __half*>(qkv), reinterpret_cast<__half*>(out), T, Hh,
                         scale);
}

int bg_op_cubic1d(const float* x, float* y, int N, int L, int C, const float* kernel8, int up, void* stream) {
  BG_TRY(bg_check_device());
  BG_REQUIRE(x && y && kernel8 && N > 0 && L >= 4 && C > 0 && (up || L % 2 == 0), "cubic1d: bad arguments");
  return cubic1d(op_ctx(N, stream), x, y, L, C, kernel8, up != 0);
}

int bg_op_cast_split(const float* x, void* y, int64_t rows, int C, void* stream) {
  BG_TRY(bg_check_device());
  BG_REQUIRE(x && y && rows > 0 && C > 0, "cast_split: bad arguments");
  return cast_split(op_ctx(1, stream), x, reinterpret_cast<__half*>(y), C, (size_t)rows);
}

int bg_op_upsample2x_split(const float* x, void* y, int N, int H, int W, int C, void* stream) {
  BG_TRY(bg_check_device());
  BG_REQUIRE(x && y && N > 0 && H > 0 && W > 0 && C > 0, "upsample2x_split: bad arguments");
  return upsample2x_split(op_ctx(N, stream), x, reinterpret_cast<__half*>(y), H, W, C);
}

int bg_op_postquant(const float* z, const float* w, const float* b, void* y, int N, int P, void* stream) {
  BG_TRY(bg_check_device());
  BG_REQUIRE(z && w && b && y && N > 0 && P > 0, "postquant: bad arguments");
  return postquant(op_ctx(N, stream), z, w, b, reinterpret_cast<__half*>(y), P);
}

int bg_op_im2col(const void* in, int ldin, void* A, int ldA, int N, int H, int W, int C, int kh, int kw, int stride,
                 int Kpad, void* stream) {
  BG_TRY(bg_check_device());
  BG_REQUIRE(in && A && N > 0 && H > 0 && W > 0 && C > 0 && kh > 0 && kw > 0 && (stride == 1 || stride == 2) &&
                 H >= stride && W >= stride && Kpad >= kh * kw * C && ldin >= C && ldA >= Kpad &&
                 (C % 8 != 0 || (ldin % 8 == 0 && ldA % 8 == 0 && Kpad % 8 == 0)),
             "im2col: bad arguments");
  return im2col(op_ctx(N, stream), reinterpret_cast<const __half*>(in), ldin, reinterpret_cast<__half*>(A), ldA, H, W, C,
                kh, kw, stride, Kpad);
}

}  // extern "C"
