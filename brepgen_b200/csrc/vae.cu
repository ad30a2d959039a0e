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
#include <map>
#include <string>
#include <vector>

#include "../../include/brepgen_b200.h"
#include "bg_internal.h"

#include <stdlib.h>

namespace bg {
namespace {

inline size_t align_up(size_t x, size_t a = 256) { return (x + a - 1) / a * a; }
inline int round64(int k) { return (k + 63) / 64 * 64; }

// Number of product terms of the compensated GEMMs, fixed per handle at creation:
//   3: A_hi W_hi + A_lo W_hi + A_hi W_lo   (activations AND weights split)
//   2: A_hi W_hi + A_hi W_lo               (weights split only: the systematic part of the fp16 error) -- 1/3 less GEMM work
//                                           and no lo plane in the im2col matrices
// Relative L2 errors against the fp32 oracle (bar 1e-3), measured on an H100 with 3 / 2 terms: surface decoder 9.4e-5 /
// 1.3e-3, edge decoder 3.6e-5 / 4.1-4.3e-4, encoders <= 1.1e-4 / 6.4-9.0e-4.  So the edge decoder defaults to 2 terms (a
// third less GEMM work); the surface decoder, over the bar with 2, and the encoders, close to it, keep 3.  BREPGEN_B200_VAE_TERMS = 2 | 3 overrides.
int vae_terms_for(int kind) {
  const char* e = getenv("BREPGEN_B200_VAE_TERMS");
  if (e && (atoi(e) == 2 || atoi(e) == 3)) return atoi(e);
  return kind == 1 ? 2 : 3;
}

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
// plain linear [N][K] fp32 -> rows [row0, row0+N) of a [*][3K] hi|hi|lo operand
__global__ void pack_linear_split_kernel(const float* __restrict__ w, __half* __restrict__ dst, int N, int K, int row0, int terms) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)N * K) return;
  const int n = (int)(i / K), k = (int)(i % K);
  const float v = w[i];
  const __half hi = __float2half_rn(v), lo = __float2half_rn(v - __half2float(hi));
  dst[(size_t)(row0 + n) * 3 * K + k] = hi;
  dst[(size_t)(row0 + n) * 3 * K + K + k] = terms == 3 ? hi : lo;
  dst[(size_t)(row0 + n) * 3 * K + 2 * K + k] = lo;
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

// in (N, H, W, C) fp16 -> A (N*Ho*Wo, Kpad) fp16, 3x3 pad 1 on the (optionally nearest-2x upsampled) image
// stride 1 / pad_lo 1: the usual 3x3 pad-1 convolution; stride 2 / pad_lo 0: diffusers Downsample2D(padding=0), i.e.
// zero padding on the right / bottom only.  Hs x Ws = upsampled source extent, Ho x Wo = output extent.
__global__ void im2col2d_kernel(const __half* __restrict__ in, int ldin, __half* __restrict__ A, int ldA, int H, int W, int C,
                                int up, int stride, int pad_lo, int Kpad, size_t total_vec, int vec) {
  const int Hs = H * up, Ws = W * up;
  const int Ho = Hs / stride, Wo = Ws / stride;
  const int kvec = Kpad / vec;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total_vec; i += (size_t)gridDim.x * blockDim.x) {
    const size_t row = i / kvec;
    const int k = (int)(i % kvec) * vec;
    const int x = (int)(row % Wo), y = (int)((row / Wo) % Ho);
    const size_t n = row / ((size_t)Wo * Ho);
    __half* dst = A + row * ldA + k;
    if (vec == 8) {
      uint4 v = make_uint4(0, 0, 0, 0);
      if (k < 9 * C) {
        const int tap = k / C, c = k % C;
        const int yy = y * stride + tap / 3 - pad_lo, xx = x * stride + tap % 3 - pad_lo;
        if (yy >= 0 && yy < Hs && xx >= 0 && xx < Ws)
          v = *reinterpret_cast<const uint4*>(in + ((n * H + yy / up) * W + xx / up) * ldin + c);
      }
      *reinterpret_cast<uint4*>(dst) = v;
    } else {
      __half v = __float2half_rn(0.f);
      if (k < 9 * C) {
        const int tap = k / C, c = k % C;
        const int yy = y * stride + tap / 3 - pad_lo, xx = x * stride + tap % 3 - pad_lo;
        if (yy >= 0 && yy < Hs && xx >= 0 && xx < Ws) v = in[((n * H + yy / up) * W + xx / up) * ldin + c];
      }
      *dst = v;
    }
  }
}

// in (N, L, C) fp16 -> A (N*L, Kpad) fp16, kernel size ks (odd), pad ks/2
__global__ void im2col1d_kernel(const __half* __restrict__ in, int ldin, __half* __restrict__ A, int ldA, int L, int C, int ks,
                                int Kpad, size_t total_vec, int vec) {
  const int kvec = Kpad / vec;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total_vec; i += (size_t)gridDim.x * blockDim.x) {
    const size_t row = i / kvec;
    const int k = (int)(i % kvec) * vec;
    const int l = (int)(row % L);
    const size_t n = row / L;
    __half* dst = A + row * ldA + k;
    if (vec == 8) {
      uint4 v = make_uint4(0, 0, 0, 0);
      if (k < ks * C) {
        const int tap = k / C, c = k % C;
        const int ll = l + tap - ks / 2;
        if (ll >= 0 && ll < L) v = *reinterpret_cast<const uint4*>(in + (n * L + ll) * ldin + c);
      }
      *reinterpret_cast<uint4*>(dst) = v;
    } else {
      __half v = __float2half_rn(0.f);
      if (k < ks * C) {
        const int tap = k / C, c = k % C;
        const int ll = l + tap - ks / 2;
        if (ll >= 0 && ll < L) v = in[(n * L + ll) * ldin + c];
      }
      *dst = v;
    }
  }
}

__device__ __forceinline__ float act_fn(float y, int act) {
  if (act == 1) return y / (1.f + __expf(-y));                       // SiLU
  if (act == 2) return 0.5f * y * (1.f + erff(y * 0.70710678118f));   // exact (erf) GELU
  return y;
}

// GroupNorm over (P positions x C/G channels) per sample and group, then activation, then optional residual add.
// x (N, P, C) fp32 (pitch ldx per position); one CTA per sample, blockDim == C, thread <-> channel.
__global__ void groupnorm_kernel(const float* __restrict__ x, int ldx, int P, int C, int G, float eps,
                                 const float* __restrict__ gamma, const float* __restrict__ beta, int act,
                                 const float* __restrict__ resid, float* __restrict__ out32, __half* __restrict__ out16) {
  __shared__ float s_part[32];
  __shared__ float s_stat[64];     // mean[G], rstd[G]
  const int n = blockIdx.x, c = threadIdx.x;
  const int cpg = C / G;
  const int g = c / cpg;
  const float* xs = x + (size_t)n * P * ldx;
  const int lane = c & 31, warp = c >> 5, nwarp = blockDim.x >> 5;
  const float cnt = (float)P * cpg;

  auto group_reduce = [&](float v) -> float {      // sum of v over all threads of this thread's group
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
  };
  (void)nwarp;

  float s = 0.f;
  for (int p = 0; p < P; ++p) s += xs[(size_t)p * ldx + c];
  const float mean = group_reduce(s) / cnt;
  float q = 0.f;
  for (int p = 0; p < P; ++p) {
    const float d = xs[(size_t)p * ldx + c] - mean;
    q += d * d;
  }
  const float rstd = rsqrtf(group_reduce(q) / cnt + eps);
  (void)s_stat;
  const float ga = gamma[c] * rstd, be = beta[c] - mean * gamma[c] * rstd;
  for (int p = 0; p < P; ++p) {
    float y = act_fn(xs[(size_t)p * ldx + c] * ga + be, act);
    const size_t o = ((size_t)n * P + p) * C + c;
    if (resid) y += resid[o];
    if (out32) out32[o] = y;
    if (out16) store_hl(out16 + ((size_t)n * P + p) * 2 * C + c, C, y);
  }
}

// Same for P <= 64 positions (every 1-D stage, the 4x4 / 8x8 2-D stages): the thread's P values stay in registers, so the
// activation is read once instead of three times (this kernel was 30 % of the edge decoder).
template <int P>
__global__ void groupnorm_regs_kernel(const float* __restrict__ x, int ldx, int C, int G, float eps,
                                      const float* __restrict__ gamma, const float* __restrict__ beta, int act,
                                      const float* __restrict__ resid, float* __restrict__ out32, __half* __restrict__ out16) {
  __shared__ float s_part[32];
  const int n = blockIdx.x, c = threadIdx.x;
  const int cpg = C / G;
  const float* xs = x + (size_t)n * P * ldx;
  const int lane = c & 31, warp = c >> 5;
  const float cnt = (float)P * cpg;
  auto group_reduce = [&](float v) -> float {
    if (cpg <= 32) {
      for (int o = cpg >> 1; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      return v;
    }
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if (lane == 0) s_part[warp] = v;
    __syncthreads();
    const int wpg = cpg >> 5;
    float t = 0.f;
    const int w0 = (warp / wpg) * wpg;
    for (int w = 0; w < wpg; ++w) t += s_part[w0 + w];
    return t;
  };
  float v[P];
  float s = 0.f;
#pragma unroll
  for (int p = 0; p < P; ++p) {
    v[p] = xs[(size_t)p * ldx + c];
    s += v[p];
  }
  const float mean = group_reduce(s) / cnt;
  float q = 0.f;
#pragma unroll
  for (int p = 0; p < P; ++p) {
    const float d = v[p] - mean;
    q += d * d;
  }
  const float rstd = rsqrtf(group_reduce(q) / cnt + eps);
  const float ga = gamma[c] * rstd, be = beta[c] - mean * gamma[c] * rstd;
#pragma unroll
  for (int p = 0; p < P; ++p) {
    float y = act_fn(v[p] * ga + be, act);
    const size_t o = ((size_t)n * P + p) * C + c;
    if (resid) y += resid[o];
    if (out32) out32[o] = y;
    if (out16) store_hl(out16 + ((size_t)n * P + p) * 2 * C + c, C, y);
  }
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
  int terms = 3;                // product terms of the compensated GEMMs (vae_terms_for)
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

struct VPacker {
  std::map<std::string, const BgNamedTensor*> by_name;
  char* base = nullptr;
  size_t off = 0;
  bool dry = true;
  cudaStream_t st = nullptr;
  int err = 0;
  int terms = 3;

  const float* find(const std::string& name, int64_t numel) {
    auto it = by_name.find(name);
    if (it == by_name.end()) {
      if (!err) err = set_error(BG_ERR_MISSING_WEIGHT, "missing weight: " + name);
      return nullptr;
    }
    if (it->second->numel != numel) {
      if (!err) err = set_error(BG_ERR_BAD_ARG, "weight " + name + " has the wrong number of elements");
      return nullptr;
    }
    return it->second->data;
  }
  template <class T>
  T* take(size_t n) {
    T* p = dry ? nullptr : reinterpret_cast<T*>(base + off);
    off += align_up(n * sizeof(T));
    return p;
  }
  float* copy(const std::string& name, int64_t numel) {
    const float* src = find(name, numel);
    float* dst = take<float>(numel);
    if (!dry && src && !err) err = check_cuda(cudaMemcpyAsync(dst, src, numel * 4, cudaMemcpyDeviceToDevice, st), "copy");
    return dst;
  }
  float* zeros(int64_t numel) {
    float* dst = take<float>(numel);
    if (!dry && !err) err = check_cuda(cudaMemsetAsync(dst, 0, numel * 4, st), "memset");
    return dst;
  }
  Norm norm(const std::string& name, int c) {
    Norm n;
    n.g = copy(name + ".weight", c);
    n.b = copy(name + ".bias", c);
    return n;
  }
  Conv conv(const std::string& name, int cout, int cin, int taps, bool bias = true, int cout_pad = 0) {
    Conv c;
    c.cin = cin; c.cout = cout; c.taps = taps;
    c.kpad = round64(cin * taps);
    c.cout_pad = cout_pad ? cout_pad : cout;
    const float* w = find(name + ".weight", (int64_t)cout * cin * taps);
    c.w = take<__half>((size_t)c.cout_pad * 3 * c.kpad);
    if (!dry && w && !err) {
      const size_t tot = (size_t)c.cout_pad * c.kpad;
      pack_conv_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, st>>>(w, c.w, cout, cin, taps, c.kpad, c.cout_pad, terms);
      err = check_launch("pack_conv_kernel launch");
    }
    if (bias) {
      if (c.cout_pad == cout) {
        c.bias = copy(name + ".bias", cout);
      } else {
        const float* b = find(name + ".bias", cout);
        c.bias = zeros(c.cout_pad);
        if (!dry && b && !err) err = check_cuda(cudaMemcpyAsync(c.bias, b, cout * 4, cudaMemcpyDeviceToDevice, st), "copy");
      }
    }
    return c;
  }
  // q | k | v linears (C -> C each) concatenated into one [3C][C] operand
  Conv qkv(const std::string& a, const char* qn, const char* kn, const char* vn, int C) {
    Conv c;
    c.cin = C; c.cout = 3 * C; c.taps = 1; c.kpad = C; c.cout_pad = 3 * C;
    c.w = take<__half>((size_t)3 * C * 3 * C);
    c.bias = take<float>(3 * C);
    const char* names[3] = {qn, kn, vn};
    for (int i = 0; i < 3; ++i) {
      const float* w = find(a + "." + names[i] + ".weight", (int64_t)C * C);
      const float* b = find(a + "." + names[i] + ".bias", C);
      if (!dry && w && b && !err) {
        pack_linear_split_kernel<<<(C * C + 255) / 256, 256, 0, st>>>(w, c.w, C, C, i * C, terms);
        err = check_launch("pack_linear_split_kernel launch");
        if (!err) err = check_cuda(cudaMemcpyAsync(c.bias + i * C, b, C * 4, cudaMemcpyDeviceToDevice, st), "copy");
      }
    }
    return c;
  }
};

int pack_encoder(BgVae* m, VPacker& pk);

int pack_vae(BgVae* m, VPacker& pk) {
  if (m->kind >= 2) return pack_encoder(m, pk);
  const std::string d = "decoder.";
  const int taps_in = m->kind == 0 ? 9 : 3;
  m->pq_w = pk.copy("post_quant_conv.weight", 9);
  m->pq_b = pk.copy("post_quant_conv.bias", 3);
  m->conv_in = pk.conv(d + "conv_in", 512, 3, taps_in);
  if (m->kind == 0) {
    auto res2d = [&](const std::string& n, int cin, int cout) {
      Res2d r;
      r.n1 = pk.norm(n + ".norm1", cin);
      r.c1 = pk.conv(n + ".conv1", cout, cin, 9);
      r.n2 = pk.norm(n + ".norm2", cout);
      r.c2 = pk.conv(n + ".conv2", cout, cout, 9);
      r.has_sc = cin != cout;
      if (r.has_sc) r.sc = pk.conv(n + ".conv_shortcut", cout, cin, 1);
      return r;
    };
    m->s_mid[0] = res2d(d + "mid_block.resnets.0", 512, 512);
    const std::string a = d + "mid_block.attentions.0";
    m->s_attn.gn = pk.norm(a + ".group_norm", 512);
    m->s_attn.qkv = pk.qkv(a, "to_q", "to_k", "to_v", 512);
    m->s_attn.proj = pk.conv(a + ".to_out.0", 512, 512, 1);
    m->s_mid[1] = res2d(d + "mid_block.resnets.1", 512, 512);
    const int chans[4][2] = {{512, 512}, {512, 512}, {512, 256}, {256, 128}};
    for (int i = 0; i < 4; ++i) {
      for (int j = 0; j < 3; ++j)
        m->s_up[i][j] = res2d(d + "up_blocks." + std::to_string(i) + ".resnets." + std::to_string(j),
                              j == 0 ? chans[i][0] : chans[i][1], chans[i][1]);
      if (i < 3) m->s_upconv[i] = pk.conv(d + "up_blocks." + std::to_string(i) + ".upsamplers.0.conv", chans[i][1], chans[i][1], 9);
    }
    m->norm_out = pk.norm(d + "conv_norm_out", 128);
    m->conv_out = pk.conv(d + "conv_out", 3, 128, 9, true, 128);
  } else {
    auto res1d = [&](const std::string& n, int cin, int cmid, int cout) {
      Res1d r;
      r.has_skip = cin != cout;
      if (r.has_skip) r.skip = pk.conv(n + ".conv_skip", cout, cin, 1, false);
      r.c1 = pk.conv(n + ".conv_1", cmid, cin, 5);
      r.n1 = pk.norm(n + ".group_norm_1", cmid);
      r.c2 = pk.conv(n + ".conv_2", cout, cmid, 5);
      r.n2 = pk.norm(n + ".group_norm_2", cout);
      return r;
    };
    for (int i = 0; i < 6; ++i) m->e_mid[i] = res1d(d + "mid_block.resnets." + std::to_string(i), 512, 512, 512);
    for (int i = 0; i < 6; ++i) {
      const std::string a = d + "mid_block.attentions." + std::to_string(i);
      m->e_attn[i].gn = pk.norm(a + ".group_norm", 512);
      m->e_attn[i].qkv = pk.qkv(a, "query", "key", "value", 512);
      m->e_attn[i].proj = pk.conv(a + ".proj_attn", 512, 512, 1);
    }
    const int chans[3][2] = {{512, 512}, {512, 256}, {256, 128}};
    for (int i = 0; i < 3; ++i) {
      const std::string b = d + "up_blocks." + std::to_string(i);
      m->e_up[i][0] = res1d(b + ".resnets.0", chans[i][0], chans[i][0], chans[i][0]);
      m->e_up[i][1] = res1d(b + ".resnets.1", chans[i][0], chans[i][0], chans[i][0]);
      m->e_up[i][2] = res1d(b + ".resnets.2", chans[i][0], chans[i][0], chans[i][1]);
    }
    m->up_kernel = pk.copy(d + "up_blocks.0.up.kernel", 8);   // the same fixed 8-tap buffer in all three blocks
    m->norm_out = pk.norm(d + "conv_norm_out", 128);
    m->conv_out = pk.conv(d + "conv_out", 3, 128, 3, true, 128);
  }
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
    auto res2d = [&](const std::string& n, int cin, int cout) {
      Res2d r;
      r.n1 = pk.norm(n + ".norm1", cin);
      r.c1 = pk.conv(n + ".conv1", cout, cin, 9);
      r.n2 = pk.norm(n + ".norm2", cout);
      r.c2 = pk.conv(n + ".conv2", cout, cout, 9);
      r.has_sc = cin != cout;
      if (r.has_sc) r.sc = pk.conv(n + ".conv_shortcut", cout, cin, 1);
      return r;
    };
    const int chans[4][2] = {{128, 128}, {128, 256}, {256, 512}, {512, 512}};
    for (int i = 0; i < 4; ++i) {
      for (int j = 0; j < 2; ++j)
        m->s_down[i][j] = res2d(e + "down_blocks." + std::to_string(i) + ".resnets." + std::to_string(j),
                                j == 0 ? chans[i][0] : chans[i][1], chans[i][1]);
      if (i < 3) m->s_downconv[i] = pk.conv(e + "down_blocks." + std::to_string(i) + ".downsamplers.0.conv", chans[i][1], chans[i][1], 9);
    }
    m->s_mid[0] = res2d(e + "mid_block.resnets.0", 512, 512);
    const std::string a = e + "mid_block.attentions.0";
    m->s_attn.gn = pk.norm(a + ".group_norm", 512);
    m->s_attn.qkv = pk.qkv(a, "to_q", "to_k", "to_v", 512);
    m->s_attn.proj = pk.conv(a + ".to_out.0", 512, 512, 1);
    m->s_mid[1] = res2d(e + "mid_block.resnets.1", 512, 512);
    m->norm_out = pk.norm(e + "conv_norm_out", 512);
    m->conv_out = pk.conv(e + "conv_out", 6, 512, 9, true, 128);
  } else {
    auto res1d = [&](const std::string& n, int cin, int cmid, int cout) {
      Res1d r;
      r.has_skip = cin != cout;
      if (r.has_skip) r.skip = pk.conv(n + ".conv_skip", cout, cin, 1, false);
      r.c1 = pk.conv(n + ".conv_1", cmid, cin, 5);
      r.n1 = pk.norm(n + ".group_norm_1", cmid);
      r.c2 = pk.conv(n + ".conv_2", cout, cmid, 5);
      r.n2 = pk.norm(n + ".group_norm_2", cout);
      return r;
    };
    const int chans[3][2] = {{128, 128}, {128, 256}, {256, 512}};
    for (int i = 0; i < 3; ++i) {
      const std::string b = e + "down_blocks." + std::to_string(i);
      m->e_down[i][0] = res1d(b + ".resnets.0", chans[i][0], chans[i][1], chans[i][1]);
      m->e_down[i][1] = res1d(b + ".resnets.1", chans[i][1], chans[i][1], chans[i][1]);
      m->e_down[i][2] = res1d(b + ".resnets.2", chans[i][1], chans[i][1], chans[i][1]);
    }
    m->down_kernel = pk.copy(e + "down_blocks.0.down.kernel", 8);
    for (int i = 0; i < 6; ++i) m->e_mid[i] = res1d(e + "mid_block.resnets." + std::to_string(i), 512, 512, 512);
    for (int i = 0; i < 6; ++i) {
      const std::string a = e + "mid_block.attentions." + std::to_string(i);
      m->e_attn[i].gn = pk.norm(a + ".group_norm", 512);
      m->e_attn[i].qkv = pk.qkv(a, "query", "key", "value", 512);
      m->e_attn[i].proj = pk.conv(a + ".proj_attn", 512, 512, 1);
    }
    m->norm_out = pk.norm(e + "conv_norm_out", 512);
    m->conv_out = pk.conv(e + "conv_out", 6, 512, 3, true, 128);
  }
  m->q_w = pk.copy("quant_conv.weight", 36);
  m->q_b = pk.copy("quant_conv.bias", 6);
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

struct Ctx {
  cudaStream_t st;
  size_t N;
  VaeWs w;
  int terms = 3;
  int implicit = 1;
};

// A: [rows][2 * cv.kpad] fp16 = [A_hi | A_lo]
int gemm(const Ctx& c, const __half* A, const Conv& cv, size_t rows, float* out32, __half* out16, const float* resid) {
  GemmEpilogue ep;
  ep.out = out16 ? (void*)out16 : (void*)out32;
  ep.out_f16 = out16 ? 1 : 0;
  ep.ldo = cv.cout_pad;
  ep.bias = cv.bias;
  ep.resid = resid;
  ep.ldr = cv.cout_pad;
  if (c.terms == 3) {
    ep.a_kwrap = 2 * cv.kpad;    // [A_hi | A_lo | A_hi] x [W_hi | W_hi | W_lo]
    return launch_gemm_f16(c.st, A, 2 * cv.kpad, cv.w, 3 * cv.kpad, (int)rows, cv.cout_pad, 3 * cv.kpad, ep);
  }
  ep.a_kwrap = cv.kpad;          // [A_hi | A_hi] x [W_hi | W_lo]  (the lo plane of A is not read)
  return launch_gemm_f16(c.st, A, 2 * cv.kpad, cv.w, 3 * cv.kpad, (int)rows, cv.cout_pad, 2 * cv.kpad, ep);
}
// shapes the implicit convolution covers: a 128-row tile of output pixels must be a box {W, box_h, box_n} of whole image rows
bool conv_implicit_ok(int H, int W, int C) {
  const int hw = H * W;
  return C % 64 == 0 && W <= 128 && 128 % W == 0 && (hw % 128 == 0 || 128 % hw == 0);
}
// stride-1 "same" convolution (taps = kh * kw) of the [hi | lo] fp16 image `in` (N, H, W, 2 * cv.cin) as an implicit GEMM
int conv_gemm(const Ctx& c, const __half* in, int H, int W, int taps, int kw, const Conv& cv, float* out32, __half* out16,
              const float* resid) {
  GemmEpilogue ep;
  ep.out = out16 ? (void*)out16 : (void*)out32;
  ep.out_f16 = out16 ? 1 : 0;
  ep.ldo = cv.cout_pad;
  ep.bias = cv.bias;
  ep.resid = resid;
  ep.ldr = cv.cout_pad;
  ep.conv.taps = taps; ep.conv.kw = kw; ep.conv.C = cv.cin; ep.conv.W = W; ep.conv.H = H; ep.conv.N = (int)c.N;
  ep.conv.lo_plane = 1; ep.conv.terms = c.terms;
  return launch_gemm_f16(c.st, in, 2 * cv.cin, cv.w, 3 * cv.kpad, (int)(c.N * H * W), cv.cout_pad, c.terms * cv.kpad, ep);
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
int im2col2d(const Ctx& c, const __half* in, int H, int W, int C, int up, int kpad, int stride = 1) {
  const int vec = (C % 8 == 0) ? 8 : 1;
  const int pad_lo = stride == 1 ? 1 : 0;
  const size_t tot = c.N * (size_t)(H * up / stride) * (W * up / stride) * (kpad / vec);
  for (int part = 0; part < c.terms - 1; ++part) {   // hi plane, then (3-term mode) lo plane of the [hi | lo] activation
    im2col2d_kernel<<<grid_for(tot), 256, 0, c.st>>>(in + part * C, 2 * C, c.w.A + part * kpad, 2 * kpad, H, W, C, up, stride, pad_lo, kpad, tot, vec);
    BG_TRY(check_launch("im2col2d_kernel launch"));
  }
  return BG_OK;
}
int im2col1d(const Ctx& c, const __half* in, int L, int C, int ks, int kpad) {
  const int vec = (C % 8 == 0) ? 8 : 1;
  const size_t tot = c.N * (size_t)L * (kpad / vec);
  for (int part = 0; part < c.terms - 1; ++part) {
    im2col1d_kernel<<<grid_for(tot), 256, 0, c.st>>>(in + part * C, 2 * C, c.w.A + part * kpad, 2 * kpad, L, C, ks, kpad, tot, vec);
    BG_TRY(check_launch("im2col1d_kernel launch"));
  }
  return BG_OK;
}
int conv3x3(const Ctx& c, const __half* in, int H, const Conv& cv, float* out32, const float* resid) {
  if (c.implicit && conv_implicit_ok(H, H, cv.cin)) return conv_gemm(c, in, H, H, 9, 3, cv, out32, nullptr, resid);
  BG_TRY(im2col2d(c, in, H, H, cv.cin, 1, cv.kpad));
  return gemm(c, c.w.A, cv, c.N * H * H, out32, nullptr, resid);
}
int conv1d(const Ctx& c, const __half* in, int L, int ks, const Conv& cv, float* out32, const float* resid) {
  if (c.implicit && conv_implicit_ok(1, L, cv.cin)) return conv_gemm(c, in, 1, L, ks, ks, cv, out32, nullptr, resid);
  BG_TRY(im2col1d(c, in, L, cv.cin, ks, cv.kpad));
  return gemm(c, c.w.A, cv, c.N * L, out32, nullptr, resid);
}
int attention(const Ctx& c, int T, int Hh, int dh, float scale) {
  const int C = Hh * dh;
  const size_t smem = (size_t)(3 * T * C + Hh * T * T) * 4;
  BG_TRY(ensure_dynamic_smem(reinterpret_cast<const void*>(&small_attention_kernel), 112 * 1024));
  small_attention_kernel<<<(unsigned)c.N, 256, smem, c.st>>>(c.w.Q, c.w.Q + c.N * (size_t)T * 3 * C, T, Hh, dh, scale);   // out: [N*T][2C]
  return check_launch("small_attention_kernel launch");
}

// x (in place, fp32 [N, P, Cout] in *px): diffusers ResnetBlock2D without time embedding
int resnet2d(const Ctx& c, const Res2d& r, float** px, float** pfree, int HW, int H) {
  const int cin = r.c1.cin, cout = r.c1.cout;
  float* x = *px;
  BG_TRY(groupnorm(c, x, HW, cin, 32, 1e-6f, r.n1, 1, nullptr, nullptr, c.w.T));
  BG_TRY(conv3x3(c, c.w.T, H, r.c1, c.w.H, nullptr));
  if (!r.has_sc) {
    BG_TRY(groupnorm(c, c.w.H, HW, cout, 32, 1e-6f, r.n2, 1, nullptr, nullptr, c.w.T));
    return conv3x3(c, c.w.T, H, r.c2, x, x);
  }
  // 1x1 shortcut on the raw input (T is free between the two convolutions), then conv2 accumulates onto it
  float* s = *pfree;
  BG_TRY(cast_split(c, x, c.w.T, cin, c.N * (size_t)HW));
  BG_TRY(gemm(c, c.w.T, r.sc, c.N * HW, s, nullptr, nullptr));
  BG_TRY(groupnorm(c, c.w.H, HW, cout, 32, 1e-6f, r.n2, 1, nullptr, nullptr, c.w.T));
  BG_TRY(conv3x3(c, c.w.T, H, r.c2, s, s));
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
  BG_TRY(conv1d(c, c.w.T, L, 5, r.c1, c.w.H, nullptr));
  BG_TRY(groupnorm(c, c.w.H, L, cmid, 1, 1e-5f, r.n1, 2, nullptr, nullptr, c.w.T));
  BG_TRY(conv1d(c, c.w.T, L, 5, r.c2, c.w.H, nullptr));
  BG_TRY(groupnorm(c, c.w.H, L, cout, 1, 1e-5f, r.n2, 2, res, out, nullptr));
  if (r.has_skip) {
    *px = out;
    *pfree = x;
  }
  return BG_OK;
}

}  // namespace

extern "C" {

int bg_vae_create(int kind, const BgNamedTensor* weights, int n_weights, void* stream, BgVae** out) {
  BG_REQUIRE(kind >= 0 && kind <= 3 && weights && n_weights > 0 && out, "vae_create: bad arguments");
  BG_TRY(bg_check_device());
  BgVae* m = new BgVae();
  m->kind = kind;
  m->terms = vae_terms_for(kind);
  if (const char* e = getenv("BREPGEN_B200_VAE_IM2COL")) m->implicit = atoi(e) ? 0 : 1;
  VPacker pk;
  pk.terms = m->terms;
  for (int i = 0; i < n_weights; ++i) pk.by_name[weights[i].name] = &weights[i];
  pk.st = reinterpret_cast<cudaStream_t>(stream);
  int s = pack_vae(m, pk);
  if (s == 0) {
    m->arena_bytes = pk.off;
    s = check_cuda(cudaMalloc(reinterpret_cast<void**>(&m->arena), m->arena_bytes), "cudaMalloc(vae weights)");
  }
  if (s == 0) {
    pk.dry = false; pk.base = m->arena; pk.off = 0;
    s = pack_vae(m, pk);
  }
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
  Ctx c;
  c.st = reinterpret_cast<cudaStream_t>(stream);
  c.N = (size_t)N;
  c.terms = m->terms;
  c.implicit = m->implicit;
  char* base = reinterpret_cast<char*>((reinterpret_cast<uintptr_t>(workspace) + 1023) & ~uintptr_t(1023));
  c.w = carve_vae(base, m->kind, c.N);
  if (c.w.bytes + (size_t)(base - reinterpret_cast<char*>(workspace)) > workspace_bytes)
    return set_error(BG_ERR_WORKSPACE, "vae_decode: workspace too small");
  float* x = c.w.X;
  float* spare = c.w.S;

  if (m->kind == 0) {
    int H = hw;
    const int T = hw * hw;
    postquant_kernel<<<(N * T + 255) / 256, 256, 0, c.st>>>(z, m->pq_w, m->pq_b, c.w.T, N, T);
    BG_TRY(check_launch("postquant_kernel launch"));
    BG_TRY(im2col2d(c, c.w.T, hw, hw, 3, 1, m->conv_in.kpad));
    BG_TRY(gemm(c, c.w.A, m->conv_in, c.N * T, x, nullptr, nullptr));
    BG_TRY(resnet2d(c, m->s_mid[0], &x, &spare, T, hw));
    {   // single-head attention over the hw*hw positions (legacy diffusers attention block), residual
      BG_TRY(groupnorm(c, x, T, 512, 32, 1e-6f, m->s_attn.gn, 0, nullptr, nullptr, c.w.T));
      BG_TRY(gemm(c, c.w.T, m->s_attn.qkv, c.N * T, nullptr, c.w.Q, nullptr));
      BG_TRY(attention(c, T, 1, 512, 0.044194173824159216f));   // 1 / sqrt(512)
      BG_TRY(gemm(c, c.w.Q + c.N * (size_t)T * 1536, m->s_attn.proj, c.N * T, x, nullptr, x));
    }
    BG_TRY(resnet2d(c, m->s_mid[1], &x, &spare, T, hw));
    for (int i = 0; i < 4; ++i) {
      for (int j = 0; j < 3; ++j) BG_TRY(resnet2d(c, m->s_up[i][j], &x, &spare, H * H, H));
      if (i < 3) {
        const Conv& uc = m->s_upconv[i];
        if (c.implicit && conv_implicit_ok(2 * H, 2 * H, uc.cin)) {      // nearest 2x into the convolution's input, then implicit GEMM
          const size_t tot = c.N * (size_t)4 * H * H * uc.cin;
          upsample2x_split_kernel<<<grid_for(tot), 256, 0, c.st>>>(x, c.w.T, H, H, uc.cin, tot);
          BG_TRY(check_launch("upsample2x_split_kernel launch"));
          H *= 2;
          BG_TRY(conv_gemm(c, c.w.T, H, H, 9, 3, uc, spare, nullptr, nullptr));
        } else {
          BG_TRY(cast_split(c, x, c.w.T, uc.cin, c.N * (size_t)H * H));
          BG_TRY(im2col2d(c, c.w.T, H, H, uc.cin, 2, uc.kpad));
          H *= 2;
          BG_TRY(gemm(c, c.w.A, uc, c.N * H * H, spare, nullptr, nullptr));
        }
        float* t = x; x = spare; spare = t;
      }
    }
    BG_TRY(groupnorm(c, x, H * H, 128, 32, 1e-6f, m->norm_out, 1, nullptr, nullptr, c.w.T));
    BG_TRY(conv3x3(c, c.w.T, H, m->conv_out, c.w.H, nullptr));
    slice_out_kernel<<<(N * 3 * H * H + 255) / 256, 256, 0, c.st>>>(c.w.H, 128, out, N, H * H);
    return check_launch("slice_out_kernel launch");
  }

  int L = 4;
  postquant_kernel<<<(N * 4 + 255) / 256, 256, 0, c.st>>>(z, m->pq_w, m->pq_b, c.w.T, N, 4);
  BG_TRY(check_launch("postquant_kernel launch"));
  BG_TRY(im2col1d(c, c.w.T, 4, 3, 3, m->conv_in.kpad));
  BG_TRY(gemm(c, c.w.A, m->conv_in, c.N * 4, x, nullptr, nullptr));
  for (int i = 0; i < 6; ++i) {
    BG_TRY(resconv1d(c, m->e_mid[i], &x, &spare, 4));
    const Attn& a = m->e_attn[i];
    BG_TRY(groupnorm(c, x, 4, 512, 1, 1e-5f, a.gn, 0, nullptr, nullptr, c.w.T));
    BG_TRY(gemm(c, c.w.T, a.qkv, c.N * 4, nullptr, c.w.Q, nullptr));
    BG_TRY(attention(c, 4, 16, 32, 0.17677669529663687f));      // (1/sqrt(sqrt(32)))^2
    BG_TRY(gemm(c, c.w.Q + c.N * (size_t)4 * 1536, a.proj, c.N * 4, x, nullptr, x));
  }
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) BG_TRY(resconv1d(c, m->e_up[i][j], &x, &spare, L));
    const int C = m->e_up[i][2].c2.cout;
    const size_t tot = c.N * (size_t)2 * L * C;
    cubic_up1d_kernel<<<grid_for(tot), 256, 0, c.st>>>(x, spare, L, C, m->up_kernel, tot);
    BG_TRY(check_launch("cubic_up1d_kernel launch"));
    float* t = x; x = spare; spare = t;
    L *= 2;
  }
  BG_TRY(groupnorm(c, x, 32, 128, 32, 1e-6f, m->norm_out, 1, nullptr, nullptr, c.w.T));
  BG_TRY(conv1d(c, c.w.T, 32, 3, m->conv_out, c.w.H, nullptr));
  slice_out_kernel<<<(N * 3 * 32 + 255) / 256, 256, 0, c.st>>>(c.w.H, 128, out, N, 32);
  return check_launch("slice_out_kernel launch");
}

int bg_vae_encode(BgVae* m, const float* xin, int N, int hw, float* out, void* workspace, size_t workspace_bytes, void* stream) {
  BG_REQUIRE(m && xin && out && workspace && N > 0, "vae_encode: bad arguments");
  BG_REQUIRE(m->kind == 2 || m->kind == 3, "vae_encode: handle is not an encoder");
  BG_REQUIRE(m->kind == 2 ? (hw == 8 || hw == 16 || hw == 24 || hw == 32) : hw == 32,
             "vae_encode: input extent must be 8/16/24/32 (surface) or 32 (edge)");
  Ctx c;
  c.st = reinterpret_cast<cudaStream_t>(stream);
  c.N = (size_t)N;
  c.terms = m->terms;
  c.implicit = m->implicit;
  char* base = reinterpret_cast<char*>((reinterpret_cast<uintptr_t>(workspace) + 1023) & ~uintptr_t(1023));
  c.w = carve_vae(base, m->kind, c.N);
  if (c.w.bytes + (size_t)(base - reinterpret_cast<char*>(workspace)) > workspace_bytes)
    return set_error(BG_ERR_WORKSPACE, "vae_encode: workspace too small");
  float* x = c.w.X;
  float* spare = c.w.S;

  if (m->kind == 2) {
    int H = hw;
    postquant_kernel<<<(N * H * H + 255) / 256, 256, 0, c.st>>>(xin, m->pq_w, m->pq_b, c.w.T, N, H * H);   // identity: cast
    BG_TRY(check_launch("postquant_kernel launch"));
    BG_TRY(im2col2d(c, c.w.T, H, H, 3, 1, m->conv_in.kpad));
    BG_TRY(gemm(c, c.w.A, m->conv_in, c.N * H * H, x, nullptr, nullptr));
    for (int i = 0; i < 4; ++i) {
      for (int j = 0; j < 2; ++j) BG_TRY(resnet2d(c, m->s_down[i][j], &x, &spare, H * H, H));
      if (i < 3) {
        const Conv& dc = m->s_downconv[i];
        BG_TRY(cast_split(c, x, c.w.T, dc.cin, c.N * (size_t)H * H));
        BG_TRY(im2col2d(c, c.w.T, H, H, dc.cin, 1, dc.kpad, 2));
        H /= 2;
        BG_TRY(gemm(c, c.w.A, dc, c.N * H * H, spare, nullptr, nullptr));
        float* t = x; x = spare; spare = t;
      }
    }
    const int T = H * H;
    BG_TRY(resnet2d(c, m->s_mid[0], &x, &spare, T, H));
    BG_TRY(groupnorm(c, x, T, 512, 32, 1e-6f, m->s_attn.gn, 0, nullptr, nullptr, c.w.T));
    BG_TRY(gemm(c, c.w.T, m->s_attn.qkv, c.N * T, nullptr, c.w.Q, nullptr));
    BG_TRY(attention(c, T, 1, 512, 0.044194173824159216f));
    BG_TRY(gemm(c, c.w.Q + c.N * (size_t)T * 1536, m->s_attn.proj, c.N * T, x, nullptr, x));
    BG_TRY(resnet2d(c, m->s_mid[1], &x, &spare, T, H));
    BG_TRY(groupnorm(c, x, T, 512, 32, 1e-6f, m->norm_out, 1, nullptr, nullptr, c.w.T));
    BG_TRY(im2col2d(c, c.w.T, H, H, 512, 1, m->conv_out.kpad));
    BG_TRY(gemm(c, c.w.A, m->conv_out, c.N * T, c.w.H, nullptr, nullptr));
    quant_mode_kernel<<<(N * 3 * T + 255) / 256, 256, 0, c.st>>>(c.w.H, 128, m->q_w, m->q_b, out, N, T);
    return check_launch("quant_mode_kernel launch");
  }

  int L = 32;
  postquant_kernel<<<(N * L + 255) / 256, 256, 0, c.st>>>(xin, m->pq_w, m->pq_b, c.w.T, N, L);
  BG_TRY(check_launch("postquant_kernel launch"));
  BG_TRY(im2col1d(c, c.w.T, L, 3, 3, m->conv_in.kpad));
  BG_TRY(gemm(c, c.w.A, m->conv_in, c.N * L, x, nullptr, nullptr));
  for (int i = 0; i < 3; ++i) {
    const int C = m->e_down[i][0].c1.cin;
    const size_t tot = c.N * (size_t)(L / 2) * C;
    cubic_down1d_kernel<<<grid_for(tot), 256, 0, c.st>>>(x, spare, L, C, m->down_kernel, tot);
    BG_TRY(check_launch("cubic_down1d_kernel launch"));
    float* t = x; x = spare; spare = t;
    L /= 2;
    for (int j = 0; j < 3; ++j) BG_TRY(resconv1d(c, m->e_down[i][j], &x, &spare, L));
  }
  for (int i = 0; i < 6; ++i) {
    BG_TRY(resconv1d(c, m->e_mid[i], &x, &spare, 4));
    const Attn& a = m->e_attn[i];
    BG_TRY(groupnorm(c, x, 4, 512, 1, 1e-5f, a.gn, 0, nullptr, nullptr, c.w.T));
    BG_TRY(gemm(c, c.w.T, a.qkv, c.N * 4, nullptr, c.w.Q, nullptr));
    BG_TRY(attention(c, 4, 16, 32, 0.17677669529663687f));
    BG_TRY(gemm(c, c.w.Q + c.N * (size_t)4 * 1536, a.proj, c.N * 4, x, nullptr, x));
  }
  BG_TRY(groupnorm(c, x, 4, 512, 32, 1e-6f, m->norm_out, 1, nullptr, nullptr, c.w.T));
  BG_TRY(im2col1d(c, c.w.T, 4, 512, 3, m->conv_out.kpad));
  BG_TRY(gemm(c, c.w.A, m->conv_out, c.N * 4, c.w.H, nullptr, nullptr));
  quant_mode_kernel<<<(N * 3 * 4 + 255) / 256, 256, 0, c.st>>>(c.w.H, 128, m->q_w, m->q_b, out, N, 4);
  return check_launch("quant_mode_kernel launch");
}

}  // extern "C"
