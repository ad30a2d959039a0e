// CUDA-core kernels around the tensor-core contractions: LayerNorm -> fp16, the tiny-K / tiny-N ends of the embed
// MLPs, conditioning vectors, casts.  All HBM-bound: coalesced 16-byte accesses, one warp per token row.
//
// Reference: the Linear -> LayerNorm -> SiLU -> Linear embed MLPs and norm1/norm2/final norm of the encoder,
// network.py:1080-1099 (and the analogous blocks of the other three nets); sincos_embedding :1043-1063.
#include <math.h>

#include "bg_internal.h"

namespace bg {

namespace {

constexpr int D = 768;
constexpr float LN_EPS = 1e-5f;

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float silu(float x) { return x / (1.f + __expf(-x)); }

// v[24] holds row elements {lane*4 + 128*j + i}; normalise in place (two-pass, fp32)
__device__ __forceinline__ void ln_row(float (&v)[24], const float* __restrict__ g, const float* __restrict__ b, int lane,
                                       int act) {
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < 24; ++i) s += v[i];
  const float mean = warp_sum(s) * (1.f / D);
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < 24; ++i) {
    const float d = v[i] - mean;
    q += d * d;
  }
  const float rstd = rsqrtf(warp_sum(q) * (1.f / D) + LN_EPS);
#pragma unroll
  for (int j = 0; j < 6; ++j) {
    const float4 gg = __ldg(reinterpret_cast<const float4*>(g + lane * 4 + 128 * j));
    const float4 bb = __ldg(reinterpret_cast<const float4*>(b + lane * 4 + 128 * j));
    float y0 = (v[4 * j] - mean) * rstd * gg.x + bb.x;
    float y1 = (v[4 * j + 1] - mean) * rstd * gg.y + bb.y;
    float y2 = (v[4 * j + 2] - mean) * rstd * gg.z + bb.z;
    float y3 = (v[4 * j + 3] - mean) * rstd * gg.w + bb.w;
    if (act == 1) { y0 = silu(y0); y1 = silu(y1); y2 = silu(y2); y3 = silu(y3); }
    v[4 * j] = y0; v[4 * j + 1] = y1; v[4 * j + 2] = y2; v[4 * j + 3] = y3;
  }
}

__device__ __forceinline__ void store_row_f16(const float (&v)[24], __half* y, int lane, int lo_offset = 0) {
#pragma unroll
  for (int j = 0; j < 6; ++j) {
    __half2 h0 = __floats2half2_rn(v[4 * j], v[4 * j + 1]);
    __half2 h1 = __floats2half2_rn(v[4 * j + 2], v[4 * j + 3]);
    uint2 u;
    u.x = *reinterpret_cast<uint32_t*>(&h0);
    u.y = *reinterpret_cast<uint32_t*>(&h1);
    *reinterpret_cast<uint2*>(y + lane * 4 + 128 * j) = u;
    if (lo_offset > 0) {   // rounding residual, exactly representable difference of two nearby floats
      const float2 f0 = __half22float2(h0), f1 = __half22float2(h1);
      __half2 l0 = __floats2half2_rn(v[4 * j] - f0.x, v[4 * j + 1] - f0.y);
      __half2 l1 = __floats2half2_rn(v[4 * j + 2] - f1.x, v[4 * j + 3] - f1.y);
      u.x = *reinterpret_cast<uint32_t*>(&l0);
      u.y = *reinterpret_cast<uint32_t*>(&l1);
      *reinterpret_cast<uint2*>(y + lo_offset + lane * 4 + 128 * j) = u;
    }
  }
}

__global__ void __launch_bounds__(256) layernorm_f16_kernel(const float* __restrict__ x, int ldx, const float* __restrict__ g,
                                                            const float* __restrict__ b, __half* __restrict__ y, int ldy,
                                                            int rows, int act, int lo_offset,
                                                            const int* __restrict__ rows_dev) {
  const int lane = threadIdx.x & 31;
  const int wpb = blockDim.x >> 5;
  if (rows_dev) rows = min(rows, *rows_dev);      // token compaction: the number of valid rows lives on the device
  for (int row = blockIdx.x * wpb + (threadIdx.x >> 5); row < rows; row += gridDim.x * wpb) {
    const float* xr = x + (size_t)row * ldx;
    float v[24];
#pragma unroll
    for (int j = 0; j < 6; ++j) {
      const float4 t = *reinterpret_cast<const float4*>(xr + lane * 4 + 128 * j);
      v[4 * j] = t.x; v[4 * j + 1] = t.y; v[4 * j + 2] = t.z; v[4 * j + 3] = t.w;
    }
    ln_row(v, g, b, lane, act);
    store_row_f16(v, y + (size_t)row * ldy, lane, lo_offset);
  }
}

// Linear(d_in -> 768) + LayerNorm + SiLU -> fp16.  W0t: [d_in][768].
__global__ void __launch_bounds__(256) embed_in_kernel(const float* __restrict__ x, int ldx, int d_in,
                                                       const float* __restrict__ W0t, const float* __restrict__ b0,
                                                       const float* __restrict__ g, const float* __restrict__ b,
                                                       __half* __restrict__ y, int ldy, int rows,
                                                       const int* __restrict__ rows_dev, const int* __restrict__ row_map) {
  const int lane = threadIdx.x & 31;
  const int wpb = blockDim.x >> 5;
  if (rows_dev) rows = min(rows, *rows_dev);
  for (int row = blockIdx.x * wpb + (threadIdx.x >> 5); row < rows; row += gridDim.x * wpb) {
    const float* xr = x + (size_t)(row_map ? row_map[row] : row) * ldx;      // compaction: gather the source token
    float v[24];
#pragma unroll
    for (int j = 0; j < 6; ++j) {
      const float4 t = __ldg(reinterpret_cast<const float4*>(b0 + lane * 4 + 128 * j));
      v[4 * j] = t.x; v[4 * j + 1] = t.y; v[4 * j + 2] = t.z; v[4 * j + 3] = t.w;
    }
    for (int k = 0; k < d_in; ++k) {
      const float xk = __ldg(xr + k);
      const float* wr = W0t + (size_t)k * D;
#pragma unroll
      for (int j = 0; j < 6; ++j) {
        const float4 t = __ldg(reinterpret_cast<const float4*>(wr + lane * 4 + 128 * j));
        v[4 * j] = fmaf(xk, t.x, v[4 * j]);
        v[4 * j + 1] = fmaf(xk, t.y, v[4 * j + 1]);
        v[4 * j + 2] = fmaf(xk, t.z, v[4 * j + 2]);
        v[4 * j + 3] = fmaf(xk, t.w, v[4 * j + 3]);
      }
    }
    ln_row(v, g, b, lane, 1);
    store_row_f16(v, y + (size_t)row * ldy, lane);
  }
}

// out[row, o] = bias[o] + sum_k SiLU(LN(x[row]))[k] W[o,k];  all fp32; warp per row, W ([d_out][768]) in shared memory.
// (fc_out.1 -> SiLU -> fc_out.3 of network.py:1094-1099; fused so the hidden vector never leaves registers.)
__global__ void __launch_bounds__(256) ln_silu_head_kernel(const float* __restrict__ x, int ldx, const float* __restrict__ g,
                                                           const float* __restrict__ b, const float* __restrict__ W,
                                                           const float* __restrict__ bias, float* __restrict__ out, int d_out,
                                                           int rows, const int* __restrict__ rows_dev,
                                                           const int* __restrict__ row_map) {
  extern __shared__ float sW[];   // [d_out][768]
  if (rows_dev) rows = min(rows, *rows_dev);
  for (int i = threadIdx.x; i < d_out * D / 4; i += blockDim.x)
    reinterpret_cast<float4*>(sW)[i] = __ldg(reinterpret_cast<const float4*>(W) + i);
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int wpb = blockDim.x >> 5;
  for (int row = blockIdx.x * wpb + (threadIdx.x >> 5); row < rows; row += gridDim.x * wpb) {
    const float* xr = x + (size_t)row * ldx;
    float v[24];
#pragma unroll
    for (int j = 0; j < 6; ++j) {
      const float4 t = *reinterpret_cast<const float4*>(xr + lane * 4 + 128 * j);
      v[4 * j] = t.x; v[4 * j + 1] = t.y; v[4 * j + 2] = t.z; v[4 * j + 3] = t.w;
    }
    ln_row(v, g, b, lane, 1);
    float mine = 0.f;
    for (int o = 0; o < d_out; ++o) {
      const float* wr = sW + o * D;
      float acc = 0.f;
#pragma unroll
      for (int j = 0; j < 6; ++j) {
        const float4 t = *reinterpret_cast<const float4*>(wr + lane * 4 + 128 * j);
        acc = fmaf(v[4 * j], t.x, acc);
        acc = fmaf(v[4 * j + 1], t.y, acc);
        acc = fmaf(v[4 * j + 2], t.z, acc);
        acc = fmaf(v[4 * j + 3], t.w, acc);
      }
      acc = warp_sum(acc);
      if ((o & 31) == lane) mine = acc + __ldg(bias + o);
      if ((o & 31) == 31 || o == d_out - 1) {
        const int o0 = o & ~31;
        if (o0 + lane <= o) out[(size_t)(row_map ? row_map[row] : row) * d_out + o0 + lane] = mine;   // compaction: scatter
      }
    }
  }
}

__global__ void cond_kernel(const float* __restrict__ time_table, const int64_t* __restrict__ t, int n_t,
                            const float* __restrict__ class_table, const int64_t* __restrict__ label,
                            float* __restrict__ cond, int B) {
  const int b = blockIdx.x;
  // A timestep outside the 1000-row table or a class label outside the 11-row embedding is an error in the caller (the
  // reference's nn.Embedding raises a device assert).  There is no error channel from a stream-ordered kernel, so the
  // sample's conditioning is poisoned with NaN instead of reading out of bounds: every output of that sample is NaN.
  const long long tt = t[n_t == 1 ? 0 : b];
  const long long lb = class_table ? label[b] : 0;
  const bool bad = tt < 0 || tt > 999 || lb < 0 || lb >= 11;
  const float* tr = time_table + (size_t)(bad ? 0 : tt) * D;
  const float* cr = class_table ? class_table + (size_t)(bad ? 0 : lb) * D : nullptr;
  const float poison = bad ? __int_as_float(0x7fc00000) : 0.f;
  for (int i = threadIdx.x; i < D; i += blockDim.x) cond[(size_t)b * D + i] = tr[i] + (cr ? cr[i] : 0.f) + poison;
}

__global__ void sincos_table_kernel(float* __restrict__ out, int n) {
  const int t = blockIdx.x;
  if (t >= n) return;
  for (int i = threadIdx.x; i < D / 2; i += blockDim.x) {
    // fp32 like the reference: freqs = exp(-ln(1e4) * i / 384); args = float(t) * freqs
    const float f = expf(-9.210340371976184f * (float)i / 384.f);
    const float a = (float)t * f;
    out[(size_t)t * D + i] = cosf(a);
    out[(size_t)t * D + D / 2 + i] = sinf(a);
  }
}

__global__ void cast_kernel(const float* __restrict__ x, __half* __restrict__ y, size_t n) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) y[i] = __float2half_rn(x[i]);
}

__global__ void mask_expand_kernel(const uint8_t* __restrict__ face_mask, uint8_t* __restrict__ edge_mask, int BS, int E) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < BS * E) edge_mask[i] = face_mask[i / E];
}

// ---- mask-aware token compaction (SURVEY.md 0.7 / 8a row 10: padded tokens are never attended to and their outputs are
// discarded downstream, sample.py:245,284, so dropping them is result-preserving for the valid tokens) ----
// pass 1 (grid B): seq_len[b] = number of valid tokens of sample b
__global__ void compact_count_kernel(const uint8_t* __restrict__ mask, int L, int* __restrict__ seq_len) {
  const int b = blockIdx.x;
  int n = 0;
  for (int i = threadIdx.x; i < L; i += blockDim.x) n += mask[(size_t)b * L + i] == 0;
  n = (int)warp_sum((float)n);           // counts <= 8192 per warp: exact in fp32
  __shared__ int part[8];
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = n;
  __syncthreads();
  if (threadIdx.x == 0) {
    int t = 0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += part[w];
    seq_len[b] = t;
  }
}
// pass 2 (one block): seq_row0 = exclusive prefix sum of seq_len, m_valid = total
__global__ void compact_scan_kernel(const int* __restrict__ seq_len, int B, int* __restrict__ seq_row0, int* __restrict__ m_valid) {
  if (threadIdx.x == 0) {
    int acc = 0;
    for (int b = 0; b < B; ++b) {
      seq_row0[b] = acc;
      acc += seq_len[b];
    }
    *m_valid = acc;
  }
}
// pass 3 (grid B, one warp): row_map[seq_row0[b] + rank] = b * L + token for the valid tokens in order
__global__ void compact_map_kernel(const uint8_t* __restrict__ mask, int L, const int* __restrict__ seq_row0,
                                   int* __restrict__ row_map) {
  const int b = blockIdx.x, lane = threadIdx.x;
  int base = seq_row0[b];
  for (int i0 = 0; i0 < L; i0 += 32) {
    const int i = i0 + lane;
    const bool ok = i < L && mask[(size_t)b * L + i] == 0;
    const uint32_t bal = __ballot_sync(0xffffffffu, ok);
    if (ok) row_map[base + __popc(bal & ((1u << lane) - 1))] = b * L + i;
    base += __popc(bal);
  }
}

// zero `nrows` rows of a fp16 matrix starting at row *row0_dev (clipped to max_rows): the variable-length attention reads up
// to 127 rows past the last valid token (masked keys, p = 0) and 0 x NaN from stale memory must not reach the accumulator
__global__ void zero_rows_kernel(__half* __restrict__ y, int ld, int cols, const int* __restrict__ row0_dev, int nrows, int max_rows) {
  const int r0 = *row0_dev;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < nrows * (cols / 8); i += gridDim.x * blockDim.x) {
    const int r = r0 + i / (cols / 8), c = (i % (cols / 8)) * 8;
    if (r < max_rows) *reinterpret_cast<uint4*>(y + (size_t)r * ld + c) = make_uint4(0, 0, 0, 0);
  }
}

inline int row_grid(int rows, int wpb) {
  const int want = (rows + wpb - 1) / wpb;
  const int cap = num_sms() * 8;
  return want < cap ? (want > 0 ? want : 1) : cap;
}

}  // namespace

int launch_layernorm_f16(cudaStream_t st, const float* x, int ldx, const float* g, const float* b, __half* y, int ldy,
                         int rows, int act, int lo_offset, const int* rows_dev) {
  BG_REQUIRE(rows > 0 && ldx % 4 == 0 && ldy % 4 == 0 && lo_offset % 4 == 0, "layernorm: bad shape");
  layernorm_f16_kernel<<<row_grid(rows, 8), 256, 0, st>>>(x, ldx, g, b, y, ldy, rows, act, lo_offset, rows_dev);
  return check_launch("layernorm_f16_kernel launch");
}

int launch_embed_in(cudaStream_t st, const float* x, int ldx, int d_in, const float* W0t, const float* b0, const float* g,
                    const float* b, __half* y, int ldy, int rows, const int* rows_dev, const int* row_map) {
  BG_REQUIRE(rows > 0 && d_in > 0 && ldy % 4 == 0, "embed_in: bad shape");
  embed_in_kernel<<<row_grid(rows, 8), 256, 0, st>>>(x, ldx, d_in, W0t, b0, g, b, y, ldy, rows, rows_dev, row_map);
  return check_launch("embed_in_kernel launch");
}

int launch_ln_silu_head(cudaStream_t st, const float* x, int ldx, const float* g, const float* b, const float* W,
                        const float* bias, float* out, int d_out, int rows, const int* rows_dev, const int* row_map) {
  BG_REQUIRE(rows > 0 && d_out > 0 && d_out <= 64 && ldx % 4 == 0, "ln_silu_head: bad shape");
  const int smem = d_out * D * 4;
  BG_TRY(ensure_dynamic_smem(reinterpret_cast<const void*>(&ln_silu_head_kernel), 64 * D * 4));
  const int want = (rows + 7) / 8;
  const int cap = num_sms() * 2;
  ln_silu_head_kernel<<<want < cap ? want : cap, 256, smem, st>>>(x, ldx, g, b, W, bias, out, d_out, rows, rows_dev, row_map);
  return check_launch("ln_silu_head_kernel launch");
}

int launch_compact(cudaStream_t st, const uint8_t* mask, int B, int L, int* seq_len, int* seq_row0, int* m_valid, int* row_map) {
  BG_REQUIRE(mask && B > 0 && L > 0 && seq_len && seq_row0 && m_valid && row_map, "compact: bad arguments");
  compact_count_kernel<<<B, 256, 0, st>>>(mask, L, seq_len);
  compact_scan_kernel<<<1, 32, 0, st>>>(seq_len, B, seq_row0, m_valid);
  compact_map_kernel<<<B, 32, 0, st>>>(mask, L, seq_row0, row_map);
  return check_launch("compact kernels launch");
}

int launch_zero_rows_f16(cudaStream_t st, __half* y, int ld, int cols, const int* row0_dev, int nrows, int max_rows) {
  BG_REQUIRE(y && row0_dev && cols % 8 == 0 && ld % 8 == 0 && nrows > 0, "zero_rows: bad arguments");
  zero_rows_kernel<<<64, 256, 0, st>>>(y, ld, cols, row0_dev, nrows, max_rows);
  return check_launch("zero_rows_kernel launch");
}

int launch_cond(cudaStream_t st, const float* time_table, const int64_t* t, int n_t, const float* class_table,
                const int64_t* label, float* cond, int B) {
  BG_REQUIRE(B > 0 && (n_t == 1 || n_t == B), "cond: timesteps must have 1 or B entries");
  BG_REQUIRE(class_table == nullptr || label != nullptr, "cond: class table without labels");
  cond_kernel<<<B, 256, 0, st>>>(time_table, t, n_t, class_table, label, cond, B);
  return check_launch("cond_kernel launch");
}

int launch_sincos_table(cudaStream_t st, float* out, int n) {
  sincos_table_kernel<<<n, 128, 0, st>>>(out, n);
  return check_launch("sincos_table_kernel launch");
}

int launch_cast_f32_to_f16(cudaStream_t st, const float* x, __half* y, size_t n) {
  if (n == 0) return BG_OK;
  size_t blocks = (n + 255) / 256;
  if (blocks > (size_t)num_sms() * 16) blocks = (size_t)num_sms() * 16;
  cast_kernel<<<(unsigned)blocks, 256, 0, st>>>(x, y, n);
  return check_launch("cast_kernel launch");
}

int launch_mask_expand(cudaStream_t st, const uint8_t* face_mask, uint8_t* edge_mask, int BS, int E) {
  const int n = BS * E;
  mask_expand_kernel<<<(n + 255) / 256, 256, 0, st>>>(face_mask, edge_mask, BS, E);
  return check_launch("mask_expand_kernel launch");
}

}  // namespace bg
