// Parameters, implicit-convolution coordinates and register epilogue of the wgmma GEMM kernel (gemm.cu).
#pragma once
#include "bg_internal.h"
#include "ptx.cuh"

namespace bg {

struct GemmParams {
  int M, N, K;
  int a_kwrap;   // 0, or the K period of A: A column = k % a_kwrap (K-concatenated weights [W_hi | W_lo] reuse A)
  void* out;
  int ldo;
  int out_f16;
  int relu;
  const float* bias;
  const float* resid;
  int ldr;
  const float* rowvec;
  int rows_per_vec;
  int ldv;
  int n_short, k_short; // column tiles with n0 < n_short run only k_short / 64 k-blocks (partly split weight matrix)
  const int* m_dev;     // optional device int: the kernels work on min(M, *m_dev) rows (token compaction)
  const int* row_map;   // optional: rowvec row = row_map[row] / rows_per_vec
  // implicit-GEMM convolution (conv_taps > 0): see ConvGeom in bg_internal.h
  int conv_taps, conv_kw, conv_cpb /* C / 64 */, conv_C, conv_W, conv_HW, conv_pad_w, conv_pad_h, conv_lo_term;
};

// coordinates of the A box of k-block kb for the tile whose first row (output pixel) is row0: {channel, x, y, image}
__device__ __forceinline__ void conv_coords(const GemmParams& p, int kb, int row0, int& c0, int& x, int& y, int& n) {
  const int per_term = p.conv_taps * p.conv_cpb;
  const int term = kb / per_term, r = kb - term * per_term;
  const int tap = r / p.conv_cpb, cc = r - tap * p.conv_cpb;
  c0 = (term == p.conv_lo_term ? p.conv_C : 0) + cc * 64;
  x = tap % p.conv_kw - p.conv_pad_w;
  n = row0 / p.conv_HW;
  y = (row0 - n * p.conv_HW) / p.conv_W + tap / p.conv_kw - p.conv_pad_h;
}

// the kernels' working copy of the parameters with the row count resolved on the device
__device__ __forceinline__ GemmParams gemm_resolve(const GemmParams& p) {
  GemmParams q = p;
  if (p.m_dev) q.M = min(p.M, *p.m_dev);
  return q;
}


// One consumer warpgroup, one 64 x BN accumulator tile held in registers in the wgmma m64nBN fp32 layout: warp w of
// the warpgroup owns rows 16w + lane / 4 (acc[4i], acc[4i + 1]) and 16w + 8 + lane / 4 (acc[4i + 2], acc[4i + 3]) at
// columns 8i + 2 (lane % 4) + {0, 1}.  Each quad of lanes therefore covers 8 contiguous columns (32 B in fp32) of a row,
// and the epilogue works on column pairs: float2 loads of bias / residual, float2 or half2 stores.
template <int BN>
__device__ __forceinline__ void gemm_epilogue_regs(const GemmParams& p, const float (&acc)[BN / 2], int row0, int col0,
                                                   int warp_in_wg, int lane) {
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    const int row = row0 + warp_in_wg * 16 + hr * 8 + (lane >> 2);
    if (row >= p.M) continue;
    const float* rv = (p.rowvec && !p.out_f16)
                          ? p.rowvec + (size_t)((p.row_map ? p.row_map[row] : row) / p.rows_per_vec) * p.ldv : nullptr;
    const float* rs = (p.resid && !p.out_f16) ? p.resid + (size_t)row * p.ldr : nullptr;
#pragma unroll
    for (int i = 0; i < BN / 8; ++i) {
      const int col = col0 + 8 * i + 2 * (lane & 3);
      float v0 = acc[4 * i + 2 * hr], v1 = acc[4 * i + 2 * hr + 1];
      if (p.bias) {
        const float2 b = __ldg(reinterpret_cast<const float2*>(p.bias + col));
        v0 += b.x;
        v1 += b.y;
      }
      if (rv) {
        v0 += __ldg(rv + col);
        v1 += __ldg(rv + col + 1);
      }
      if (rs) {
        const float2 r = *reinterpret_cast<const float2*>(rs + col);
        v0 += r.x;
        v1 += r.y;
      }
      if (p.relu) {
        v0 = fmaxf(v0, 0.f);
        v1 = fmaxf(v1, 0.f);
      }
      if (p.out_f16)
        *reinterpret_cast<uint32_t*>(reinterpret_cast<__half*>(p.out) + (size_t)row * p.ldo + col) = pack_half2(v0, v1);
      else
        *reinterpret_cast<float2*>(reinterpret_cast<float*>(p.out) + (size_t)row * p.ldo + col) = make_float2(v0, v1);
    }
  }
}

}  // namespace bg
