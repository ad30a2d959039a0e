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


// Warms L2 with the residual rows of the tile [row0, row0 + BM) x [col0, col0 + BN): one bulk prefetch per row, issued
// by the producer thread when it starts the tile, so the bytes arrive while the tile's MMAs run and the epilogue reads
// them from L2 instead of HBM.  The range is widened to 16-byte boundaries (the bulk-copy granule); the widened ends lie
// in granules that hold bytes of the row, so no address outside mapped memory is touched.
template <int BM, int BN>
__device__ __forceinline__ void gemm_prefetch_resid(const GemmParams& p, int row0, int col0) {
  if (!p.resid || p.out_f16) return;
  const int rows = min(BM, p.M - row0);
  for (int r = 0; r < rows; ++r) {
    const uintptr_t a = reinterpret_cast<uintptr_t>(p.resid + (size_t)(row0 + r) * p.ldr + col0);
    const uintptr_t lo = a & ~uintptr_t(15), hi = (a + BN * sizeof(float) + 15) & ~uintptr_t(15);
    prefetch_l2_bulk(reinterpret_cast<const void*>(lo), (uint32_t)(hi - lo));
  }
}

// One consumer warpgroup, one 64 x BN accumulator tile held in registers in the wgmma m64nBN fp32 layout: warp w of
// the warpgroup owns rows 16w + lane / 4 (acc[4i], acc[4i + 1]) and 16w + 8 + lane / 4 (acc[4i + 2], acc[4i + 3]) at
// columns 8i + 2 (lane % 4) + {0, 1}.  Each quad of lanes therefore covers 8 contiguous columns (32 B in fp32) of a row,
// and the epilogue works on column pairs: float2 loads of bias / residual, float2 or half2 stores.
//
// Per row and group of EPI_GROUP column pairs, two passes: the first adds bias, row vector and residual into acc, the
// second applies ReLU, converts and stores.  `out` and `resid` may be the same array (the in-place residual stream), so
// the compiler cannot hoist a residual load above a store; with a group's loads ahead of its stores they are in flight
// together instead of one or two at a time.  Each thread reads only the elements it writes, so the order is safe.  The
// group size bounds the registers the loads in flight take (the accumulators already hold BN / 2 of them).
//
// fp16 outputs (bias and ReLU only) are stored 16 B per lane: the four lanes of a quad transpose their packed column
// pairs of four consecutive 8-column groups by shuffles, so that lane q holds all 8 columns of group q, and the quad writes
// 64 contiguous bytes of its row (two whole 32 B sectors) with one store instead of four half-sector stores.
constexpr int EPI_GROUP = 8;

template <int BN>
__device__ __forceinline__ void gemm_epilogue_f16(const GemmParams& p, const float (&acc)[BN / 2], int row0, int col0,
                                                  int warp_in_wg, int lane) {
  const int q = lane & 3;
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    const int row = row0 + warp_in_wg * 16 + hr * 8 + (lane >> 2);
    __half* orow = reinterpret_cast<__half*>(p.out) + (size_t)row * p.ldo + col0;
#pragma unroll
    for (int i0 = 0; i0 < BN / 8; i0 += 4) {
      uint32_t u[4];         // this lane's column pair of groups i0 .. i0 + 3
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int i = i0 + j;
        float v0 = acc[4 * i + 2 * hr], v1 = acc[4 * i + 2 * hr + 1];
        if (p.bias) {
          const float2 b = __ldg(reinterpret_cast<const float2*>(p.bias + col0 + 8 * i + 2 * q));
          v0 += b.x;
          v1 += b.y;
        }
        if (p.relu) {
          v0 = fmaxf(v0, 0.f);
          v1 = fmaxf(v1, 0.f);
        }
        u[j] = pack_half2(v0, v1);
      }
      // 4 x 4 transpose within the quad in two butterfly steps (lane bit 0, then bit 1), all register indices static.
      // The whole warp takes part, rows past M included, so the shuffles stay convergent; only the store is guarded.
      const bool b0 = q & 1, b1 = q & 2;
      const uint32_t x0 = __shfl_xor_sync(0xffffffffu, b0 ? u[0] : u[1], 1);
      const uint32_t x1 = __shfl_xor_sync(0xffffffffu, b0 ? u[2] : u[3], 1);
      const uint32_t t0 = b0 ? x0 : u[0], t1 = b0 ? u[1] : x0, t2 = b0 ? x1 : u[2], t3 = b0 ? u[3] : x1;
      const uint32_t y0 = __shfl_xor_sync(0xffffffffu, b1 ? t0 : t2, 2);
      const uint32_t y1 = __shfl_xor_sync(0xffffffffu, b1 ? t1 : t3, 2);
      const uint4 w = b1 ? make_uint4(y0, y1, t2, t3) : make_uint4(t0, t1, y0, y1);   // lane q: group i0 + q
      if (row < p.M) *reinterpret_cast<uint4*>(orow + 8 * (i0 + q)) = w;
    }
  }
}

template <int BN>
__device__ __forceinline__ void gemm_epilogue_regs(const GemmParams& p, float (&acc)[BN / 2], int row0, int col0,
                                                   int warp_in_wg, int lane) {
  // The loop below still tests out_f16, although fp16 outputs never reach it.  Without those tests the compiler
  // scheduled the fp32 path differently, and linear2 measured 2-4 % slower.
  if (p.out_f16) {
    gemm_epilogue_f16<BN>(p, acc, row0, col0, warp_in_wg, lane);
    return;
  }
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    const int row = row0 + warp_in_wg * 16 + hr * 8 + (lane >> 2);
    if (row >= p.M) continue;
    const float* rv = (p.rowvec && !p.out_f16)
                          ? p.rowvec + (size_t)((p.row_map ? p.row_map[row] : row) / p.rows_per_vec) * p.ldv : nullptr;
    const float* rs = (p.resid && !p.out_f16) ? p.resid + (size_t)row * p.ldr : nullptr;
#pragma unroll
    for (int g = 0; g < BN / 8; g += EPI_GROUP) {
#pragma unroll
      for (int i = g; i < g + EPI_GROUP; ++i) {
        const int col = col0 + 8 * i + 2 * (lane & 3);
        float& v0 = acc[4 * i + 2 * hr];
        float& v1 = acc[4 * i + 2 * hr + 1];
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
      }
#pragma unroll
      for (int i = g; i < g + EPI_GROUP; ++i) {
        const int col = col0 + 8 * i + 2 * (lane & 3);
        float v0 = acc[4 * i + 2 * hr], v1 = acc[4 * i + 2 * hr + 1];
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
}

}  // namespace bg
