// wgmma GEMM for sm_90a:  out[M,N] = epi( A[M,K] * W[N,K]^T ),  fp16 operands, fp32 accumulation in registers.
//
// This is the only dense linear contraction of the denoisers (reference: torch F.linear inside
// nn.TransformerEncoderLayer / the embed MLPs, network.py:1076-1099) and of the VAE convs (implicit GEMMs, ConvGeom).
// nn.Linear stores W as [N][K] row-major == K-major B operand, so weights are used as packed.
//
// Structure (one persistent CTA per SM, 384 threads = 3 warpgroups, tile 128 x BN, BN = 128 or 256):
//   warpgroup 0    : TMA producer (one elected thread: A tile 128x64, W tile BNx64, SWIZZLE_128B, STAGES-deep
//                    mbarrier ring); gives its registers to the consumers (setmaxnreg)
//   warpgroups 1-2 : consumers, one 64-row half of the tile each: 4 x wgmma m64nBNk16 per 64-wide k-block with both
//                    operands read from shared memory, one k-block in flight while the previous stage is released;
//                    the epilogue works straight from the accumulator registers while the producer already fills the
//                    ring for the next tile; the producer also prefetches the tile's residual rows into L2 when it
//                    starts the tile, so the epilogue's residual reads hit L2 rather than HBM
// Roofline: tensor-bound; 2*M*N*K flop per launch.
#include <stdlib.h>

#include "bg_internal.h"
#include "gemm_epilogue.cuh"
#include "ptx.cuh"

namespace bg {

namespace {

constexpr int BM = 128;
constexpr int BK = 64;

template <int BN>
struct Cfg {
  static constexpr int STAGES = (BN == 256) ? 4 : 6;
  static constexpr int A_BYTES = BM * BK * 2;
  static constexpr int B_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int BAR_BYTES = 256;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + BAR_BYTES + 1024;  // +1024: manual 1 KB alignment
};

template <int BN>
__device__ __forceinline__ void wgmma_tile_k16(float (&acc)[BN / 2], uint64_t a, uint64_t b, uint32_t accumulate) {
  if constexpr (BN == 256) wgmma_m64n256k16_ss(acc, a, b, accumulate);
  else wgmma_m64n128k16_ss(acc, a, b, accumulate);
}

template <int BN>
__global__ void __launch_bounds__(384, 1)
gemm_f16_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GemmParams p_in) {
  const GemmParams p = gemm_resolve(p_in);
  using C = Cfg<BN>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + C::STAGES * C::STAGE_BYTES);
  uint64_t* empty = full + C::STAGES;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = threadIdx.x >> 7;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int i = 0; i < C::STAGES; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], 256);     // every consumer thread releases the stage after its wgmma reads are complete
    }
    fence_barrier_init();
  }
  __syncthreads();

  const int num_m = (p.M + BM - 1) / BM;
  const int num_n = p.N / BN;
  const int num_tiles = num_m * num_n;
  const int num_k = p.K / BK;

  if (wg == 0) {
    setmaxnreg_dec<40>();
    if (warp == 0 && elect_one()) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int m_blk = tile / num_n, n_blk = tile % num_n;
        const int nk = (n_blk * BN < p.n_short) ? p.k_short / BK : num_k;
        gemm_prefetch_resid<BM, BN>(p, m_blk * BM, n_blk * BN);
        for (int kb = 0; kb < nk; ++kb) {
          mbar_wait(&empty[stage], phase ^ 1);
          uint8_t* sA = smem + stage * C::STAGE_BYTES;
          uint8_t* sB = sA + C::A_BYTES;
          mbar_arrive_expect_tx(&full[stage], C::STAGE_BYTES);
          if (p.conv_taps) {      // implicit convolution: the A tile is a shifted box of the channels-last image
            int c0, x, y, n;
            conv_coords(p, kb, m_blk * BM, c0, x, y, n);
            tma_load_4d(sA, &tmA, &full[stage], c0, x, y, n);
          } else {
            const int ka = p.a_kwrap ? (kb * BK) % p.a_kwrap : kb * BK;
            tma_load_2d(sA, &tmA, &full[stage], ka, m_blk * BM);
          }
          tma_load_2d(sB, &tmB, &full[stage], kb * BK, n_blk * BN);
          if (++stage == C::STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    setmaxnreg_inc<232>();
    const int half = wg - 1;                  // rows [64 half, 64 half + 64) of the tile
    float acc[BN / 2];
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int m_blk = tile / num_n, n_blk = tile % num_n;
      const int nk = (n_blk * BN < p.n_short) ? p.k_short / BK : num_k;
      int prev = -1;
      for (int kb = 0; kb < nk; ++kb) {
        mbar_wait(&full[stage], phase);
        const uint32_t a_addr = smem_u32(smem + stage * C::STAGE_BYTES) + half * 64 * 128;
        const uint32_t b_addr = smem_u32(smem + stage * C::STAGE_BYTES + C::A_BYTES);
        wgmma_fence_operand(acc);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k)
          wgmma_tile_k16<BN>(acc, make_sw128_desc(a_addr + k * 32), make_sw128_desc(b_addr + k * 32), (kb | k) != 0 ? 1u : 0u);
        wgmma_commit();
        wgmma_fence_operand(acc);
        wgmma_wait<1>();                      // the previous k-block's MMAs are done: release its stage
        if (prev >= 0) mbar_arrive(&empty[prev]);
        prev = stage;
        if (++stage == C::STAGES) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      wgmma_fence_operand(acc);
      mbar_arrive(&empty[prev]);
      gemm_epilogue_regs<BN>(p, acc, m_blk * BM + half * 64, n_blk * BN, warp & 3, lane);
    }
  }
}

template <int BN>
int launch_bn(cudaStream_t st, const CUtensorMap& tmA, const CUtensorMap& tmB, const GemmParams& p) {
  using C = Cfg<BN>;
  BG_TRY(ensure_dynamic_smem(reinterpret_cast<const void*>(&gemm_f16_kernel<BN>), C::SMEM_BYTES));
  const int num_tiles = ((p.M + BM - 1) / BM) * (p.N / BN);
  const int grid = num_tiles < num_sms() ? num_tiles : num_sms();
  gemm_f16_kernel<BN><<<grid, 384, C::SMEM_BYTES, st>>>(tmA, tmB, p);
  return check_launch("gemm_f16_kernel launch");
}

}  // namespace

int launch_gemm_f16(cudaStream_t st, const __half* A, int lda, const __half* W, int ldw, int M, int N, int K,
                    const GemmEpilogue& ep) {
  BG_REQUIRE(M > 0 && N > 0 && K > 0, "gemm: empty problem");
  BG_REQUIRE(K % BK == 0, "gemm: K must be a multiple of 64");
  BG_REQUIRE(N % 128 == 0, "gemm: N must be a multiple of 128");
  BG_REQUIRE(lda % 8 == 0 && ldw % 8 == 0, "gemm: operand pitch must be a multiple of 8 elements (16 B)");
  BG_REQUIRE((reinterpret_cast<uintptr_t>(A) & 15) == 0 && (reinterpret_cast<uintptr_t>(W) & 15) == 0,
             "gemm: operands must be 16-byte aligned");
  BG_REQUIRE(ep.out != nullptr && ep.ldo % 8 == 0, "gemm: output pitch must be a multiple of 8");
  BG_REQUIRE((reinterpret_cast<uintptr_t>(ep.out) & 15) == 0, "gemm: output must be 16-byte aligned");
  BG_REQUIRE(ep.resid == nullptr || (ep.ldr % 4 == 0 && !ep.out_f16 ? true : ep.ldr % 4 == 0), "gemm: resid pitch");
  BG_REQUIRE(ep.rowvec == nullptr || (ep.rows_per_vec > 0 && ep.ldv % 4 == 0), "gemm: rowvec");
  BG_REQUIRE(!ep.out_f16 || (ep.resid == nullptr && ep.rowvec == nullptr), "gemm: fp16 output supports bias / ReLU only");
  // the epilogue reads bias and residual as column pairs (float2)
  BG_REQUIRE((reinterpret_cast<uintptr_t>(ep.bias) & 7) == 0, "gemm: bias must be 8-byte aligned");
  BG_REQUIRE((reinterpret_cast<uintptr_t>(ep.resid) & 7) == 0, "gemm: resid must be 8-byte aligned");
  // Tile selection: 128 x 256 tiles halve the A traffic per flop; when they would leave SMs idle (the surface stages:
  // M = B x S of a few thousand rows) 128 x 128 tiles give twice as many tiles with a main loop of half the length.
  int bn = (N % 256 == 0) ? 256 : 128;
  if (bn == 256 && (long long)((M + BM - 1) / BM) * (N / 256) < num_sms()) bn = 128;
  CUtensorMap tmA, tmB;
  const int a_cols = ep.a_kwrap > 0 ? ep.a_kwrap : K;
  BG_REQUIRE(ep.a_kwrap == 0 || (ep.a_kwrap % BK == 0 && ep.a_kwrap <= K), "gemm: a_kwrap must be a multiple of 64");
  const ConvGeom& cg = ep.conv;
  if (cg.taps > 0) {
    const int hw = cg.W * cg.H;
    BG_REQUIRE(cg.C > 0 && cg.C % 64 == 0 && cg.W > 0 && cg.H > 0 && cg.N > 0 && cg.kw > 0 && cg.taps % cg.kw == 0,
               "conv gemm: bad geometry");
    BG_REQUIRE(128 % cg.W == 0 && (hw % 128 == 0 || 128 % hw == 0), "conv gemm: W * H must divide 128 or be a multiple of it");
    BG_REQUIRE(M == cg.N * hw && K == cg.terms * cg.taps * cg.C && ep.a_kwrap == 0, "conv gemm: M / K do not match the geometry");
    BG_REQUIRE(lda >= (cg.lo_plane ? 2 : 1) * cg.C, "conv gemm: channel pitch too small");
    const int box_h = hw >= 128 ? 128 / cg.W : cg.H, box_n = hw >= 128 ? 1 : 128 / hw;
    BG_TRY(make_tmap_4d_f16(&tmA, A, (uint64_t)(cg.lo_plane ? 2 : 1) * cg.C, cg.W, cg.H, cg.N, (uint64_t)lda, cg.W, box_h, box_n));
  } else {
    BG_TRY(make_tmap_2d_f16(&tmA, A, (uint64_t)M, (uint64_t)a_cols, (uint64_t)lda, BM));
  }
  BG_TRY(make_tmap_2d_f16(&tmB, W, (uint64_t)N, (uint64_t)K, (uint64_t)ldw, (uint32_t)bn));
  GemmParams p;
  p.M = M; p.N = N; p.K = K; p.a_kwrap = ep.a_kwrap; p.m_dev = ep.m_dev; p.row_map = ep.row_map;
  p.n_short = ep.n_short; p.k_short = ep.k_short;
  BG_REQUIRE(ep.n_short == 0 || (ep.n_short % 256 == 0 && ep.k_short % BK == 0 && ep.k_short > 0 && ep.k_short <= K),
             "gemm: n_short must be a multiple of 256 and k_short a multiple of 64");
  p.out = ep.out; p.ldo = ep.ldo; p.out_f16 = ep.out_f16; p.relu = ep.relu;
  p.bias = ep.bias; p.resid = ep.resid; p.ldr = ep.ldr;
  p.rowvec = ep.rowvec; p.rows_per_vec = ep.rows_per_vec; p.ldv = ep.ldv;
  p.conv_taps = cg.taps; p.conv_kw = cg.kw; p.conv_cpb = cg.C / 64; p.conv_C = cg.C; p.conv_W = cg.W; p.conv_HW = cg.W * cg.H;
  p.conv_pad_w = cg.kw / 2; p.conv_pad_h = cg.taps > 0 ? (cg.taps / cg.kw) / 2 : 0;
  p.conv_lo_term = (cg.taps > 0 && cg.lo_plane && cg.terms == 3) ? 1 : -1;
  return bn == 256 ? launch_bn<256>(st, tmA, tmB, p) : launch_bn<128>(st, tmA, tmB, p);
}

}  // namespace bg
