// wgmma GEMM for sm_90a:  out[M,N] = epi( A[M,K] * W[N,K]^T ),  fp16 operands, fp32 accumulation in registers.
//
// This is the only dense linear contraction of the denoisers (reference: torch F.linear inside
// nn.TransformerEncoderLayer / the embed MLPs, network.py:1076-1099) and of the VAE convs (implicit GEMMs, ConvGeom).
// nn.Linear stores W as [N][K] row-major == K-major B operand, so weights are used as packed.
//
// Two kernels; launch_gemm_f16 picks one per call:
//   gemm_pp_kernel  the plain 2-D forms with fp32 output (in-place residual, bias, ReLU, a_kwrap, n_short / k_short,
//                   m_dev): out_proj, linear2 and fc_out.  Ping-pong over whole tiles so that each epilogue overlaps MMAs.
//   gemm_f16_kernel fp16 outputs (QKV, linear1), the implicit convolutions (ConvGeom), the row-vector form (token
//                   embedding), residuals TMA cannot address, and every form when BREPGEN_B200_GEMM_PINGPONG=0.
//
// gemm_pp_kernel (one persistent CTA per SM, 384 threads = 3 warpgroups, tile 128 x 128):
//   warpgroup 0    : TMA producer (one elected thread: A 128x64, W 128x64, SWIZZLE_128B, 5-stage ring of 32 KB)
//   warpgroups 1-2 : consumers; consumer c owns the CTA's tiles 2i + c, all 128 rows: two wgmma m64n128k16 per k16 step,
//                    128 fp32 accumulators per thread.  An mbarrier pair hands the tensor core from one consumer's main
//                    loop to the other's, so while one consumer runs its epilogue the other issues MMAs.  The epilogue
//                    goes through one 64 KB staging tile: for residual forms the tile's fp32 residual is TMA-loaded into
//                    it during the owner's main loop; the consumer adds (acc + bias) + residual, writes the result back
//                    and one thread TMA-stores the tile, waits until the store has read the staging tile and hands it
//                    on to the other consumer's tile.  A tile that reaches past the row count (*m_dev, or a partial
//                    last tile) is stored from the registers instead.
//
// gemm_f16_kernel (one persistent CTA per SM, 384 threads = 3 warpgroups, tile 128 x BN, BN = 128 or 256):
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

// ---------------------------------------------------------------- ping-pong kernel (plain 2-D forms, fp32 output)
// Each consumer warpgroup owns whole 128 x 128 tiles (consumer c takes the CTA's tiles 2i + c), so one consumer's
// epilogue runs while the other issues MMAs.  The finished tile leaves through one 64 KB staging tile in shared memory
// by TMA stores; for residual forms the staging tile first receives the tile's fp32 residual by TMA.
namespace pp {
constexpr int BN = 128;
constexpr int STAGES = 5;
constexpr int STAGE_BYTES = (BM + BN) * BK * 2;         // A 128 x 64 + W 128 x 64, fp16
constexpr int BOX_BYTES = BM * 128;                       // one 128-row box of 128-byte rows (SWIZZLE_128B span)
constexpr int STAGING_BYTES = BM * BN * 4;               // 128 x 128 fp32: 4 boxes of 32 columns
constexpr int BAR_BYTES = 256;
constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + STAGING_BYTES + BAR_BYTES + 1024;
}  // namespace pp

__device__ __forceinline__ void pp_advance(int& stage, uint32_t& phase, int n) {
  stage += n;
  while (stage >= pp::STAGES) { stage -= pp::STAGES; phase ^= 1; }
}

// Hands the staging tile to the consumer of `tile`: loads the tile's residual into it (completing `bar` by its bytes), or,
// without a residual, arrives on `bar`.  Called by one thread once the staging tile's previous contents are no longer read.
__device__ __forceinline__ void pp_arm_staging(const GemmParams& p, const CUtensorMap* tmR, uint8_t* stg, uint64_t* bar,
                                               int tile, int num_n) {
  if (p.resid) {
    const int row0 = (tile / num_n) * BM, col0 = (tile % num_n) * pp::BN;
    mbar_arrive_expect_tx(bar, pp::STAGING_BYTES);
#pragma unroll
    for (int b = 0; b < 4; ++b) tma_load_2d(stg + b * pp::BOX_BYTES, tmR, bar, col0 + 32 * b, row0);
  } else {
    mbar_arrive(bar);
  }
}

// Epilogue of one consumer's 128 x 128 fp32 tile into the staging tile, in the order of gemm_epilogue_regs: (acc + bias)
// + residual, then ReLU.  acc[h] is the m64n128 accumulator of rows 64h .. 64h + 63 (layout in gemm_epilogue.cuh).  The
// staging tile holds the four 32-column boxes the TMA stores read, SWIZZLE_128B: the 16-byte chunk j of row r of a box
// sits at chunk j ^ (r % 8), so a warp's float2 accesses (8 rows x 32 B) hit every bank equally often.  For residual
// forms the staging tile already holds the residual in the same layout.
__device__ __forceinline__ void pp_epilogue_smem(const GemmParams& p, const float (&acc)[2][64], uint8_t* stg, int col0,
                                                 int warp_in_wg, int lane) {
  const int q = lane & 3;
#pragma unroll
  for (int i = 0; i < pp::BN / 8; ++i) {
    float2 b = make_float2(0.f, 0.f);
    if (p.bias) b = __ldg(reinterpret_cast<const float2*>(p.bias + col0 + 8 * i + 2 * q));
#pragma unroll
    for (int h = 0; h < 2; ++h) {
#pragma unroll
      for (int hr = 0; hr < 2; ++hr) {
        const int r = h * 64 + warp_in_wg * 16 + hr * 8 + (lane >> 2);
        float v0 = acc[h][4 * i + 2 * hr], v1 = acc[h][4 * i + 2 * hr + 1];
        if (p.bias) {
          v0 += b.x;
          v1 += b.y;
        }
        // box i / 4 of 32 columns, chunk 2 (i % 4) + q / 2
        float2* d = reinterpret_cast<float2*>(stg + (i >> 2) * pp::BOX_BYTES + r * 128 +
                                              (((2 * (i & 3) + (q >> 1)) ^ (r & 7)) << 4) + 8 * (q & 1));
        if (p.resid) {
          const float2 rr = *d;
          v0 += rr.x;
          v1 += rr.y;
        }
        if (p.relu) {
          v0 = fmaxf(v0, 0.f);
          v1 = fmaxf(v1, 0.f);
        }
        *d = make_float2(v0, v1);
      }
    }
  }
}

__global__ void __launch_bounds__(384, 1)
gemm_pp_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
               const __grid_constant__ CUtensorMap tmO, const __grid_constant__ CUtensorMap tmR, const GemmParams p_in) {
  const GemmParams p = gemm_resolve(p_in);
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* stg = smem + pp::STAGES * pp::STAGE_BYTES;
  uint64_t* full = reinterpret_cast<uint64_t*>(stg + pp::STAGING_BYTES);
  uint64_t* empty = full + pp::STAGES;
  uint64_t* turn = empty + pp::STAGES;   // turn[c]: the other consumer has issued its tile's MMAs; c may issue its own
  uint64_t* ready = turn + 2;            // ready[c]: the staging tile is free for c's tile (and holds its residual)

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = threadIdx.x >> 7;

  const int num_m = (p.M + BM - 1) / BM;
  const int num_n = p.N / pp::BN;
  const int num_tiles = num_m * num_n;
  const int num_k = p.K / BK;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    tma_prefetch_desc(&tmO);
    for (int i = 0; i < pp::STAGES; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], 128);     // the owning consumer's threads release the stage
    }
    for (int c = 0; c < 2; ++c) {
      mbar_init(&turn[c], 128);
      mbar_init(&ready[c], 1);
    }
    fence_barrier_init();
  }
  __syncthreads();
  if (threadIdx.x == 0 && (int)blockIdx.x < num_tiles) pp_arm_staging(p, &tmR, stg, &ready[0], blockIdx.x, num_n);

  if (wg == 0) {
    setmaxnreg_dec<40>();
    if (warp == 0 && elect_one()) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int m_blk = tile / num_n, n_blk = tile % num_n;
        const int nk = (n_blk * pp::BN < p.n_short) ? p.k_short / BK : num_k;
        for (int kb = 0; kb < nk; ++kb) {
          mbar_wait(&empty[stage], phase ^ 1);
          uint8_t* sA = smem + stage * pp::STAGE_BYTES;
          uint8_t* sB = sA + BM * BK * 2;
          mbar_arrive_expect_tx(&full[stage], pp::STAGE_BYTES);
          const int ka = p.a_kwrap ? (kb * BK) % p.a_kwrap : kb * BK;
          tma_load_2d(sA, &tmA, &full[stage], ka, m_blk * BM);
          tma_load_2d(sB, &tmB, &full[stage], kb * BK, n_blk * pp::BN);
          pp_advance(stage, phase, 1);
        }
      }
    }
  } else {
    setmaxnreg_inc<232>();
    const int c = wg - 1;
    float acc[2][64];
    int stage = 0;
    uint32_t phase = 0;
    int j = 0;                                // tiles this consumer has finished
    for (int t = 0, tile = blockIdx.x; tile < num_tiles; ++t, tile += gridDim.x) {
      const int m_blk = tile / num_n, n_blk = tile % num_n;
      const int nk = (n_blk * pp::BN < p.n_short) ? p.k_short / BK : num_k;
      if ((t & 1) != c) {                     // the other consumer's tile: skip its stages of the ring
        pp_advance(stage, phase, nk);
        continue;
      }
      if (t > 0) mbar_wait(&turn[c], ((t - 1) >> 1) & 1);
      int prev = -1;
      for (int kb = 0; kb < nk; ++kb) {
        mbar_wait(&full[stage], phase);
        const uint32_t a_addr = smem_u32(smem + stage * pp::STAGE_BYTES);
        const uint32_t b_addr = a_addr + BM * BK * 2;
        wgmma_fence_operand(acc[0]);
        wgmma_fence_operand(acc[1]);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k) {
          const uint64_t bd = make_sw128_desc(b_addr + k * 32);
          wgmma_m64n128k16_ss(acc[0], make_sw128_desc(a_addr + k * 32), bd, (kb | k) != 0 ? 1u : 0u);
          wgmma_m64n128k16_ss(acc[1], make_sw128_desc(a_addr + 64 * 128 + k * 32), bd, (kb | k) != 0 ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_fence_operand(acc[0]);
        wgmma_fence_operand(acc[1]);
        wgmma_wait<1>();                      // the previous k-block's MMAs are done: release its stage
        if (prev >= 0) mbar_arrive(&empty[prev]);
        prev = stage;
        pp_advance(stage, phase, 1);
      }
      mbar_arrive(&turn[c ^ 1]);              // every MMA of this tile is issued: the other consumer may queue its own
      wgmma_wait<0>();
      wgmma_fence_operand(acc[0]);
      wgmma_fence_operand(acc[1]);
      mbar_arrive(&empty[prev]);

      const int row0 = m_blk * BM, col0 = n_blk * pp::BN;
      mbar_wait(&ready[c], j & 1);
      const bool leader = (threadIdx.x & 127) == 0;
      if (row0 + BM <= p.M) {
        pp_epilogue_smem(p, acc, stg, col0, warp & 3, lane);
        fence_proxy_async_shared();
        named_bar_sync(1 + c, 128);
        if (leader) {
          for (int b = 0; b < 4; ++b) tma_store_2d(&tmO, stg + b * pp::BOX_BYTES, col0 + 32 * b, row0);
          bulk_commit();
          bulk_wait_read_all();
        }
      } else {
        // The tile reaches past the row count.  A TMA store writes whole boxes up to the tensor map's M rows, but rows
        // from *m_dev on must keep their contents, so this tile is stored from the registers, row by row.
        gemm_epilogue_regs<pp::BN>(p, acc[0], row0, col0, warp & 3, lane);
        gemm_epilogue_regs<pp::BN>(p, acc[1], row0 + 64, col0, warp & 3, lane);
      }
      if (leader && tile + (int)gridDim.x < num_tiles)
        pp_arm_staging(p, &tmR, stg, &ready[c ^ 1], tile + gridDim.x, num_n);
      ++j;
    }
  }
}

int launch_pp(cudaStream_t st, const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmO,
              const CUtensorMap& tmR, const GemmParams& p) {
  BG_TRY(ensure_dynamic_smem(reinterpret_cast<const void*>(&gemm_pp_kernel), pp::SMEM_BYTES));
  const int num_tiles = ((p.M + BM - 1) / BM) * (p.N / pp::BN);
  const int grid = num_tiles < num_sms() ? num_tiles : num_sms();
  gemm_pp_kernel<<<grid, 384, pp::SMEM_BYTES, st>>>(tmA, tmB, tmO, tmR, p);
  return check_launch("gemm_pp_kernel launch");
}

// BREPGEN_B200_GEMM_PINGPONG=0 sends every form to gemm_f16_kernel (for comparison); read once per process.
bool pingpong_enabled() {
  static const bool on = [] {
    const char* e = getenv("BREPGEN_B200_GEMM_PINGPONG");
    return !(e && atoi(e) == 0);
  }();
  return on;
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
  // Kernel selection: the plain 2-D forms with fp32 output (the in-place residual GEMMs out_proj and linear2, and
  // fc_out) run on gemm_pp_kernel with 128 x 128 tiles: their epilogue moves 8 B per element and measured to cost more
  // than the 128 x 128 tiles' slower main loop.  fp16 outputs (QKV, linear1) stay on gemm_f16_kernel's 128 x 256 tiles,
  // whose main loop is faster by more than their 2-byte epilogue costs (DESIGN.md §5), as do the implicit convolutions,
  // the row-vector form (token embedding) and residuals that TMA cannot address (not 16-byte aligned).
  const bool use_pp = pingpong_enabled() && !ep.out_f16 && ep.conv.taps == 0 && ep.rowvec == nullptr &&
                      ep.row_map == nullptr && (reinterpret_cast<uintptr_t>(ep.resid) & 15) == 0;
  if (use_pp) bn = pp::BN;
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
  if (use_pp) {
    CUtensorMap tmO, tmR;
    BG_TRY(make_tmap_2d_f32(&tmO, ep.out, (uint64_t)M, (uint64_t)N, (uint64_t)ep.ldo, BM, 32));
    tmR = tmO;
    if (ep.resid) BG_TRY(make_tmap_2d_f32(&tmR, ep.resid, (uint64_t)M, (uint64_t)N, (uint64_t)ep.ldr, BM, 32));
    return launch_pp(st, tmA, tmB, tmO, tmR, p);
  }
  return bn == 256 ? launch_bn<256>(st, tmA, tmB, p) : launch_bn<128>(st, tmA, tmB, p);
}

}  // namespace bg
