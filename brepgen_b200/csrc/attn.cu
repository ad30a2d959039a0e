// wgmma flash attention for the denoisers' self-attention (12 heads x 64, key-padding mask).
//
// Reference semantics: nn.MultiheadAttention inside nn.TransformerEncoderLayer with src_key_padding_mask
// (network.py:1119-1123, 1193-1197, 1279-1283, 1387-1390): softmax(q k^T / 8 + (-inf on padded keys)) v.
// Edge stages run ONE sequence of L = faces*edges <= 4000 tokens per sample (network.py:1265-1283), so this is an
// online-softmax (flash) kernel; the surface stages (L <= 100) use the same kernel with one key block.
//
// CTA = one 128-row query tile of one (sample, head), 384 threads = 3 warpgroups:
//   warpgroup 0    : TMA producer (one elected thread: Q once; K / V 128-key tiles through an ST-deep mbarrier ring);
//                    gives its registers to the consumers (setmaxnreg)
//   warpgroups 1-2 : consumers, 64 query rows each; per key block j:
//                      S = Q K_j^T          4 x wgmma m64n128k16, Q and K K-major SW128 from shared memory
//                      P = exp2(c (S - m))  in registers (fp32 online softmax, rows split over lane quads)
//                      O = O a + P V_j      8 x wgmma m64n64k16, A = P as fp16 straight from the S registers,
//                                           B = V MN-major SW128 from shared memory
//                    S, P and O never leave the registers; the two consumer warpgroups interleave on the tensor core.
// Fully padded key blocks are skipped through a per-sample block list (result-preserving: their p is exactly 0).
// Roofline: tensor-bound; 4*L*L*64 flop per (sample, head).
#include <math.h>

#include "bg_internal.h"
#include "ptx.cuh"


namespace bg {

namespace {

constexpr int DH = 64;
constexpr int NHEAD = 12;
constexpr int DMODEL = 768;
constexpr int BQ = 128;                    // query rows per CTA (two consumer warpgroups of 64)
constexpr int TILE_BYTES = 128 * DH * 2;   // 16 KB: Q / K / V tile, 128 rows x 128 B
constexpr int ST = 2;                      // K / V ring depth
constexpr int OFF_Q = 0;
constexpr int OFF_K = TILE_BYTES;
constexpr int OFF_V = OFF_K + ST * TILE_BYTES;
constexpr int OFF_BAR = OFF_V + ST * TILE_BYTES;
constexpr int OFF_MASKW = OFF_BAR + 256;   // invalid-key bit words: 4 per key block, MAX_KB blocks
constexpr int MAX_KB = 64;                 // L <= 8192
constexpr int SMEM_BYTES = OFF_MASKW + MAX_KB * 16 + 1024;
constexpr int THREADS = 384;
constexpr int CONSUMER_THREADS = 256;

struct AttnParams {
  __half* out;
  int ldo;
  int B, L, nkb;
  const uint8_t* key_mask;
  const int* blk_list;
  const int* blk_count;
  const uint32_t* blk_words;   // [B][nkb][4] invalid-key bit words of the listed blocks, list order (per forward), or null
  const int* seq_row0;         // variable-length mode: first row / number of rows of every sample, or null (dense)
  const int* seq_len;
  float scale_log2;            // log2(e) / sqrt(64)
};

__device__ __forceinline__ float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

__global__ void __launch_bounds__(THREADS, 1)
attn_kernel(const __grid_constant__ CUtensorMap tmQKV, const AttnParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + OFF_BAR);
  uint64_t* q_full = bars;
  uint64_t* k_full = q_full + 1;
  uint64_t* k_empty = k_full + ST;
  uint64_t* v_full = k_empty + ST;
  uint64_t* v_empty = v_full + ST;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = threadIdx.x >> 7;
  const int qgrp = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  // QKV / out are addressed as ONE [rows][cols] matrix; sample b owns rows [row0, row0 + len).  Dense: row0 = b * L, len = L.
  // Variable-length mode (mask-aware token compaction): rows of the valid tokens only, packed back to back.  A tile may then
  // run into the next sample's rows (or past the end: TMA zero-fills): those keys are masked (key >= len), those query rows
  // are never written.
  const int row0 = p.seq_row0 ? p.seq_row0[b] : b * p.L;
  const int len = p.seq_len ? p.seq_len[b] : p.L;
  if (qgrp * BQ >= len) return;     // variable-length mode: the grid is sized for the longest sample
  const int nblk = p.blk_count ? p.blk_count[b] : (len + 127) / 128;
  const int* blist = p.blk_list ? p.blk_list + (size_t)b * p.nkb : nullptr;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmQKV);
    mbar_init(q_full, 1);
    for (int i = 0; i < ST; ++i) {
      mbar_init(&k_full[i], 1);
      mbar_init(&k_empty[i], CONSUMER_THREADS);
      mbar_init(&v_full[i], 1);
      mbar_init(&v_empty[i], CONSUMER_THREADS);
    }
    fence_barrier_init();
  }
  // invalid-key bit words for every key block this CTA will visit (padded key or key >= len), built once: keeps the
  // global mask bytes off the per-block critical path
  uint32_t* maskw = reinterpret_cast<uint32_t*>(smem + OFF_MASKW);
  if (p.blk_words || !p.key_mask) {
    // one word per thread, no dependent global-load chain: either copied from the per-forward table or, without a
    // mask, computed (only keys >= len are invalid)
    for (int wi = threadIdx.x; wi < nblk * 4; wi += THREADS) {
      uint32_t w;
      if (p.blk_words) {      // list order: entry wi >> 2 belongs to key block blist[wi >> 2]
        w = p.blk_words[((size_t)b * p.nkb + (wi >> 2)) * 4 + (wi & 3)];
      } else {
        const int base = (wi >> 2) * 128 + (wi & 3) * 32;
        w = base + 32 <= len ? 0u : (base >= len ? 0xffffffffu : (0xffffffffu << (len - base)));
      }
      maskw[wi] = w;
    }
  } else {
    for (int wi = warp; wi < nblk * 4; wi += THREADS / 32) {
      const int kb = blist ? blist[wi >> 2] : (wi >> 2);
      const int key = kb * 128 + (wi & 3) * 32 + lane;
      bool bad = key >= len;
      if (!bad) bad = p.key_mask[(size_t)b * p.L + key] != 0;
      const uint32_t w = __ballot_sync(0xffffffffu, bad);
      if (lane == 0) maskw[wi] = w;
    }
  }
  __syncthreads();

  if (wg == 0) {
    setmaxnreg_dec<24>();
    if (warp == 0 && elect_one()) {
      mbar_arrive_expect_tx(q_full, TILE_BYTES);
      tma_load_2d(smem + OFF_Q, &tmQKV, q_full, h * DH, row0 + qgrp * BQ);
      for (int it = 0; it < nblk; ++it) {
        const int kb = blist ? blist[it] : it;
        const int s = it % ST;
        const uint32_t par = ((it / ST) & 1) ^ 1;
        mbar_wait(&k_empty[s], par);
        mbar_arrive_expect_tx(&k_full[s], TILE_BYTES);
        tma_load_2d(smem + OFF_K + s * TILE_BYTES, &tmQKV, &k_full[s], DMODEL + h * DH, row0 + kb * 128);
        mbar_wait(&v_empty[s], par);
        mbar_arrive_expect_tx(&v_full[s], TILE_BYTES);
        tma_load_2d(smem + OFF_V + s * TILE_BYTES, &tmQKV, &v_full[s], 2 * DMODEL + h * DH, row0 + kb * 128);
      }
    }
    return;
  }

  setmaxnreg_inc<240>();
  // ------------------------------------------------------------------ consumer warpgroup: 64 query rows
  // Accumulator layout (wgmma m64nN, fp32): warp w of the warpgroup owns rows 16w + lane / 4 (elements 4i, 4i + 1) and
  // 16w + 8 + lane / 4 (elements 4i + 2, 4i + 3), at columns 8i + 2 (lane % 4) + {0, 1}.  Every row is spread over one
  // lane quad, so row statistics need two shuffles.
  const int half = wg - 1;
  const int wq = warp & 3;
  const float c = p.scale_log2;
  const uint32_t q_addr = smem_u32(smem + OFF_Q) + half * 64 * 128;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  float o[DH / 2];
#pragma unroll
  for (int i = 0; i < DH / 2; ++i) o[i] = 0.f;

  mbar_wait(q_full, 0);
  for (int it = 0; it < nblk; ++it) {
    const int s = it % ST;
    const uint32_t par = (it / ST) & 1;
    float sc[64];
    mbar_wait(&k_full[s], par);
    const uint32_t k_addr = smem_u32(smem + OFF_K + s * TILE_BYTES);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < DH / 16; ++k)
      wgmma_m64n128k16_ss(sc, make_sw128_desc(q_addr + k * 32), make_sw128_desc(k_addr + k * 32), k > 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_operand(sc);
    mbar_arrive(&k_empty[s]);

    const uint4 iw = *reinterpret_cast<const uint4*>(maskw + it * 4);
    if ((iw.x | iw.y | iw.z | iw.w) != 0) {
      const uint32_t inval[4] = {iw.x, iw.y, iw.z, iw.w};
#pragma unroll
      for (int i = 0; i < 16; ++i)
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const int key = 8 * i + 2 * (lane & 3) + j;
          if ((inval[key >> 5] >> (key & 31)) & 1u) {
            sc[4 * i + j] = -INFINITY;
            sc[4 * i + 2 + j] = -INFINITY;
          }
        }
    }
    float ref[2], alpha[2];
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      float mx = -INFINITY;
#pragma unroll
      for (int i = 0; i < 16; ++i) mx = fmaxf(mx, fmaxf(sc[4 * i + 2 * hr], sc[4 * i + 2 * hr + 1]));
      const float m_new = fmaxf(m_run[hr], quad_max(mx));
      ref[hr] = m_new == -INFINITY ? 0.f : m_new;        // a row without any valid key so far keeps p = 0
      alpha[hr] = ex2((m_run[hr] - ref[hr]) * c);         // 0 while the row had no valid key (m_run = -inf)
      m_run[hr] = m_new;
      l_run[hr] *= alpha[hr];
    }
#pragma unroll
    for (int i = 0; i < DH / 8; ++i) {
      o[4 * i] *= alpha[0];
      o[4 * i + 1] *= alpha[0];
      o[4 * i + 2] *= alpha[1];
      o[4 * i + 3] *= alpha[1];
    }
    // p = exp2(c s - c m), row sums in fp32, and the fp16 A fragments of P V: the A fragment of key slice kk (16 keys)
    // is {rows r, r + 8} x {keys 16kk + 2 (lane % 4) + {0, 1}, + 8}, i.e. exactly accumulator columns 2kk and 2kk + 1
    uint32_t pa[8][4];
    const float nm0 = -ref[0] * c, nm1 = -ref[1] * c;
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const float p0 = ex2(fmaf(sc[4 * i], c, nm0)), p1 = ex2(fmaf(sc[4 * i + 1], c, nm0));
      const float p2 = ex2(fmaf(sc[4 * i + 2], c, nm1)), p3 = ex2(fmaf(sc[4 * i + 3], c, nm1));
      l_run[0] += p0 + p1;
      l_run[1] += p2 + p3;
      pa[i >> 1][(i & 1) * 2] = pack_half2(p0, p1);
      pa[i >> 1][(i & 1) * 2 + 1] = pack_half2(p2, p3);
    }

    mbar_wait(&v_full[s], par);
    const uint32_t v_addr = smem_u32(smem + OFF_V + s * TILE_BYTES);
    wgmma_fence_operand(o);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) wgmma_m64n64k16_rs_bt(o, pa[kk], make_sw128_desc(v_addr + kk * 2048), 1u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_operand(o);
    mbar_arrive(&v_empty[s]);
  }

#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    const float l = quad_sum(l_run[hr]);
    const float inv = l > 0.f ? 1.f / l : 0.f;
    const int row = qgrp * BQ + half * 64 + wq * 16 + hr * 8 + (lane >> 2);
    if (row >= len) continue;
    __half* dst = p.out + ((size_t)row0 + row) * p.ldo + h * DH + 2 * (lane & 3);
#pragma unroll
    for (int i = 0; i < DH / 8; ++i)
      *reinterpret_cast<uint32_t*>(dst + 8 * i) = pack_half2(o[4 * i + 2 * hr] * inv, o[4 * i + 2 * hr + 1] * inv);
  }
}

// one CTA per sample: which 128-key blocks hold at least one valid key (blk_list / blk_count), and the invalid-key bit
// words of the LISTED blocks in list order (blk_words[b][i][4] belongs to key block blk_list[b][i]), so that the
// attention kernels index them with their loop counter and need no dependent load
__global__ void block_list_kernel(const uint8_t* __restrict__ key_mask, int L, int nkb, int* __restrict__ blk_list,
                                  int* __restrict__ blk_count, uint32_t* __restrict__ blk_words) {
  extern __shared__ int sm_bl[];
  int* pos = sm_bl;                                           // list position of key block kb, or -1
  uint32_t* wds = reinterpret_cast<uint32_t*>(sm_bl + nkb);   // [nkb][4]
  const int b = blockIdx.x;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarp = blockDim.x >> 5;
  for (int kb = warp; kb < nkb; kb += nwarp) {
    bool any = false;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const int key = kb * 128 + c * 32 + lane;
      const bool bad = key >= L || key_mask[(size_t)b * L + key] != 0;
      const uint32_t w = __ballot_sync(0xffffffffu, bad);
      any = any || w != 0xffffffffu;
      if (lane == 0) wds[kb * 4 + c] = w;
    }
    if (lane == 0) pos[kb] = any ? 0 : -1;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int n = 0;
    for (int kb = 0; kb < nkb; ++kb)
      if (pos[kb] == 0) {
        blk_list[(size_t)b * nkb + n] = kb;
        pos[kb] = n++;
      }
    blk_count[b] = n;
  }
  __syncthreads();
  if (blk_words)
    for (int i = threadIdx.x; i < nkb * 4; i += blockDim.x)
      if (pos[i >> 2] >= 0) blk_words[((size_t)b * nkb + pos[i >> 2]) * 4 + (i & 3)] = wds[i];
}

}  // namespace

int launch_attention(cudaStream_t st, const AttnArgs& a) {
  BG_REQUIRE(a.qkv && a.out && a.B > 0 && a.L > 0, "attention: bad arguments");
  BG_REQUIRE(a.ldo % 8 == 0, "attention: output pitch must be a multiple of 8");
  BG_REQUIRE(a.L <= 128 * MAX_KB, "attention: sequence longer than 8192 tokens is not supported");
  BG_REQUIRE((a.blk_list == nullptr) == (a.blk_count == nullptr), "attention: blk_list and blk_count go together");
  CUtensorMap tm;
  BG_REQUIRE((a.seq_row0 == nullptr) == (a.seq_len == nullptr), "attention: seq_row0 and seq_len go together");
  BG_REQUIRE(a.seq_len == nullptr || (a.key_mask == nullptr && a.blk_list == nullptr), "attention: variable-length mode takes no mask");
  BG_TRY(make_tmap_2d_f16(&tm, a.qkv, (uint64_t)a.B * (uint64_t)a.L, 3 * DMODEL, 3 * DMODEL, 128));
  AttnParams p;
  p.out = a.out; p.ldo = a.ldo; p.B = a.B; p.L = a.L; p.nkb = (a.L + 127) / 128;
  p.key_mask = a.key_mask; p.blk_list = a.blk_list; p.blk_count = a.blk_count; p.blk_words = a.blk_words;
  p.seq_row0 = a.seq_row0; p.seq_len = a.seq_len;
  p.scale_log2 = 1.4426950408889634f / 8.0f;
  BG_TRY(ensure_dynamic_smem(reinterpret_cast<const void*>(&attn_kernel), SMEM_BYTES));
  dim3 grid((a.L + BQ - 1) / BQ, NHEAD, a.B);
  attn_kernel<<<grid, THREADS, SMEM_BYTES, st>>>(tm, p);
  return check_launch("attn_kernel launch");
}

int launch_build_block_list(cudaStream_t st, const uint8_t* key_mask, int B, int L, int* blk_list, int* blk_count,
                            uint32_t* blk_words) {
  BG_REQUIRE(key_mask && blk_list && blk_count && B > 0 && L > 0, "block list: bad arguments");
  const int nkb = (L + 127) / 128;
  block_list_kernel<<<B, 128, nkb * 5 * sizeof(int), st>>>(key_mask, L, nkb, blk_list, blk_count, blk_words);
  return check_launch("block_list_kernel launch");
}

}  // namespace bg
