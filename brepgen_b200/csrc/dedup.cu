// Greedy first-seen de-duplication of face / edge bounding boxes between cascade stages, on the device.
//
// Reference (host numpy loops with a D2H/H2D round trip per stage):
//   surfaces  sample.py:159-183  np.round(bbox, 4); keep-list seeded with slot 0; slot i is a duplicate
//             iff for some kept k:  max|kept_k - bbox_i| < thr  OR  max|kept_k - reversed_corners(bbox_i)| < thr;
//             survivors packed to the front, zero padded, mask True = padded.
//   edges     sample.py:242-261  same test per VALID face over its E slots, no rounding, no packing: duplicates are
//             only flagged; padded faces are fully flagged; slot 0 of a valid face is always valid.
// One warp per sample (surfaces) / per face (edges); the scan over slots is inherently sequential, the comparison
// against the keep-list is spread over the lanes.  Integer/compare work, bit-exact with the numpy loops.
//
// B-rep variations also need to know where each survivor came from (bg_dedup_surfaces_index: the input slot of every
// kept face) and which source token every slot of a varied stage starts from (bg_fill_index: the trainers' pad_repeat
// layout, utils.py:100-106, of a row's valid slots).
#include "../../include/brepgen_b200.h"
#include "bg_internal.h"

namespace bg {
namespace {

constexpr int MAX_SLOTS = 256;

__device__ __forceinline__ float round4(float v) { return __fdiv_rn(rintf(__fmul_rn(v, 10000.f)), 10000.f); }

// returns true if bbox b (6 floats: corner0 xyz, corner1 xyz) matches any kept entry, directly or corner-swapped
__device__ __forceinline__ bool is_dup(const float (*kept)[6], int n_kept, const float* b, float thr, int lane) {
  bool dup = false;
  for (int k = lane; k < n_kept; k += 32) {
    float d = 0.f, dr = 0.f;
#pragma unroll
    for (int c = 0; c < 6; ++c) {
      d = fmaxf(d, fabsf(kept[k][c] - b[c]));
      dr = fmaxf(dr, fabsf(kept[k][c] - b[(c + 3) % 6]));
    }
    dup = dup || (d < thr) || (dr < thr);
  }
  return __any_sync(0xffffffffu, dup);
}

__global__ void __launch_bounds__(32) dedup_surfaces_kernel(const float* __restrict__ pos, int S, float thr,
                                                            float* __restrict__ out_pos, uint8_t* __restrict__ out_mask,
                                                            int* __restrict__ out_index) {
  __shared__ float kept[MAX_SLOTS][6];
  __shared__ int kept_slot[MAX_SLOTS];
  __shared__ float cur[6];
  const int b = blockIdx.x, lane = threadIdx.x;
  const float* p = pos + (size_t)b * S * 6;
  int n_kept = 0;
  for (int i = 0; i < S; ++i) {
    if (lane < 6) cur[lane] = round4(p[i * 6 + lane]);
    __syncwarp();
    // the keep-list starts as {slot 0}; slot 0 then matches itself and is not appended twice
    const bool dup = (i == 0) ? false : is_dup(kept, n_kept, cur, thr, lane);
    if (!dup) {
      if (lane < 6) kept[n_kept][lane] = cur[lane];
      if (lane == 0) kept_slot[n_kept] = i;
      ++n_kept;
    }
    __syncwarp();
  }
  float* o = out_pos + (size_t)b * S * 6;
  for (int i = lane; i < S * 6; i += 32) o[i] = (i / 6 < n_kept) ? kept[i / 6][i % 6] : 0.f;
  for (int i = lane; i < S; i += 32) out_mask[(size_t)b * S + i] = i >= n_kept;
  if (out_index)
    for (int i = lane; i < S; i += 32) out_index[(size_t)b * S + i] = i < n_kept ? kept_slot[i] : -1;
}

__global__ void __launch_bounds__(32) dedup_edges_kernel(const float* __restrict__ pos, const uint8_t* __restrict__ surf_mask,
                                                         int E, float thr, uint8_t* __restrict__ edge_mask) {
  __shared__ float kept[MAX_SLOTS][6];
  __shared__ float cur[6];
  const int f = blockIdx.x, lane = threadIdx.x;      // f = b * S + s
  uint8_t* m = edge_mask + (size_t)f * E;
  if (surf_mask[f]) {
    for (int i = lane; i < E; i += 32) m[i] = 1;
    return;
  }
  const float* p = pos + (size_t)f * E * 6;
  int n_kept = 0;
  for (int i = 0; i < E; ++i) {
    if (lane < 6) cur[lane] = p[i * 6 + lane];
    __syncwarp();
    const bool dup = (i == 0) ? false : is_dup(kept, n_kept, cur, thr, lane);
    if (!dup) {
      if (lane < 6) kept[n_kept][lane] = cur[lane];
      ++n_kept;
    }
    if (lane == 0) m[i] = dup ? 1 : 0;
    __syncwarp();
  }
}

// pad_repeat (utils.py:100-106) of the n valid slots of one source row onto out_slots output slots: with r = out / n and
// sep = out - r*n, each of the first sep valid slots is repeated r + 1 times in a row, each later one r times.  One warp
// per output row r: src_row = row_map[r] (or r), -1 = no source.  out[r][j] = src_row * in_slots + (valid slot taken by
// j); -1 for every slot of a row without a source or without a valid slot; -2 (out of range: the gather poisons it) for
// every slot of a row with more valid slots than out_slots, or whose source row is out of range.
__global__ void __launch_bounds__(32) fill_index_kernel(const uint8_t* __restrict__ src_mask, const int* __restrict__ row_map,
                                                        long long n_src_rows, int in_slots, int out_slots,
                                                        int* __restrict__ out) {
  __shared__ int valid[MAX_SLOTS];
  const long long r = blockIdx.x;
  const int lane = threadIdx.x;
  int* o = out + r * out_slots;
  const long long sr = row_map ? (long long)row_map[r] : r;
  int code = 0;                                      // 0: fill, -1: no source, -2: poisoned
  if (sr == -1) code = -1;
  else if (sr < 0 || sr >= n_src_rows) code = -2;
  int n = 0;
  if (code == 0) {
    const uint8_t* m = src_mask + sr * in_slots;
    for (int base = 0; base < in_slots; base += 32) {      // compact the valid slot numbers in slot order
      const int i = base + lane;
      const bool v = i < in_slots && m[i] == 0;
      const unsigned bal = __ballot_sync(0xffffffffu, v);
      if (v) valid[n + __popc(bal & ((1u << lane) - 1u))] = i;
      n += __popc(bal);
    }
    __syncwarp();
    if (n == 0) code = -1;
    else if (n > out_slots) code = -2;
  }
  if (code != 0) {
    for (int j = lane; j < out_slots; j += 32) o[j] = code;
    return;
  }
  const int rep = out_slots / n, sep = out_slots - rep * n, head = sep * (rep + 1);
  const int base = (int)(sr * in_slots);
  for (int j = lane; j < out_slots; j += 32) {
    const int k = j < head ? j / (rep + 1) : sep + (j - head) / rep;
    o[j] = base + valid[k];
  }
}

}  // namespace
}  // namespace bg

using namespace bg;

extern "C" {

int bg_dedup_surfaces(const float* surfPos, int B, int S, float threshold, float* out_pos, uint8_t* out_mask, void* stream) {
  BG_REQUIRE(surfPos && out_pos && out_mask && B > 0 && S > 0 && S <= MAX_SLOTS, "dedup_surfaces: bad arguments");
  BG_REQUIRE(surfPos != out_pos, "dedup_surfaces: in-place is not supported");
  dedup_surfaces_kernel<<<B, 32, 0, reinterpret_cast<cudaStream_t>(stream)>>>(surfPos, S, threshold, out_pos, out_mask,
                                                                              nullptr);
  return check_launch("dedup_surfaces_kernel launch");
}

int bg_dedup_surfaces_index(const float* surfPos, int B, int S, float threshold, float* out_pos, uint8_t* out_mask,
                            int32_t* out_index, void* stream) {
  BG_REQUIRE(surfPos && out_pos && out_mask && out_index && B > 0 && S > 0 && S <= MAX_SLOTS,
             "dedup_surfaces_index: bad arguments");
  BG_REQUIRE(surfPos != out_pos, "dedup_surfaces_index: in-place is not supported");
  dedup_surfaces_kernel<<<B, 32, 0, reinterpret_cast<cudaStream_t>(stream)>>>(surfPos, S, threshold, out_pos, out_mask,
                                                                              out_index);
  return check_launch("dedup_surfaces_kernel launch");
}

int bg_fill_index(const uint8_t* src_mask, const int32_t* row_map, int64_t rows, int64_t n_src_rows, int32_t in_slots,
                  int32_t out_slots, int32_t* out_index, void* stream) {
  BG_REQUIRE(src_mask && out_index && rows > 0 && n_src_rows > 0, "fill_index: bad arguments");
  BG_REQUIRE(in_slots > 0 && in_slots <= MAX_SLOTS && out_slots > 0, "fill_index: in_slots must be in [1, 256], out_slots > 0");
  BG_REQUIRE(row_map || rows <= n_src_rows, "fill_index: without a row map, rows must not exceed n_src_rows");
  BG_REQUIRE(n_src_rows * in_slots <= 0x7FFFFFFFll && rows <= 0x7FFFFFFFll,
             "fill_index: source token indices must fit in 32 bits");
  fill_index_kernel<<<(unsigned)rows, 32, 0, reinterpret_cast<cudaStream_t>(stream)>>>(src_mask, row_map, n_src_rows, in_slots,
                                                                                       out_slots, out_index);
  return check_launch("fill_index_kernel launch");
}

int bg_dedup_edges(const float* edgePos, const uint8_t* surf_mask, int B, int S, int E, float threshold,
                   uint8_t* edge_mask, void* stream) {
  BG_REQUIRE(edgePos && surf_mask && edge_mask && B > 0 && S > 0 && E > 0 && E <= MAX_SLOTS, "dedup_edges: bad arguments");
  dedup_edges_kernel<<<B * S, 32, 0, reinterpret_cast<cudaStream_t>(stream)>>>(edgePos, surf_mask, E, threshold, edge_mask);
  return check_launch("dedup_edges_kernel launch");
}

}  // extern "C"
