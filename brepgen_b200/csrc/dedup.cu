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
                                                            float* __restrict__ out_pos, uint8_t* __restrict__ out_mask) {
  __shared__ float kept[MAX_SLOTS][6];
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
      ++n_kept;
    }
    __syncwarp();
  }
  float* o = out_pos + (size_t)b * S * 6;
  for (int i = lane; i < S * 6; i += 32) o[i] = (i / 6 < n_kept) ? kept[i / 6][i % 6] : 0.f;
  for (int i = lane; i < S; i += 32) out_mask[(size_t)b * S + i] = i >= n_kept;
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

}  // namespace
}  // namespace bg

using namespace bg;

extern "C" {

int bg_dedup_surfaces(const float* surfPos, int B, int S, float threshold, float* out_pos, uint8_t* out_mask, void* stream) {
  BG_REQUIRE(surfPos && out_pos && out_mask && B > 0 && S > 0 && S <= MAX_SLOTS, "dedup_surfaces: bad arguments");
  BG_REQUIRE(surfPos != out_pos, "dedup_surfaces: in-place is not supported");
  dedup_surfaces_kernel<<<B, 32, 0, reinterpret_cast<cudaStream_t>(stream)>>>(surfPos, S, threshold, out_pos, out_mask);
  return check_launch("dedup_surfaces_kernel launch");
}

int bg_dedup_edges(const float* edgePos, const uint8_t* surf_mask, int B, int S, int E, float threshold,
                   uint8_t* edge_mask, void* stream) {
  BG_REQUIRE(edgePos && surf_mask && edge_mask && B > 0 && S > 0 && E > 0 && E <= MAX_SLOTS, "dedup_edges: bad arguments");
  dedup_edges_kernel<<<B * S, 32, 0, reinterpret_cast<cudaStream_t>(stream)>>>(edgePos, surf_mask, E, threshold, edge_mask);
  return check_launch("dedup_edges_kernel launch");
}

}  // extern "C"
