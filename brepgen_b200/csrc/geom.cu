// Post-decode geometry glue on the device (SURVEY.md 8(f) row 3): the O(n^2) numeric cores of the reference's per-CAD
// post-processing between the VAE decoders and OpenCASCADE (construct_brep, out of scope):
//   edge end points            sample.py:316-329   (+ utils.py:48-59 compute_bbox_center_and_size)
//   nearest "other" end point  utils.py:403-421 edge2loop, and the across-face centre search utils.py:505-524
//   close-centre matrix        utils.py:556-561
//   same-endpoints / z match   utils.py:607-619 detect_shared_edge
//   edge fit to the vertices   utils.py:692-728 joint_optimize (scale, flip, offset, end-point snapping)
//   surface initialisation     utils.py:732-752
//   surface offset fit         utils.py:756-770: 200 AdamW steps on a per-face translation minimising the one-directional
//                              Chamfer distance wire -> surface; the reference makes one chamferdist call per face and
//                              iteration (25 600 faces x 200 at B = 256), here ONE launch runs all iterations of all faces.
// All of it is small, latency-bound fp32 work: one thread per point / one CTA per face, no tensor cores.  The combinatorial
// bookkeeping around these cores (loops of python lists and sets) stays on the host (brepgen_b200/postprocess.py).
// fp32 arithmetic follows numpy's operation order with explicit _rn intrinsics (no FMA contraction) where the reference
// compares or sorts the values.
#include <math.h>

#include "../../include/brepgen_b200.h"
#include "bg_internal.h"

namespace bg {
namespace {

__device__ __forceinline__ float dist3(const float* a, const float* b) {   // np.linalg.norm(a - b) in fp32, numpy's order
  const float d0 = __fsub_rn(a[0], b[0]), d1 = __fsub_rn(a[1], b[1]), d2 = __fsub_rn(a[2], b[2]);
  return __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(d0, d0), __fmul_rn(d1, d1)), __fmul_rn(d2, d2)));
}

// ---------------------------------------------------------------- sample.py:316-329
// out[e][k][:] = ncs[e][k ? 31 : 0][:] * (bsize / 2) + bcenter,  bcenter = (min + max) / 2, bsize = max extent of the edge box
__global__ void edge_endpoints_kernel(const float* __restrict__ ncs, const float* __restrict__ pos, float pos_scale, long long n,
                                      float* __restrict__ out) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  float b[6];
#pragma unroll
  for (int i = 0; i < 6; ++i) b[i] = __fmul_rn(pos[e * 6 + i], pos_scale);
  float c[3], sz = -INFINITY;
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    c[i] = __fdiv_rn(__fadd_rn(b[i], b[3 + i]), 2.f);
    sz = fmaxf(sz, __fsub_rn(b[3 + i], b[i]));
  }
  const float h = __fdiv_rn(sz, 2.f);
#pragma unroll
  for (int k = 0; k < 2; ++k)
#pragma unroll
    for (int i = 0; i < 3; ++i) out[(e * 2 + k) * 3 + i] = __fadd_rn(__fmul_rn(ncs[(e * 32 + (k ? 31 : 0)) * 3 + i], h), c[i]);
}

// ---------------------------------------------------------------- nearest point of ANOTHER group inside the same segment
// nn[i] = argmin_j { |p_j - p_i| : seg(j) == seg(i), group[j] != group[i] }, lowest j on ties, -1 if there is none
__global__ void nn_exclude_kernel(const float* __restrict__ pts, const int* __restrict__ group, const int* __restrict__ seg_off,
                                  int nseg, int* __restrict__ nn) {
  const int s = blockIdx.x;
  if (s >= nseg) return;
  const int lo = seg_off[s], hi = seg_off[s + 1];
  for (int i = lo + threadIdx.x; i < hi; i += blockDim.x) {
    float best = INFINITY;
    int arg = -1;
    const int g = group[i];
    for (int j = lo; j < hi; ++j) {
      if (group[j] == g) continue;
      const float d = dist3(pts + 3 * (size_t)j, pts + 3 * (size_t)i);
      if (d < best) { best = d; arg = j; }
    }
    nn[i] = arg;
  }
}

// out[i][j] = |p_i - p_j| < thr   (n x n, row-major)
__global__ void pairs_within_kernel(const float* __restrict__ pts, int n, float thr, uint8_t* __restrict__ out) {
  const long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= (long long)n * n) return;
  const int i = (int)(k / n), j = (int)(k % n);
  out[k] = dist3(pts + 3 * (size_t)i, pts + 3 * (size_t)j) < thr ? 1 : 0;
}

// ---------------------------------------------------------------- utils.py:607-619
// out[i][j] = i != j && {adj[i]} == {adj[j]} && mean |z_i - z_j| < thr
__global__ void edge_pair_match_kernel(const int* __restrict__ adj, const float* __restrict__ z, int zdim, int n, float thr,
                                       uint8_t* __restrict__ out) {
  const long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= (long long)n * n) return;
  const int i = (int)(k / n), j = (int)(k % n);
  uint8_t r = 0;
  if (i != j) {
    const int a0 = adj[2 * i], a1 = adj[2 * i + 1], b0 = adj[2 * j], b1 = adj[2 * j + 1];
    // set(s1) == set(s2) for two-element lists (a degenerate edge {a, a} equals {a, a} only)
    const bool same = (a0 == b0 || a0 == b1) && (a1 == b0 || a1 == b1) && (b0 == a0 || b0 == a1) && (b1 == a0 || b1 == a1);
    if (same) {
      float acc = 0.f;                      // np.abs(z1 - z2).mean(): pairwise summation differs only below fp32 round-off
      for (int q = 0; q < zdim; ++q) acc += fabsf(z[(size_t)i * zdim + q] - z[(size_t)j * zdim + q]);
      r = (acc / (float)zdim) < thr ? 1 : 0;
    }
  }
  out[k] = r;
}

// ---------------------------------------------------------------- utils.py:692-728
// per edge: scale the decoded curve so that its end points are as far apart as the two target vertices, pick the orientation
// whose start / end offsets agree better, translate by the mean offset, then snap both ends onto the vertices and spread the
// correction linearly along the 32 samples
__global__ void edge_fit_kernel(const float* __restrict__ ncs, const float* __restrict__ vse, int n, float* __restrict__ wcs) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  const float* c = ncs + (size_t)e * 96;
  const float* v = vse + (size_t)e * 6;
  const float scale = dist3(v, v + 3) / dist3(c, c + 93);
  float s0[3], s1[3], off[2][3], offr[2][3];
  for (int i = 0; i < 3; ++i) {
    s0[i] = c[i] * scale;
    s1[i] = c[93 + i] * scale;
    off[0][i] = v[i] - s0[i];
    off[1][i] = v[3 + i] - s1[i];
    offr[0][i] = v[i] - s1[i];
    offr[1][i] = v[3 + i] - s0[i];
  }
  float err = 0.f, errr = 0.f;
  for (int i = 0; i < 3; ++i) {
    err += fabsf(off[0][i] - off[1][i]);
    errr += fabsf(offr[0][i] - offr[1][i]);
  }
  const bool flip = (errr / 3.f) < (err / 3.f);
  float t[3];
  for (int i = 0; i < 3; ++i) t[i] = flip ? (offr[0][i] + offr[1][i]) / 2.f : (off[0][i] + off[1][i]) / 2.f;
  // first / last sample after scale, flip and translation -> residual vectors to the vertices
  float sv[3], ev[3];
  for (int i = 0; i < 3; ++i) {
    const float first = (flip ? c[93 + i] : c[i]) * scale + t[i];
    const float last = (flip ? c[i] : c[93 + i]) * scale + t[i];
    sv[i] = v[i] - first;
    ev[i] = v[3 + i] - last;
  }
  for (int k = 0; k < 32; ++k) {
    const int src = flip ? 31 - k : k;
    const double w = (double)k / 31.0;
    for (int i = 0; i < 3; ++i) {
      const float p = c[src * 3 + i] * scale + t[i];
      wcs[((size_t)e * 32 + k) * 3 + i] = p + (float)((double)sv[i] * (1.0 - w) + (double)ev[i] * w);
    }
  }
}

// ---------------------------------------------------------------- utils.py:732-752
// per face: bounding box of its wire (all samples of its edges), surface centre / scale from the face box (scale = 1.05 x wire
// scale when the face box is smaller than the wire), surface grid ncs -> wcs
__global__ void surf_init_kernel(const float* __restrict__ surf_ncs, const float* __restrict__ surf_pos,
                                 const float* __restrict__ edge_wcs, const int* __restrict__ adj_off, const int* __restrict__ adj,
                                 int nface, float* __restrict__ surf_wcs) {
  const int f = blockIdx.x;
  if (f >= nface) return;
  __shared__ float red[6][128];
  float mn[3] = {INFINITY, INFINITY, INFINITY}, mx[3] = {-INFINITY, -INFINITY, -INFINITY};
  const int lo = adj_off[f], hi = adj_off[f + 1];
  for (int k = threadIdx.x; k < (hi - lo) * 32; k += blockDim.x) {
    const float* p = edge_wcs + ((size_t)adj[lo + k / 32] * 32 + k % 32) * 3;
    for (int i = 0; i < 3; ++i) {
      mn[i] = fminf(mn[i], p[i]);
      mx[i] = fmaxf(mx[i], p[i]);
    }
  }
  for (int i = 0; i < 3; ++i) {
    red[i][threadIdx.x] = mn[i];
    red[3 + i][threadIdx.x] = mx[i];
  }
  __syncthreads();
  for (int s = blockDim.x / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s)
      for (int i = 0; i < 3; ++i) {
        red[i][threadIdx.x] = fminf(red[i][threadIdx.x], red[i][threadIdx.x + s]);
        red[3 + i][threadIdx.x] = fmaxf(red[3 + i][threadIdx.x], red[3 + i][threadIdx.x + s]);
      }
    __syncthreads();
  }
  const float* b = surf_pos + (size_t)f * 6;
  float c[3], sscale = -INFINITY, escale = -INFINITY;
  for (int i = 0; i < 3; ++i) {
    c[i] = (b[i] + b[3 + i]) / 2.f;
    sscale = fmaxf(sscale, b[3 + i] - b[i]);
    escale = fmaxf(escale, red[3 + i][0] - red[i][0]);
  }
  if (sscale < escale) sscale = 1.05f * escale;
  const float h = sscale / 2.f;
  for (int k = threadIdx.x; k < 1024 * 3; k += blockDim.x)
    surf_wcs[(size_t)f * 3072 + k] = surf_ncs[(size_t)f * 3072 + k] * h + c[k % 3];
}

// ---------------------------------------------------------------- utils.py:756-770
// One CTA per face, ALL iterations in one launch.  Parameter = the face translation o (3 floats; the reference's scale
// parameter surf_st[:, 0] never enters the loss).  Loss of the CAD = mean over its faces of
//   sum_{e in wire samples} min_{s in surface samples} |s + o - e|^2       (chamferdist: bidirectional=False, reverse=True,
//                                                                           point_reduction "sum")
// so dL/do = (2 / nface_cad) * sum_e (s*(e) + o - e).  torch.optim.AdamW(lr, betas, eps, weight_decay) update in fp32.
// Output = surface + the offset BEFORE the last step (the reference returns surf_updated of the last iteration, computed
// before that iteration's optimizer.step()).
constexpr int SOPT_THREADS = 256;
__global__ void __launch_bounds__(SOPT_THREADS) surf_offset_opt_kernel(
    const float* __restrict__ surf_init, const float* __restrict__ edge_wcs, const int* __restrict__ adj_off,
    const int* __restrict__ adj, const float* __restrict__ inv_nface, int nface, int iters, float lr, float beta1, float beta2,
    float eps, float wd, float* __restrict__ surf_out, float* __restrict__ offset_out) {
  const int f = blockIdx.x;
  if (f >= nface) return;
  extern __shared__ float sm[];
  float* sp = sm;                    // 1024 x 3 surface samples
  float* ep = sm + 3072;             // wire samples (ne x 32 x 3)
  __shared__ float red[3][SOPT_THREADS / 32];
  __shared__ float o_s[3];
  const int lo = adj_off[f], hi = adj_off[f + 1];
  const int npt = (hi - lo) * 32;
  for (int k = threadIdx.x; k < 3072; k += blockDim.x) sp[k] = surf_init[(size_t)f * 3072 + k];
  for (int k = threadIdx.x; k < npt * 3; k += blockDim.x) ep[k] = edge_wcs[((size_t)adj[lo + k / 96]) * 96 + k % 96];
  if (threadIdx.x < 3) o_s[threadIdx.x] = 0.f;
  __syncthreads();
  const float gscale = 2.f * inv_nface[f];
  float m[3] = {0.f, 0.f, 0.f}, v[3] = {0.f, 0.f, 0.f}, o[3] = {0.f, 0.f, 0.f}, o_prev[3] = {0.f, 0.f, 0.f};
  float b1t = 1.f, b2t = 1.f;
  for (int it = 0; it < iters; ++it) {
    float g[3] = {0.f, 0.f, 0.f};
    for (int k = threadIdx.x; k < npt; k += blockDim.x) {
      const float ex = ep[3 * k] - o[0], ey = ep[3 * k + 1] - o[1], ez = ep[3 * k + 2] - o[2];   // e - o
      float best = INFINITY;
      int arg = 0;
      for (int s = 0; s < 1024; ++s) {
        const float dx = sp[3 * s] - ex, dy = sp[3 * s + 1] - ey, dz = sp[3 * s + 2] - ez;
        const float d = dx * dx + dy * dy + dz * dz;
        if (d < best) { best = d; arg = s; }
      }
      g[0] += sp[3 * arg] - ex;
      g[1] += sp[3 * arg + 1] - ey;
      g[2] += sp[3 * arg + 2] - ez;
    }
    for (int i = 0; i < 3; ++i) {
      float x = g[i];
      for (int s = 16; s > 0; s >>= 1) x += __shfl_xor_sync(0xffffffffu, x, s);
      if ((threadIdx.x & 31) == 0) red[i][threadIdx.x >> 5] = x;
    }
    __syncthreads();
    b1t *= beta1;
    b2t *= beta2;
    for (int i = 0; i < 3; ++i) {
      float gi = 0.f;
      for (int w = 0; w < SOPT_THREADS / 32; ++w) gi += red[i][w];
      gi *= gscale;
      o_prev[i] = o[i];
      o[i] *= 1.f - lr * wd;                                   // decoupled weight decay
      m[i] = beta1 * m[i] + (1.f - beta1) * gi;
      v[i] = beta2 * v[i] + (1.f - beta2) * gi * gi;
      const float denom = sqrtf(v[i]) / sqrtf(1.f - b2t) + eps;
      o[i] -= (lr / (1.f - b1t)) * (m[i] / denom);
    }
    __syncthreads();
  }
  for (int k = threadIdx.x; k < 3072; k += blockDim.x) surf_out[(size_t)f * 3072 + k] = sp[k] + o_prev[k % 3];
  if (offset_out && threadIdx.x < 3) offset_out[(size_t)f * 3 + threadIdx.x] = o_prev[threadIdx.x];
}

}  // namespace
}  // namespace bg

using namespace bg;

extern "C" {

int bg_edge_endpoints(const float* edge_ncs, const float* edge_pos, float pos_scale, int64_t n_edges, float* out, void* stream) {
  BG_REQUIRE(edge_ncs && edge_pos && out && n_edges > 0, "edge_endpoints: bad arguments");
  edge_endpoints_kernel<<<(unsigned)((n_edges + 127) / 128), 128, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      edge_ncs, edge_pos, pos_scale, n_edges, out);
  return check_launch("edge_endpoints_kernel launch");
}

int bg_nn_exclude(const float* pts, const int32_t* group, const int32_t* seg_off, int n_seg, int32_t* nn, void* stream) {
  BG_REQUIRE(pts && group && seg_off && nn && n_seg > 0, "nn_exclude: bad arguments");
  nn_exclude_kernel<<<n_seg, 128, 0, reinterpret_cast<cudaStream_t>(stream)>>>(pts, group, seg_off, n_seg, nn);
  return check_launch("nn_exclude_kernel launch");
}

int bg_pairs_within(const float* pts, int n, float threshold, uint8_t* out, void* stream) {
  BG_REQUIRE(pts && out && n > 0 && n <= 46340, "pairs_within: bad arguments");
  pairs_within_kernel<<<(unsigned)(((long long)n * n + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(pts, n,
                                                                                                                       threshold, out);
  return check_launch("pairs_within_kernel launch");
}

int bg_edge_pair_match(const int32_t* edge_vertex_adj, const float* z, int z_dim, int n, float threshold, uint8_t* out,
                       void* stream) {
  BG_REQUIRE(edge_vertex_adj && z && out && n > 0 && n <= 46340 && z_dim > 0, "edge_pair_match: bad arguments");
  edge_pair_match_kernel<<<(unsigned)(((long long)n * n + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      edge_vertex_adj, z, z_dim, n, threshold, out);
  return check_launch("edge_pair_match_kernel launch");
}

int bg_edge_fit(const float* edge_ncs, const float* vertex_se, int n_edges, float* edge_wcs, void* stream) {
  BG_REQUIRE(edge_ncs && vertex_se && edge_wcs && n_edges > 0, "edge_fit: bad arguments");
  edge_fit_kernel<<<(n_edges + 63) / 64, 64, 0, reinterpret_cast<cudaStream_t>(stream)>>>(edge_ncs, vertex_se, n_edges, edge_wcs);
  return check_launch("edge_fit_kernel launch");
}

int bg_surf_init(const float* surf_ncs, const float* surf_pos, const float* edge_wcs, const int32_t* adj_off, const int32_t* adj,
                 int n_faces, float* surf_wcs, void* stream) {
  BG_REQUIRE(surf_ncs && surf_pos && edge_wcs && adj_off && adj && surf_wcs && n_faces > 0, "surf_init: bad arguments");
  surf_init_kernel<<<n_faces, 128, 0, reinterpret_cast<cudaStream_t>(stream)>>>(surf_ncs, surf_pos, edge_wcs, adj_off, adj, n_faces,
                                                                                surf_wcs);
  return check_launch("surf_init_kernel launch");
}

int bg_surf_offset_opt(const float* surf_init, const float* edge_wcs, const int32_t* adj_off, const int32_t* adj,
                       const float* inv_nface, int n_faces, int max_edges_per_face, int iters, float lr, float beta1, float beta2,
                       float eps, float weight_decay, float* surf_out, float* offset_out, void* stream) {
  BG_REQUIRE(surf_init && edge_wcs && adj_off && adj && inv_nface && surf_out && n_faces > 0 && iters > 0,
             "surf_offset_opt: bad arguments");
  BG_REQUIRE(max_edges_per_face > 0 && max_edges_per_face <= 512, "surf_offset_opt: at most 512 edges per face");
  const int smem = (3072 + max_edges_per_face * 96) * (int)sizeof(float);
  BG_TRY(ensure_dynamic_smem(reinterpret_cast<const void*>(&surf_offset_opt_kernel), smem));
  surf_offset_opt_kernel<<<n_faces, SOPT_THREADS, smem, reinterpret_cast<cudaStream_t>(stream)>>>(
      surf_init, edge_wcs, adj_off, adj, inv_nface, n_faces, iters, lr, beta1, beta2, eps, weight_decay, surf_out, offset_out);
  return check_launch("surf_offset_opt_kernel launch");
}

}  // extern "C"
