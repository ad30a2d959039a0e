// Fused scheduler updates (HBM-bound elementwise): classifier-free-guidance combine + DDPM posterior step with
// in-kernel Philox noise, and the PNDM transfer step with its Adams-Bashforth / Runge-Kutta combination of the eps
// history.  Replaces ~15 scalar-broadcast torch launches per diffusers step (SURVEY.md Appendix A.3/A.4;
// call sites sample.py:132-137,148-153,195-202,...).
// Algorithmic bytes per element: DDPM 4 (eps) [+4 uncond] + 4 (x) + 4 (out) [+4 explicit noise]; PNDM 4*(2 + #history).
#include <math.h>

#include "../../include/brepgen_b200.h"
#include "bg_internal.h"

namespace bg {
namespace {

// Philox4x32-10 (Salmon et al. 2011): counter = (offset + element_group, 0), key = seed.
__device__ __forceinline__ void philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0, uint32_t k1,
                                              uint32_t (&out)[4]) {
#pragma unroll
  for (int i = 0; i < 10; ++i) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
    const uint32_t n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
  out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}
__device__ __forceinline__ void box_muller(uint32_t a, uint32_t b, float& z0, float& z1) {
  const float u1 = ((float)a + 1.0f) * 2.3283064365386963e-10f;   // (0, 1]
  const float u2 = (float)b * 2.3283064365386963e-10f;            // [0, 1)
  const float rr = sqrtf(-2.0f * __logf(u1));
  float s, c;
  __sincosf(6.283185307179586f * u2, &s, &c);
  z0 = rr * c;
  z1 = rr * s;
}

struct DdpmP {
  const float *eps_c, *eps_u, *x, *noise;
  float* out;
  long long n;
  float w, sb, sa, clip, c_x0, c_x, sigma;
  unsigned long long seed, offset;
};

__global__ void __launch_bounds__(256) ddpm_step_kernel(const DdpmP p) {
  const long long n4 = (p.n + 3) / 4;
  for (long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x; g < n4; g += (long long)gridDim.x * blockDim.x) {
    float z[4] = {0.f, 0.f, 0.f, 0.f};
    if (p.sigma != 0.f && p.noise == nullptr) {
      uint32_t r[4];
      const unsigned long long ctr = p.offset + (unsigned long long)g;
      philox4x32_10((uint32_t)ctr, (uint32_t)(ctr >> 32), 0u, 0u, (uint32_t)p.seed, (uint32_t)(p.seed >> 32), r);
      box_muller(r[0], r[1], z[0], z[1]);
      box_muller(r[2], r[3], z[2], z[3]);
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const long long i = g * 4 + j;
      if (i >= p.n) break;
      float e = p.eps_c[i];
      if (p.eps_u) e = e * (1.f + p.w) - p.eps_u[i] * p.w;
      const float xv = p.x[i];
      float x0 = (xv - p.sb * e) / p.sa;
      if (p.clip > 0.f) x0 = fminf(fmaxf(x0, -p.clip), p.clip);
      float o = p.c_x0 * x0 + p.c_x * xv;
      if (p.sigma != 0.f) o += p.sigma * (p.noise ? p.noise[i] : z[j]);
      p.out[i] = o;
    }
  }
}

// Table-driven form for CUDA-graph replay: nothing step-specific is a kernel argument.  The coefficients of step k live in
// coef[k][0..4] = (sqrt(1-abar_t), sqrt(abar_t), c_x0, c_x, sigma), k = *step is a device counter that bg_step_advance moves
// on once per step, and the Philox counter starts at offset0 + k * offset_stride.
struct DdpmTabP {
  const float *eps_c, *eps_u, *x;
  float* out;
  long long n;
  float w, clip;
  const float* coef;
  const int* step;
  unsigned long long seed, offset0, offset_stride;
};
__global__ void __launch_bounds__(256) ddpm_step_tab_kernel(const DdpmTabP p) {
  const int k = *p.step;
  const float* cf = p.coef + 5 * (long long)k;
  const float sb = cf[0], sa = cf[1], c_x0 = cf[2], c_x = cf[3], sigma = cf[4];
  const unsigned long long offset = p.offset0 + (unsigned long long)k * p.offset_stride;
  const long long n4 = (p.n + 3) / 4;
  for (long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x; g < n4; g += (long long)gridDim.x * blockDim.x) {
    float z[4] = {0.f, 0.f, 0.f, 0.f};
    if (sigma != 0.f) {
      uint32_t r[4];
      const unsigned long long ctr = offset + (unsigned long long)g;
      philox4x32_10((uint32_t)ctr, (uint32_t)(ctr >> 32), 0u, 0u, (uint32_t)p.seed, (uint32_t)(p.seed >> 32), r);
      box_muller(r[0], r[1], z[0], z[1]);
      box_muller(r[2], r[3], z[2], z[3]);
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const long long i = g * 4 + j;
      if (i >= p.n) break;
      float e = p.eps_c[i];
      if (p.eps_u) e = e * (1.f + p.w) - p.eps_u[i] * p.w;
      const float xv = p.x[i];
      float x0 = (xv - sb * e) / sa;
      if (p.clip > 0.f) x0 = fminf(fmaxf(x0, -p.clip), p.clip);
      float o = c_x0 * x0 + c_x * xv;
      if (sigma != 0.f) o += sigma * z[j];
      p.out[i] = o;
    }
  }
}
// one thread: k = ++(*step);  *t_cur = ts[k]   (the denoiser reads its timestep from t_cur, the step kernel reads k)
__global__ void step_advance_kernel(const long long* __restrict__ ts, int n, int* __restrict__ step, long long* __restrict__ t_cur) {
  int k = *step + 1;
  if (k >= n) k = n - 1;
  *step = k;
  *t_cur = ts[k];
}

struct PndmP {
  const float* x;
  float* out;
  long long n;
  float cs, ce;
  const float* e[4];
  float w[4];
};
__global__ void __launch_bounds__(256) pndm_step_kernel(const PndmP p) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < p.n; i += (long long)gridDim.x * blockDim.x) {
    float acc = 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j)
      if (p.e[j]) acc += p.w[j] * p.e[j][i];
    p.out[i] = p.cs * p.x[i] - p.ce * acc;
  }
}
__global__ void __launch_bounds__(256) axpby_kernel(const float* x, float a, const float* y, float b, float* out, long long n) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    out[i] = a * x[i] + (y ? b * y[i] : 0.f);
}

inline unsigned grid_for(long long work) {
  long long blocks = (work + 255) / 256;
  const long long cap = (long long)num_sms() * 16;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  return (unsigned)blocks;
}

}  // namespace
}  // namespace bg

using namespace bg;

extern "C" {

int bg_ddpm_step(const float* eps_cond, const float* eps_uncond, float cfg_w, const float* x, float* out,
                 const float* noise, uint64_t seed, uint64_t offset, int64_t n, float sqrt_one_minus_abar,
                 float sqrt_abar, float clip, float c_x0, float c_x, float sigma, void* stream) {
  BG_REQUIRE(eps_cond && x && out && n > 0, "ddpm_step: bad arguments");
  BG_REQUIRE(sqrt_abar > 0.f, "ddpm_step: sqrt_abar must be positive");
  DdpmP p;
  p.eps_c = eps_cond; p.eps_u = eps_uncond; p.x = x; p.noise = noise; p.out = out; p.n = n;
  p.w = cfg_w; p.sb = sqrt_one_minus_abar; p.sa = sqrt_abar; p.clip = clip; p.c_x0 = c_x0; p.c_x = c_x; p.sigma = sigma;
  p.seed = seed; p.offset = offset;
  ddpm_step_kernel<<<grid_for((n + 3) / 4), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(p);
  return check_launch("ddpm_step_kernel launch");
}

int bg_ddpm_step_tab(const float* eps_cond, const float* eps_uncond, float cfg_w, const float* x, float* out, uint64_t seed,
                     uint64_t offset0, uint64_t offset_stride, int64_t n, const float* coef_table, const int32_t* step,
                     float clip, void* stream) {
  BG_REQUIRE(eps_cond && x && out && n > 0 && coef_table && step, "ddpm_step_tab: bad arguments");
  DdpmTabP p;
  p.eps_c = eps_cond; p.eps_u = eps_uncond; p.x = x; p.out = out; p.n = n; p.w = cfg_w; p.clip = clip;
  p.coef = coef_table; p.step = step; p.seed = seed; p.offset0 = offset0; p.offset_stride = offset_stride;
  ddpm_step_tab_kernel<<<grid_for((n + 3) / 4), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(p);
  return check_launch("ddpm_step_tab_kernel launch");
}

int bg_step_advance(const int64_t* timesteps, int n_steps, int32_t* step, int64_t* t_cur, void* stream) {
  BG_REQUIRE(timesteps && n_steps > 0 && step && t_cur, "step_advance: bad arguments");
  step_advance_kernel<<<1, 1, 0, reinterpret_cast<cudaStream_t>(stream)>>>(reinterpret_cast<const long long*>(timesteps), n_steps,
                                                                           step, reinterpret_cast<long long*>(t_cur));
  return check_launch("step_advance_kernel launch");
}

int bg_pndm_step(const float* x, float* out, int64_t n, float c_sample, float c_eps, const float* e0, float w0,
                 const float* e1, float w1, const float* e2, float w2, const float* e3, float w3, void* stream) {
  BG_REQUIRE(x && out && n > 0, "pndm_step: bad arguments");
  PndmP p;
  p.x = x; p.out = out; p.n = n; p.cs = c_sample; p.ce = c_eps;
  p.e[0] = e0; p.e[1] = e1; p.e[2] = e2; p.e[3] = e3;
  p.w[0] = w0; p.w[1] = w1; p.w[2] = w2; p.w[3] = w3;
  pndm_step_kernel<<<grid_for(n), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(p);
  return check_launch("pndm_step_kernel launch");
}

int bg_axpby(const float* x, float a, const float* y, float b, float* out, int64_t n, void* stream) {
  BG_REQUIRE(x && out && n > 0, "axpby: bad arguments");
  axpby_kernel<<<grid_for(n), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(x, a, y, b, out, n);
  return check_launch("axpby_kernel launch");
}

}  // extern "C"
