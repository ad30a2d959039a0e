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

// Per-sample noise streams: element j of sample b is normal (j % 4) of Philox4x32-10 with key keys[b] and counter
// (j / 4 as 64 bits, t, domain); domain 0 = DDPM step noise at timestep t, 1 = initial noise (t = 0).  A group of 4 never
// straddles two samples (the last group of a sample uses its first per_sample % 4 normals), so a sample's noise does not
// depend on the batch it sits in, on its position there, or on the rank that runs it.
__device__ __forceinline__ void keyed_normal4(unsigned long long key, unsigned long long q, uint32_t t, uint32_t domain,
                                              float (&z)[4]) {
  uint32_t r[4];
  philox4x32_10((uint32_t)q, (uint32_t)(q >> 32), t, domain, (uint32_t)key, (uint32_t)(key >> 32), r);
  box_muller(r[0], r[1], z[0], z[1]);
  box_muller(r[2], r[3], z[2], z[3]);
}

struct RandnKeyedP {
  const unsigned long long* keys;
  float* out;
  long long n_samples, per_sample;
  uint32_t domain, t;
};
__global__ void __launch_bounds__(256) randn_keyed_kernel(const RandnKeyedP p) {
  const long long gps = (p.per_sample + 3) / 4, ng = p.n_samples * gps;
  for (long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x; g < ng; g += (long long)gridDim.x * blockDim.x) {
    const long long b = g / gps, q = g - b * gps;
    float z[4];
    keyed_normal4(p.keys[b], (unsigned long long)q, p.t, p.domain, z);
    float* o = p.out + b * p.per_sample;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const long long i = q * 4 + j;
      if (i >= p.per_sample) break;
      o[i] = z[j];
    }
  }
}

// Start of a varied stage (SDEdit: diffusers' img2img add_noise on a gathered source): for every element i of output
// token g = i / per_token,  out[i] = sa*(scale*src[index[g] * per_token + i % per_token]) + sb*z[i],  every product and
// the sum rounded on its own (the fp32 torch expression).  index[g] == -1: out[i] = z[i] (a slot without a source starts
// from pure noise); any other index outside [0, n_src): NaN.  z: explicit `noise`, else the per-sample keys (keyed_normal4
// at counter (e / 4, t, domain), e = i % per_sample: bg_randn_keyed's normals).  One thread per group of 4 elements of a
// sample, as the keyed kernels; without keys the whole tensor is one sample.
struct GatherP {
  const float *src, *noise;
  const int* index;
  float* out;
  long long n, per_sample, per_token, n_src;
  float scale, sa, sb;
  const unsigned long long* keys;
  uint32_t t, domain;
};
__global__ void __launch_bounds__(256) add_noise_gather_kernel(const GatherP p) {
  const long long gps = (p.per_sample + 3) / 4, ng = (p.n / p.per_sample) * gps;
  for (long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x; g < ng; g += (long long)gridDim.x * blockDim.x) {
    const long long b = g / gps, q = g - b * gps;
    const long long i0 = b * p.per_sample + q * 4;
    const int cnt = (int)min(4ll, p.per_sample - q * 4);
    float z[4] = {0.f, 0.f, 0.f, 0.f};
    if (p.noise) {
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (j < cnt) z[j] = p.noise[i0 + j];
    } else {
      keyed_normal4(p.keys[b], (unsigned long long)q, p.t, p.domain, z);
    }
    long long tok = i0 / p.per_token, r = i0 - tok * p.per_token;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (j < cnt) {
        const long long s = p.index[tok];
        float o;
        if (s == -1) o = z[j];
        else if (s < 0 || s >= p.n_src) o = __int_as_float(0x7fc00000);
        else o = __fadd_rn(__fmul_rn(p.sa, __fmul_rn(p.scale, p.src[s * p.per_token + r])), __fmul_rn(p.sb, z[j]));
        p.out[i0 + j] = o;
        if (++r == p.per_token) { ++tok; r = 0; }
      }
    }
  }
}

// The four normals the DDPM, DDIM and DPM-Solver++ steps add to group q of sample b: the per-sample stream of keys[b] at
// timestep t (domain 0) when keys != NULL, else the batch stream (seed, offset + q): the same Philox block under key seed
// at counter (offset + q, 0, 0).  Without keys the whole tensor is one sample (per_sample = n), so q is the batch stream's
// element group.
__device__ __forceinline__ void step_normal4(const unsigned long long* keys, long long b, long long q, long long t,
                                             unsigned long long seed, unsigned long long offset, float (&z)[4]) {
  if (keys) keyed_normal4(keys[b], (unsigned long long)q, (uint32_t)t, 0u, z);
  else keyed_normal4(seed, offset + (unsigned long long)q, 0u, 0u, z);
}

// DDPM step (diffusers 0.27 DDPMScheduler.step, epsilon prediction, fixed_small variance), per element:
//   e = e*(1+w) - eu*w;  x0 = (x - sb*e) / sa, clamped to +-clip;  out = c_x0*x0 + c_x*x [+ sigma*z].
// Every rounding is spelled out (one FMA each for e, x - sb*e, c_x*x + c_x0*x0 and + sigma*z), so that no compiler
// contraction can move a bit of a sample.  Noise (only when sigma != 0): explicit `noise`, else step_normal4.  Table
// form (coef != NULL): coefficients (sb, sa, c_x0, c_x, sigma) from coef[*step], t from *t_cur and the batch-stream
// offset offset + k * offset_stride.
struct DdpmP {
  const float *eps_c, *eps_u, *x, *noise;
  float* out;
  long long n, per_sample;
  float w, sb, sa, c_x0, c_x, sigma, clip;
  const unsigned long long* keys;
  long long t;
  unsigned long long seed, offset, offset_stride;
  const float* coef;
  const int* step;
  const long long* t_cur;
};
__global__ void __launch_bounds__(256) ddpm_step_kernel(const DdpmP p) {
  float sb = p.sb, sa = p.sa, c_x0 = p.c_x0, c_x = p.c_x, sigma = p.sigma;
  long long t = p.t;
  unsigned long long offset = p.offset;
  if (p.coef) {
    const int k = *p.step;
    const float* cf = p.coef + 5 * (long long)k;
    sb = cf[0]; sa = cf[1]; c_x0 = cf[2]; c_x = cf[3]; sigma = cf[4];
    if (p.t_cur) t = *p.t_cur;
    offset += (unsigned long long)k * p.offset_stride;
  }
  const long long gps = (p.per_sample + 3) / 4, ng = (p.n / p.per_sample) * gps;
  for (long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x; g < ng; g += (long long)gridDim.x * blockDim.x) {
    const long long b = p.keys ? g / gps : 0, q = g - b * gps;   // without keys: one sample, no division
    float z[4] = {0.f, 0.f, 0.f, 0.f};
    if (sigma != 0.f && p.noise == nullptr) step_normal4(p.keys, b, q, t, p.seed, offset, z);
    const long long base = b * p.per_sample;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const long long js = q * 4 + j;
      if (js >= p.per_sample) break;
      const long long i = base + js;
      float e = p.eps_c[i];
      if (p.eps_u) e = __fmaf_rn(e, 1.f + p.w, -__fmul_rn(p.eps_u[i], p.w));
      const float xv = p.x[i];
      float x0 = __fdiv_rn(__fmaf_rn(-sb, e, xv), sa);
      if (p.clip > 0.f) x0 = fminf(fmaxf(x0, -p.clip), p.clip);
      float o = __fmaf_rn(c_x, xv, __fmul_rn(c_x0, x0));
      if (sigma != 0.f) o = __fmaf_rn(sigma, p.noise ? p.noise[i] : z[j], o);
      p.out[i] = o;
    }
  }
}

// DDIM step (diffusers 0.27 DDIMScheduler.step, epsilon prediction), diffusers' order of operations in fp32:
//   x0 = (x - sb*e) / sa, clamped to +-clip;  e_dir = e, or (x - sa*x0) / sb with use_clipped_eps;
//   out = sa_prev*x0 + c_dir*e_dir [+ sigma*z].
// Noise (only when sigma != 0): explicit `noise`, else step_normal4, the normals the DDPM step draws at the same t.  Table
// form (coef != NULL): coefficients (sb, sa, sa_prev, c_dir, sigma) from coef[*step], t from *t_cur and the batch-stream
// offset offset + k * offset_stride.
struct DdimP {
  const float *eps_c, *eps_u, *x, *noise;
  float* out;
  long long n, per_sample;
  float w, sb, sa, sa_prev, c_dir, sigma, clip;
  int use_clipped_eps;
  const unsigned long long* keys;
  long long t;
  unsigned long long seed, offset, offset_stride;
  const float* coef;
  const int* step;
  const long long* t_cur;
};
__global__ void __launch_bounds__(256) ddim_step_kernel(const DdimP p) {
  float sb = p.sb, sa = p.sa, sa_prev = p.sa_prev, c_dir = p.c_dir, sigma = p.sigma;
  long long t = p.t;
  unsigned long long offset = p.offset;
  if (p.coef) {
    const int k = *p.step;
    const float* cf = p.coef + 5 * (long long)k;
    sb = cf[0]; sa = cf[1]; sa_prev = cf[2]; c_dir = cf[3]; sigma = cf[4];
    if (p.t_cur) t = *p.t_cur;
    offset += (unsigned long long)k * p.offset_stride;
  }
  const long long gps = (p.per_sample + 3) / 4, ng = (p.n / p.per_sample) * gps;
  for (long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x; g < ng; g += (long long)gridDim.x * blockDim.x) {
    const long long b = g / gps, q = g - b * gps;
    float z[4] = {0.f, 0.f, 0.f, 0.f};
    if (sigma != 0.f && p.noise == nullptr) step_normal4(p.keys, b, q, t, p.seed, offset, z);
    const long long base = b * p.per_sample;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const long long js = q * 4 + j;
      if (js >= p.per_sample) break;
      const long long i = base + js;
      float e = p.eps_c[i];
      if (p.eps_u) e = e * (1.f + p.w) - p.eps_u[i] * p.w;
      const float xv = p.x[i];
      float x0 = (xv - sb * e) / sa;
      if (p.clip > 0.f) x0 = fminf(fmaxf(x0, -p.clip), p.clip);
      if (p.use_clipped_eps) e = (xv - sa * x0) / sb;
      float o = sa_prev * x0 + c_dir * e;
      if (sigma != 0.f) o += sigma * (p.noise ? p.noise[i] : z[j]);
      p.out[i] = o;
    }
  }
}

// DPM-Solver++ multistep step (diffusers 0.27 DPMSolverMultistepScheduler, epsilon prediction, midpoint), first or second
// order, ODE ("dpmsolver++", c_z = 0) or SDE ("sde-dpmsolver++"):
//   x0 = (x - sigma_s*e) / alpha_s, clamped to +-clip;  m1 = hist[i];  hist[i] = x0;  D1 = (x0 - m1) * inv_r0;
//   out = c_x*x + c_0*x0 + c_1*D1 + c_z*z.
// Every product and sum is rounded on its own, in diffusers' order (D1 first, then the sum left to right), so the step
// tracks the fp32 torch oracle rather than an FMA-contracted variant of it.  c_1 == 0 (a first-order step) never reads
// hist; hist == NULL skips the store.  hist[i] is read and written by the thread that owns element i, so the update is
// in place.  Noise (only when c_z != 0) and the table form (coefficients from coef[7 * *step], t from *t_cur, batch offset
// offset + k * offset_stride) as ddim_step_kernel.
struct DpmP {
  const float *eps_c, *eps_u, *x, *noise;
  float *out, *hist;
  long long n, per_sample;
  float w, alpha_s, sigma_s, c_x, c_0, c_1, inv_r0, c_z, clip;
  const unsigned long long* keys;
  long long t;
  unsigned long long seed, offset, offset_stride;
  const float* coef;
  const int* step;
  const long long* t_cur;
};
__global__ void __launch_bounds__(256) dpm_step_kernel(const DpmP p) {
  float alpha_s = p.alpha_s, sigma_s = p.sigma_s, c_x = p.c_x, c_0 = p.c_0, c_1 = p.c_1, inv_r0 = p.inv_r0, c_z = p.c_z;
  long long t = p.t;
  unsigned long long offset = p.offset;
  if (p.coef) {
    const int k = *p.step;
    const float* cf = p.coef + 7 * (long long)k;
    alpha_s = cf[0]; sigma_s = cf[1]; c_x = cf[2]; c_0 = cf[3]; c_1 = cf[4]; inv_r0 = cf[5]; c_z = cf[6];
    if (p.t_cur) t = *p.t_cur;
    offset += (unsigned long long)k * p.offset_stride;
  }
  const long long gps = (p.per_sample + 3) / 4, ng = (p.n / p.per_sample) * gps;
  for (long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x; g < ng; g += (long long)gridDim.x * blockDim.x) {
    const long long b = g / gps, q = g - b * gps;
    float z[4] = {0.f, 0.f, 0.f, 0.f};
    if (c_z != 0.f && p.noise == nullptr) step_normal4(p.keys, b, q, t, p.seed, offset, z);
    // the group's loads first, then the math and the stores: no load waits behind a store it might alias
    const long long i0 = b * p.per_sample + q * 4;
    const int cnt = (int)min(4ll, p.per_sample - q * 4);
    float e[4], xv[4], m1[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (j < cnt) {
        e[j] = p.eps_c[i0 + j];
        if (p.eps_u) e[j] = __fsub_rn(__fmul_rn(e[j], 1.f + p.w), __fmul_rn(p.eps_u[i0 + j], p.w));
        xv[j] = p.x[i0 + j];
        if (c_1 != 0.f) m1[j] = p.hist[i0 + j];
        if (c_z != 0.f && p.noise) z[j] = p.noise[i0 + j];
      }
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (j < cnt) {
        float x0 = __fdiv_rn(__fsub_rn(xv[j], __fmul_rn(sigma_s, e[j])), alpha_s);
        if (p.clip > 0.f) x0 = fminf(fmaxf(x0, -p.clip), p.clip);
        float o = __fadd_rn(__fmul_rn(c_x, xv[j]), __fmul_rn(c_0, x0));
        if (c_1 != 0.f) o = __fadd_rn(o, __fmul_rn(c_1, __fmul_rn(__fsub_rn(x0, m1[j]), inv_r0)));
        if (c_z != 0.f) o = __fadd_rn(o, __fmul_rn(c_z, z[j]));
        if (p.hist) p.hist[i0 + j] = x0;
        p.out[i0 + j] = o;
      }
    }
  }
}

// UniPC multistep step (diffusers UniPCMultistepScheduler, predict_x0, epsilon prediction, "bh1" / "bh2"), one row of
// BG_UNIPC_ROW coefficients (layout in include/brepgen_b200.h):
//   x0 = (x - sigma_s*e) / alpha_s, clamped to +-clip;  m_i = hist[slot_i] = x0 of i steps back;
//   corrector (UniC, corr order c > 0):  xc = cc_x*last - cc_m0*m1 - cc_B*(sum_{i<c} rc_i*(m_{i+1} - m1)/rc_r_i
//                                                                        + rc_t*(x0 - m1));  else xc = x;
//   last = xc;  hist[slot_new] = x0;
//   predictor (UniP, order p):  out = cp_x*xc - cp_m0*x0 - cp_B*sum_{i<p} rp_i*(m_i - x0)/rp_r_i.
// Every product, quotient and sum is rounded on its own, in diffusers' order (the differences first, the sums left to
// right), so the step tracks the fp32 torch oracle.  The ring hist (n_slots slots of n elements) and last are read and
// written in place by the thread that owns the element, all of a group's loads before any store; out may alias x.  The
// row comes by value (eager form) or from coef[BG_UNIPC_ROW * *step] (table form).  No noise: UniPC is deterministic.
struct UnipcP {
  const float *eps_c, *eps_u, *x;
  float *out, *last, *hist;
  long long n, per_sample;
  float w, clip;
  float row[BG_UNIPC_ROW];
  const float* coef;
  const int* step;
};
__global__ void __launch_bounds__(256) unipc_step_kernel(const UnipcP p) {
  const float* r = p.row;
  if (p.coef) r = p.coef + (long long)BG_UNIPC_ROW * *p.step;
  const float alpha_s = r[0], sigma_s = r[1];
  const int corr = (int)r[2], pord = (int)r[3];
  const long long s_new = (long long)r[4] * p.n;
  const long long s1 = (long long)r[5] * p.n, s2 = (long long)r[6] * p.n, s3 = (long long)r[7] * p.n;
  const float cc_x = r[8], cc_m0 = r[9], cc_b = r[10], cr1 = r[11], cr2 = r[12], crho1 = r[13], crho2 = r[14];
  const float crho_t = r[15];
  const float cp_x = r[16], cp_m0 = r[17], cp_b = r[18], pr1 = r[19], pr2 = r[20], prho1 = r[21], prho2 = r[22];
  const int nread = max(corr, pord - 1);     // history slots this step reads: x0 of 1..nread steps back
  const long long gps = (p.per_sample + 3) / 4, ng = (p.n / p.per_sample) * gps;
  for (long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x; g < ng; g += (long long)gridDim.x * blockDim.x) {
    const long long b = g / gps, q = g - b * gps;
    const long long i0 = b * p.per_sample + q * 4;
    const int cnt = (int)min(4ll, p.per_sample - q * 4);
    float e[4], xv[4], lv[4] = {0.f, 0.f, 0.f, 0.f}, m1[4] = {0.f, 0.f, 0.f, 0.f}, m2[4] = {0.f, 0.f, 0.f, 0.f},
        m3[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (j < cnt) {
        const long long i = i0 + j;
        e[j] = p.eps_c[i];
        if (p.eps_u) e[j] = __fsub_rn(__fmul_rn(e[j], 1.f + p.w), __fmul_rn(p.eps_u[i], p.w));
        xv[j] = p.x[i];
        if (corr > 0) lv[j] = p.last[i];
        if (nread >= 1) m1[j] = p.hist[s1 + i];
        if (nread >= 2) m2[j] = p.hist[s2 + i];
        if (nread >= 3) m3[j] = p.hist[s3 + i];
      }
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (j < cnt) {
        const long long i = i0 + j;
        float x0 = __fdiv_rn(__fsub_rn(xv[j], __fmul_rn(sigma_s, e[j])), alpha_s);
        if (p.clip > 0.f) x0 = fminf(fmaxf(x0, -p.clip), p.clip);
        float xc = xv[j];
        if (corr > 0) {
          float res = 0.f;
          if (corr >= 2) res = __fmul_rn(crho1, __fdiv_rn(__fsub_rn(m2[j], m1[j]), cr1));
          if (corr >= 3) res = __fadd_rn(res, __fmul_rn(crho2, __fdiv_rn(__fsub_rn(m3[j], m1[j]), cr2)));
          const float tail = __fmul_rn(crho_t, __fsub_rn(x0, m1[j]));
          res = corr >= 2 ? __fadd_rn(res, tail) : tail;
          xc = __fsub_rn(__fsub_rn(__fmul_rn(cc_x, lv[j]), __fmul_rn(cc_m0, m1[j])), __fmul_rn(cc_b, res));
        }
        float o = __fsub_rn(__fmul_rn(cp_x, xc), __fmul_rn(cp_m0, x0));
        if (pord >= 2) {
          float res = __fmul_rn(prho1, __fdiv_rn(__fsub_rn(m1[j], x0), pr1));
          if (pord >= 3) res = __fadd_rn(res, __fmul_rn(prho2, __fdiv_rn(__fsub_rn(m2[j], x0), pr2)));
          o = __fsub_rn(o, __fmul_rn(cp_b, res));
        }
        if (p.last) p.last[i] = xc;
        p.hist[s_new + i] = x0;
        p.out[i] = o;
      }
    }
  }
}

// known[j] = whether the token of element i0 + j (token = element / per_token) has its mask byte set, for j < cnt; returns
// whether any is.  One division per group of 4: at most 4 mask bytes, usually 1 or 2 distinct.
__device__ __forceinline__ bool known_flags(const unsigned char* mask, long long i0, long long per_token, int cnt,
                                            bool (&known)[4]) {
  long long tok = i0 / per_token, r = i0 - tok * per_token;
  bool any = false;
#pragma unroll
  for (int j = 0; j < 4; ++j)
    if (j < cnt) {
      known[j] = mask[tok] != 0;
      any |= known[j];
      if (++r == per_token) { ++tok; r = 0; }
    }
  return any;
}

// Known-token replacement (B-rep completion): x[i] = sa*known[i] + sb*z for every element of a token whose mask byte is
// set; every other element is neither read nor written.  z: explicit `noise`, else per-sample keys (keyed_normal4, domain
// 2, counter word t_ctr), else the batch key `seed` over the whole tensor as one sample (per_sample = n).  Groups of 4
// never straddle two samples, as in the keyed steps.  Table form (coef != NULL): (sa, sb) from coef[*step], t_ctr from
// *t_cur.  Traffic: the mask byte of each token, plus known (4 B) and x (4 B) per element of a known token.
struct ReplaceP {
  float* x;
  const float *known, *noise;
  const unsigned char* mask;
  long long n, per_token, per_sample;
  float sa, sb;
  unsigned long long seed;
  const unsigned long long* keys;
  long long t;
  const float* coef;
  const int* step;
  const long long* t_cur;
};
__global__ void __launch_bounds__(256) replace_known_kernel(const ReplaceP p) {
  float sa = p.sa, sb = p.sb;
  long long t = p.t;
  if (p.coef) {
    const float* cf = p.coef + 2 * (long long)*p.step;
    sa = cf[0]; sb = cf[1];
    t = *p.t_cur;
  }
  const long long gps = (p.per_sample + 3) / 4, ng = (p.n / p.per_sample) * gps;
  for (long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x; g < ng; g += (long long)gridDim.x * blockDim.x) {
    const long long b = g / gps, q = g - b * gps;
    const long long base = b * p.per_sample, js0 = q * 4;
    const int cnt = (int)min(4ll, p.per_sample - js0);
    bool known[4] = {false, false, false, false};
    if (!known_flags(p.mask, base + js0, p.per_token, cnt, known)) continue;
    float z[4] = {0.f, 0.f, 0.f, 0.f};
    if (p.noise == nullptr) keyed_normal4(p.keys ? p.keys[b] : p.seed, (unsigned long long)q, (uint32_t)t, 2u, z);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (!known[j]) continue;
      const long long i = base + js0 + j;
      const float kv = p.known[i];
      // sb == 0 (the last step, abar_prev = 1): sa*kv keeps the sign of a zero, so the token ends at known bit for bit
      p.x[i] = sb == 0.f ? sa * kv : fmaf(sa, kv, sb * (p.noise ? p.noise[i] : z[j]));
    }
  }
}

// RePaint step (diffusers 0.27 RePaintScheduler.step, epsilon prediction): the DDIM update of ddim_step_kernel for the
// unknown tokens, written with exactly its expressions (so with nothing known and the same noise it is bg_ddim_step bit
// for bit), and for the elements of tokens whose mask byte is set the known part sa_prev*known + sb_prev*z, written as
// replace_known_kernel writes it.  One z serves both: the variance term sigma*z and the known part draw the same normal.
// z is drawn only when sigma != 0 or the group holds a known token: explicit `noise`, else per-sample keys
// (keyed_normal4, domain 3, counter word k = the entry's index in the stage's RePaint list), else the batch key `seed`
// over the whole tensor as one sample.  Table form (coef != NULL): (sb, sa, sa_prev, c_dir, sigma, sb_prev) from
// coef[6 * *step] and k = *step.
struct RepaintP {
  const float *eps_c, *eps_u, *x, *noise, *known;
  float* out;
  const unsigned char* mask;
  long long n, per_token, per_sample;
  float w, sb, sa, sa_prev, c_dir, sigma, sb_prev, clip;
  unsigned long long seed;
  const unsigned long long* keys;
  long long k;
  const float* coef;
  const int* step;
};
__global__ void __launch_bounds__(256) repaint_step_kernel(const RepaintP p) {
  float sb = p.sb, sa = p.sa, sa_prev = p.sa_prev, c_dir = p.c_dir, sigma = p.sigma, sb_prev = p.sb_prev;
  long long k = p.k;
  if (p.coef) {
    k = *p.step;
    const float* cf = p.coef + 6 * k;
    sb = cf[0]; sa = cf[1]; sa_prev = cf[2]; c_dir = cf[3]; sigma = cf[4]; sb_prev = cf[5];
  }
  const long long gps = (p.per_sample + 3) / 4, ng = (p.n / p.per_sample) * gps;
  for (long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x; g < ng; g += (long long)gridDim.x * blockDim.x) {
    const long long b = g / gps, q = g - b * gps;
    const long long base = b * p.per_sample, js0 = q * 4;
    const int cnt = (int)min(4ll, p.per_sample - js0);
    bool known[4] = {false, false, false, false};
    const bool any = p.mask && known_flags(p.mask, base + js0, p.per_token, cnt, known);
    float z[4] = {0.f, 0.f, 0.f, 0.f};
    if ((sigma != 0.f || any) && p.noise == nullptr)
      keyed_normal4(p.keys ? p.keys[b] : p.seed, (unsigned long long)q, (uint32_t)k, 3u, z);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (j >= cnt) break;
      const long long i = base + js0 + j;
      const float zj = p.noise && (sigma != 0.f || known[j]) ? p.noise[i] : z[j];
      float o;
      if (known[j]) {
        const float kv = p.known[i];
        // sb_prev == 0 (the last step, abar_prev = 1): sa_prev*kv keeps the sign of a zero, so the token ends at known
        o = sb_prev == 0.f ? __fmul_rn(sa_prev, kv) : __fmaf_rn(sa_prev, kv, __fmul_rn(sb_prev, zj));
      } else {
        // the roundings ddim_step_kernel compiles to (its FMA contractions spelled out, so no other contraction can
        // differ):  e*(1+w) - eu*w;  (x - sb*e) / sa;  sa_prev*x0 + c_dir*e;  + sigma*z
        float e = p.eps_c[i];
        if (p.eps_u) e = __fmaf_rn(e, 1.f + p.w, -__fmul_rn(p.eps_u[i], p.w));
        const float xv = p.x[i];
        float x0 = __fdiv_rn(__fmaf_rn(-sb, e, xv), sa);
        if (p.clip > 0.f) x0 = fminf(fmaxf(x0, -p.clip), p.clip);
        o = __fmaf_rn(sa_prev, x0, __fmul_rn(c_dir, e));
        if (sigma != 0.f) o = __fmaf_rn(sigma, zj, o);
      }
      p.out[i] = o;
    }
  }
}

// RePaint undo (diffusers 0.27 RePaintScheduler.undo_step): n_trans forward-diffusion transitions of one undo entry in
// registers, in place, x = sqrt(1-beta_i)*x + sqrt(beta_i)*z_i for i = 0..n_trans-1, every product and the sum rounded
// on their own (the fp32 torch chain).  cf[2i], cf[2i+1] = (sqrt(1-beta), sqrt(beta)) of transition i.  z_i: explicit
// `noise` of shape (n_trans, n), else per-sample keys (keyed_normal4, domain 4, counter word k * n_trans + i), else the
// batch key `seed` over the whole tensor as one sample.  Table form (coef != NULL): cf = coef + 2 * n_trans * *step and
// k = *step.
struct UndoP {
  float* x;
  const float* noise;
  long long n, per_sample;
  int n_trans;
  const float* cf;
  unsigned long long seed;
  const unsigned long long* keys;
  long long k;
  const float* coef;
  const int* step;
};
__global__ void __launch_bounds__(256) repaint_undo_kernel(const UndoP p) {
  const float* cf = p.cf;
  long long k = p.k;
  if (p.coef) {
    k = *p.step;
    cf = p.coef + 2ll * p.n_trans * k;
  }
  const long long gps = (p.per_sample + 3) / 4, ng = (p.n / p.per_sample) * gps;
  for (long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x; g < ng; g += (long long)gridDim.x * blockDim.x) {
    const long long b = g / gps, q = g - b * gps;
    const long long i0 = b * p.per_sample + q * 4;
    const int cnt = (int)min(4ll, p.per_sample - q * 4);
    const unsigned long long key = p.keys ? p.keys[b] : p.seed;
    float v[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) v[j] = j < cnt ? p.x[i0 + j] : 0.f;
#pragma unroll 1
    for (int s = 0; s < p.n_trans; ++s) {
      const float a = cf[2 * s], c = cf[2 * s + 1];
      float z[4];
      if (p.noise) {
        const float* nz = p.noise + (long long)s * p.n + i0;
#pragma unroll
        for (int j = 0; j < 4; ++j) z[j] = j < cnt ? nz[j] : 0.f;
      } else {
        keyed_normal4(key, (unsigned long long)q, (uint32_t)(k * p.n_trans + s), 4u, z);
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) v[j] = __fadd_rn(__fmul_rn(a, v[j]), __fmul_rn(c, z[j]));
    }
#pragma unroll
    for (int j = 0; j < 4; ++j)
      if (j < cnt) p.x[i0 + j] = v[j];
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
// Per-sample classifier-free combine (mixed-class batches): sample b of eps_c is guided by row uncond_row[b] of eps_u
// with weight w[b], each operation rounded on its own (the fp32 torch expression pc*(1+w) - pu[row]*w, as dpm_step_kernel
// and unipc_step_kernel round their fused combine); uncond_row[b] == -1 leaves the sample as it is (copied, or neither
// read nor written when out aliases eps_c); any other row outside [0, n_uncond) writes NaN.  One thread per group of 4
// elements of a sample, as launch_grouped; float4 accesses when every row starts 16-byte aligned (vec), else scalar
// accesses with the sample's last group cut to per_sample % 4 elements.
struct CfgP {
  const float *eps_c, *eps_u, *w;
  const int* row;
  float* out;
  long long n_samples, n_uncond, per_sample;
  bool vec;
};
__global__ void __launch_bounds__(256) cfg_combine_kernel(const CfgP p) {
  const long long gps = (p.per_sample + 3) / 4, ng = p.n_samples * gps;
  for (long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x; g < ng; g += (long long)gridDim.x * blockDim.x) {
    const long long b = g / gps, q = g - b * gps;
    const long long r = p.row[b];
    const long long i0 = b * p.per_sample + q * 4;
    if (r == -1 && p.out == p.eps_c) continue;
    const int cnt = (int)min(4ll, p.per_sample - q * 4);
    float e[4], u[4] = {0.f, 0.f, 0.f, 0.f};
    const bool bad = r < -1 || r >= p.n_uncond;
    const float* pu = (r >= 0 && !bad) ? p.eps_u + r * p.per_sample + q * 4 : nullptr;
    if (p.vec) {
      const float4 v = *reinterpret_cast<const float4*>(p.eps_c + i0);
      e[0] = v.x; e[1] = v.y; e[2] = v.z; e[3] = v.w;
      if (pu) {
        const float4 y = __ldg(reinterpret_cast<const float4*>(pu));
        u[0] = y.x; u[1] = y.y; u[2] = y.z; u[3] = y.w;
      }
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        e[j] = j < cnt ? p.eps_c[i0 + j] : 0.f;
        if (pu && j < cnt) u[j] = pu[j];
      }
    }
    if (bad) {
#pragma unroll
      for (int j = 0; j < 4; ++j) e[j] = __int_as_float(0x7fc00000);
    } else if (pu) {
      const float wb = p.w[b], w1 = __fadd_rn(1.f, wb);
#pragma unroll
      for (int j = 0; j < 4; ++j) e[j] = __fsub_rn(__fmul_rn(e[j], w1), __fmul_rn(u[j], wb));
    }
    if (p.vec) {
      *reinterpret_cast<float4*>(p.out + i0) = make_float4(e[0], e[1], e[2], e[3]);
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (j < cnt) p.out[i0 + j] = e[j];
    }
  }
}

__global__ void __launch_bounds__(256) axpby_kernel(const float* x, float a, const float* y, float b, float* out, long long n) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    out[i] = a * x[i] + (y ? b * y[i] : 0.f);
}

// Spherical interpolation of two noises per sample (B-rep interpolation between two DDIM-inverted designs).  One CTA per
// sample: a.b, |a|^2 and |b|^2 over the elements of unmasked tokens, each thread summing a fixed stride of elements in
// fp64 and then a fixed shared-memory tree, so the result depends on neither the batch nor the launch; then
//   theta = acos(clamp(cos, -1, 1)),  out = sin((1-alpha) theta)/sin theta * a + sin(alpha theta)/sin theta * b,
// or the lerp (1-alpha) a + alpha b when |cos| > 0.9995 or a norm is zero, in fp64 rounded once to fp32.  alpha == 0 and
// alpha == 1 copy a and b; masked tokens copy a.  Every element is read in the reduction before the barrier and written
// only after it by the thread that reads it again, so out may alias a.
constexpr int kSlerpThreads = 512;
struct SlerpP {
  const float *a, *b, *alpha;
  const unsigned char* mask;
  float* out;
  long long per_sample, per_token;
};
__global__ void __launch_bounds__(kSlerpThreads) slerp_kernel(const SlerpP p) {
  __shared__ double red[3][kSlerpThreads];
  const int tid = threadIdx.x;
  const long long base = (long long)blockIdx.x * p.per_sample;
  const float* a = p.a + base;
  const float* b = p.b + base;
  float* o = p.out + base;
  const unsigned char* m = p.mask ? p.mask + base / p.per_token : nullptr;
  const float al = p.alpha[blockIdx.x];
  double ab = 0.0, aa = 0.0, bb = 0.0;
  for (long long i = tid; i < p.per_sample; i += kSlerpThreads) {
    if (m && m[i / p.per_token]) continue;
    const double x = a[i], y = b[i];
    ab = fma(x, y, ab);
    aa = fma(x, x, aa);
    bb = fma(y, y, bb);
  }
  red[0][tid] = ab; red[1][tid] = aa; red[2][tid] = bb;
  for (int s = kSlerpThreads / 2; s > 0; s >>= 1) {
    __syncthreads();
    if (tid < s) {
      red[0][tid] += red[0][tid + s];
      red[1][tid] += red[1][tid + s];
      red[2][tid] += red[2][tid + s];
    }
  }
  __syncthreads();
  const int mode = al == 0.f ? 0 : (al == 1.f ? 1 : 2);   // copy a, copy b, combine
  double ca = 1.0 - (double)al, cb = (double)al;          // the lerp
  if (mode == 2) {
    const double nn = sqrt(red[1][0] * red[2][0]);
    const double c = nn > 0.0 ? fmin(fmax(red[0][0] / nn, -1.0), 1.0) : 1.0;
    if (fabs(c) <= 0.9995) {
      const double th = acos(c), s = sin(th);
      ca = sin((1.0 - (double)al) * th) / s;
      cb = sin((double)al * th) / s;
    }
  }
  for (long long i = tid; i < p.per_sample; i += kSlerpThreads) {
    const float x = a[i];
    float v = x;
    if (!(m && m[i / p.per_token])) {
      if (mode == 1) v = b[i];
      else if (mode == 2) v = (float)fma(ca, (double)x, cb * (double)b[i]);
    }
    o[i] = v;
  }
}

inline unsigned grid_for(long long work) {
  long long blocks = (work + 255) / 256;
  const long long cap = (long long)num_sms() * 16;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  return (unsigned)blocks;
}

// Launches one of the grouped step kernels (one thread per group of 4 elements of a sample) over n / per_sample samples.
// Without sample keys the whole tensor is one sample (per_sample = n), so a group is the batch stream's element group.
template <class P>
int launch_grouped(void (*kernel)(P), P& p, const uint64_t* sample_keys, int64_t per_sample, void* stream,
                   const char* what) {
  p.keys = reinterpret_cast<const unsigned long long*>(sample_keys);
  p.per_sample = sample_keys ? per_sample : p.n;
  kernel<<<grid_for((p.n / p.per_sample) * ((p.per_sample + 3) / 4)), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(p);
  return check_launch(what);
}

// One thread per group of 4 elements of a sample, as launch_grouped; the step draws no noise, so it takes no keys.
int launch_unipc(UnipcP& p, int64_t per_sample, void* stream) {
  p.per_sample = per_sample;
  unipc_step_kernel<<<grid_for((p.n / per_sample) * ((per_sample + 3) / 4)), 256, 0,
                      reinterpret_cast<cudaStream_t>(stream)>>>(p);
  return check_launch("unipc_step_kernel launch");
}

}  // namespace
}  // namespace bg

using namespace bg;

extern "C" {

int bg_ddpm_step(const float* eps_cond, const float* eps_uncond, float cfg_w, const float* x, float* out,
                 const float* noise, uint64_t seed, uint64_t offset, const uint64_t* sample_keys, int64_t per_sample,
                 int64_t t, int64_t n, float sqrt_one_minus_abar, float sqrt_abar, float clip, float c_x0, float c_x,
                 float sigma, void* stream) {
  BG_REQUIRE(eps_cond && x && out && n > 0, "ddpm_step: bad arguments");
  BG_REQUIRE(!sample_keys || (per_sample > 0 && n % per_sample == 0),
             "ddpm_step: n must be a positive multiple of per_sample");
  BG_REQUIRE(t >= 0 && t <= 0xFFFFFFFFll, "ddpm_step: t must be a 32-bit unsigned value");
  BG_REQUIRE(sqrt_abar > 0.f, "ddpm_step: sqrt_abar must be positive");
  DdpmP p = {};
  p.eps_c = eps_cond; p.eps_u = eps_uncond; p.x = x; p.noise = noise; p.out = out; p.n = n;
  p.w = cfg_w; p.sb = sqrt_one_minus_abar; p.sa = sqrt_abar; p.c_x0 = c_x0; p.c_x = c_x; p.sigma = sigma; p.clip = clip;
  p.t = t; p.seed = seed; p.offset = offset;
  return launch_grouped(ddpm_step_kernel, p, sample_keys, per_sample, stream, "ddpm_step_kernel launch");
}

int bg_ddpm_step_tab(const float* eps_cond, const float* eps_uncond, float cfg_w, const float* x, float* out, uint64_t seed,
                     uint64_t offset0, uint64_t offset_stride, const uint64_t* sample_keys, int64_t per_sample,
                     const int64_t* t_cur, int64_t n, const float* coef_table, const int32_t* step, float clip,
                     void* stream) {
  BG_REQUIRE(eps_cond && x && out && n > 0 && coef_table && step, "ddpm_step_tab: bad arguments");
  BG_REQUIRE(!sample_keys || (t_cur && per_sample > 0 && n % per_sample == 0),
             "ddpm_step_tab: keyed noise needs t_cur and n a positive multiple of per_sample");
  DdpmP p = {};
  p.eps_c = eps_cond; p.eps_u = eps_uncond; p.x = x; p.out = out; p.n = n; p.w = cfg_w; p.clip = clip;
  p.seed = seed; p.offset = offset0; p.offset_stride = offset_stride;
  p.coef = coef_table; p.step = step; p.t_cur = reinterpret_cast<const long long*>(t_cur);
  return launch_grouped(ddpm_step_kernel, p, sample_keys, per_sample, stream, "ddpm_step_kernel launch");
}

int bg_randn_keyed(const uint64_t* sample_keys, int64_t n_samples, int64_t per_sample, int32_t domain, int64_t t, float* out,
                   void* stream) {
  BG_REQUIRE(sample_keys && out, "randn_keyed: sample_keys and out must not be NULL");
  BG_REQUIRE(n_samples > 0 && per_sample > 0, "randn_keyed: n_samples and per_sample must be positive");
  BG_REQUIRE(domain >= 0 && t >= 0 && t <= 0xFFFFFFFFll, "randn_keyed: domain and t must be 32-bit unsigned values");
  RandnKeyedP p;
  p.keys = reinterpret_cast<const unsigned long long*>(sample_keys); p.out = out;
  p.n_samples = n_samples; p.per_sample = per_sample; p.domain = (uint32_t)domain; p.t = (uint32_t)t;
  randn_keyed_kernel<<<grid_for(n_samples * ((per_sample + 3) / 4)), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(p);
  return check_launch("randn_keyed_kernel launch");
}

int bg_add_noise_gather(const float* src, int64_t n_src_tokens, const int32_t* index, int64_t n_tokens, int32_t dim,
                        float scale, float sqrt_abar, float sqrt_one_minus_abar, const float* noise,
                        const uint64_t* sample_keys, int64_t tokens_per_sample, int32_t domain, int64_t t, float* out,
                        void* stream) {
  BG_REQUIRE(src && index && out && n_src_tokens > 0 && n_tokens > 0 && dim > 0, "add_noise_gather: bad arguments");
  BG_REQUIRE((noise == nullptr) != (sample_keys == nullptr), "add_noise_gather: give exactly one of noise and sample_keys");
  BG_REQUIRE(!sample_keys || (tokens_per_sample > 0 && n_tokens % tokens_per_sample == 0),
             "add_noise_gather: n_tokens must be a positive multiple of tokens_per_sample");
  BG_REQUIRE(domain >= 0 && t >= 0 && t <= 0xFFFFFFFFll, "add_noise_gather: domain and t must be 32-bit unsigned values");
  GatherP p = {};
  p.src = src; p.noise = noise; p.index = index; p.out = out;
  p.n = n_tokens * dim; p.per_token = dim; p.n_src = n_src_tokens;
  p.scale = scale; p.sa = sqrt_abar; p.sb = sqrt_one_minus_abar;
  p.keys = reinterpret_cast<const unsigned long long*>(sample_keys);
  p.per_sample = sample_keys ? tokens_per_sample * dim : p.n;
  p.t = (uint32_t)t; p.domain = (uint32_t)domain;
  add_noise_gather_kernel<<<grid_for((p.n / p.per_sample) * ((p.per_sample + 3) / 4)), 256, 0,
                            reinterpret_cast<cudaStream_t>(stream)>>>(p);
  return check_launch("add_noise_gather_kernel launch");
}

int bg_ddim_step(const float* eps_cond, const float* eps_uncond, float cfg_w, const float* x, float* out,
                 const float* noise, uint64_t seed, uint64_t offset, const uint64_t* sample_keys, int64_t per_sample,
                 int64_t t, int64_t n, float sqrt_one_minus_abar, float sqrt_abar, float sqrt_abar_prev, float c_dir,
                 float sigma, float clip, int32_t use_clipped_eps, void* stream) {
  BG_REQUIRE(eps_cond && x && out && n > 0, "ddim_step: bad arguments");
  BG_REQUIRE(!sample_keys || (per_sample > 0 && n % per_sample == 0),
             "ddim_step: n must be a positive multiple of per_sample");
  BG_REQUIRE(t >= 0 && t <= 0xFFFFFFFFll, "ddim_step: t must be a 32-bit unsigned value");
  BG_REQUIRE(sqrt_abar > 0.f, "ddim_step: sqrt_abar must be positive");
  DdimP p = {};
  p.eps_c = eps_cond; p.eps_u = eps_uncond; p.x = x; p.noise = noise; p.out = out; p.n = n;
  p.w = cfg_w; p.sb = sqrt_one_minus_abar; p.sa = sqrt_abar; p.sa_prev = sqrt_abar_prev; p.c_dir = c_dir; p.sigma = sigma;
  p.clip = clip; p.use_clipped_eps = use_clipped_eps != 0; p.t = t; p.seed = seed; p.offset = offset;
  return launch_grouped(ddim_step_kernel, p, sample_keys, per_sample, stream, "ddim_step_kernel launch");
}

int bg_ddim_step_tab(const float* eps_cond, const float* eps_uncond, float cfg_w, const float* x, float* out, uint64_t seed,
                     uint64_t offset0, uint64_t offset_stride, const uint64_t* sample_keys, int64_t per_sample,
                     const int64_t* t_cur, int64_t n, const float* coef_table, const int32_t* step, float clip,
                     int32_t use_clipped_eps, void* stream) {
  BG_REQUIRE(eps_cond && x && out && n > 0 && coef_table && step, "ddim_step_tab: bad arguments");
  BG_REQUIRE(!sample_keys || (t_cur && per_sample > 0 && n % per_sample == 0),
             "ddim_step_tab: keyed noise needs t_cur and n a positive multiple of per_sample");
  DdimP p = {};
  p.eps_c = eps_cond; p.eps_u = eps_uncond; p.x = x; p.out = out; p.n = n; p.w = cfg_w; p.clip = clip;
  p.use_clipped_eps = use_clipped_eps != 0; p.seed = seed; p.offset = offset0; p.offset_stride = offset_stride;
  p.coef = coef_table; p.step = step; p.t_cur = reinterpret_cast<const long long*>(t_cur);
  return launch_grouped(ddim_step_kernel, p, sample_keys, per_sample, stream, "ddim_step_kernel launch");
}

int bg_dpm_step(const float* eps_cond, const float* eps_uncond, float cfg_w, const float* x, float* out, float* hist,
                const float* noise, uint64_t seed, uint64_t offset, const uint64_t* sample_keys, int64_t per_sample,
                int64_t t, int64_t n, float alpha_s, float sigma_s, float c_x, float c_0, float c_1, float inv_r0, float c_z,
                float clip, void* stream) {
  BG_REQUIRE(eps_cond && x && out && n > 0, "dpm_step: bad arguments");
  BG_REQUIRE(hist || c_1 == 0.f, "dpm_step: a second-order step (c_1 != 0) needs hist");
  BG_REQUIRE(!sample_keys || (per_sample > 0 && n % per_sample == 0),
             "dpm_step: n must be a positive multiple of per_sample");
  BG_REQUIRE(t >= 0 && t <= 0xFFFFFFFFll, "dpm_step: t must be a 32-bit unsigned value");
  BG_REQUIRE(alpha_s > 0.f, "dpm_step: alpha_s must be positive");
  DpmP p = {};
  p.eps_c = eps_cond; p.eps_u = eps_uncond; p.x = x; p.noise = noise; p.out = out; p.hist = hist; p.n = n; p.w = cfg_w;
  p.alpha_s = alpha_s; p.sigma_s = sigma_s; p.c_x = c_x; p.c_0 = c_0; p.c_1 = c_1; p.inv_r0 = inv_r0; p.c_z = c_z;
  p.clip = clip; p.t = t; p.seed = seed; p.offset = offset;
  return launch_grouped(dpm_step_kernel, p, sample_keys, per_sample, stream, "dpm_step_kernel launch");
}

int bg_dpm_step_tab(const float* eps_cond, const float* eps_uncond, float cfg_w, const float* x, float* out, float* hist,
                    uint64_t seed, uint64_t offset0, uint64_t offset_stride, const uint64_t* sample_keys, int64_t per_sample,
                    const int64_t* t_cur, int64_t n, const float* coef_table, const int32_t* step, float clip, void* stream) {
  BG_REQUIRE(eps_cond && x && out && hist && n > 0 && coef_table && step, "dpm_step_tab: bad arguments");
  BG_REQUIRE(!sample_keys || (t_cur && per_sample > 0 && n % per_sample == 0),
             "dpm_step_tab: keyed noise needs t_cur and n a positive multiple of per_sample");
  DpmP p = {};
  p.eps_c = eps_cond; p.eps_u = eps_uncond; p.x = x; p.out = out; p.hist = hist; p.n = n; p.w = cfg_w; p.clip = clip;
  p.seed = seed; p.offset = offset0; p.offset_stride = offset_stride;
  p.coef = coef_table; p.step = step; p.t_cur = reinterpret_cast<const long long*>(t_cur);
  return launch_grouped(dpm_step_kernel, p, sample_keys, per_sample, stream, "dpm_step_kernel launch");
}

int bg_unipc_step(const float* eps_cond, const float* eps_uncond, float cfg_w, const float* x, float* out, float* last,
                  float* hist, int32_t n_slots, int64_t per_sample, int64_t n, const float* coef, float clip,
                  void* stream) {
  BG_REQUIRE(eps_cond && x && out && hist && coef && n > 0, "unipc_step: bad arguments");
  BG_REQUIRE(per_sample > 0 && n % per_sample == 0, "unipc_step: n must be a positive multiple of per_sample");
  BG_REQUIRE(n_slots >= 1 && n_slots <= 3, "unipc_step: n_slots must be 1, 2 or 3");
  BG_REQUIRE(coef[0] > 0.f, "unipc_step: alpha_s must be positive");
  const float fc = coef[2], fp = coef[3];
  BG_REQUIRE((fc == 0.f || fc == 1.f || fc == 2.f || fc == 3.f) && (fp == 1.f || fp == 2.f || fp == 3.f),
             "unipc_step: the corrector order must be 0-3 and the predictor order 1-3");
  BG_REQUIRE(last || fc == 0.f, "unipc_step: a corrector step needs last");
  const int reads = max((int)fc, (int)fp - 1);
  for (int s = 4; s < 8; ++s)
    BG_REQUIRE(s - 4 > reads || (coef[s] == floorf(coef[s]) && coef[s] >= 0.f && coef[s] < (float)n_slots),
               "unipc_step: a slot the step uses lies outside the ring of n_slots slots");
  UnipcP p = {};
  p.eps_c = eps_cond; p.eps_u = eps_uncond; p.x = x; p.out = out; p.last = last; p.hist = hist; p.n = n;
  p.w = cfg_w; p.clip = clip;
  for (int j = 0; j < BG_UNIPC_ROW; ++j) p.row[j] = coef[j];
  return launch_unipc(p, per_sample, stream);
}

int bg_unipc_step_tab(const float* eps_cond, const float* eps_uncond, float cfg_w, const float* x, float* out, float* last,
                      float* hist, int64_t per_sample, int64_t n, const float* coef_table, const int32_t* step, float clip,
                      void* stream) {
  BG_REQUIRE(eps_cond && x && out && last && hist && coef_table && step && n > 0, "unipc_step_tab: bad arguments");
  BG_REQUIRE(per_sample > 0 && n % per_sample == 0, "unipc_step_tab: n must be a positive multiple of per_sample");
  UnipcP p = {};
  p.eps_c = eps_cond; p.eps_u = eps_uncond; p.x = x; p.out = out; p.last = last; p.hist = hist; p.n = n;
  p.w = cfg_w; p.clip = clip; p.coef = coef_table; p.step = step;
  return launch_unipc(p, per_sample, stream);
}

int bg_replace_known(float* x, const float* known, const uint8_t* token_mask, int64_t n, int64_t per_token,
                     const float* noise, uint64_t seed, const uint64_t* sample_keys, int64_t per_sample, int64_t t_ctr,
                     float sqrt_abar, float sqrt_one_minus_abar, void* stream) {
  BG_REQUIRE(x && known && token_mask && n > 0, "replace_known: bad arguments");
  BG_REQUIRE(per_token > 0 && n % per_token == 0, "replace_known: n must be a positive multiple of per_token");
  BG_REQUIRE(!sample_keys || (per_sample > 0 && per_sample % per_token == 0 && n % per_sample == 0),
             "replace_known: per_sample must be a positive multiple of per_token that divides n");
  BG_REQUIRE(t_ctr >= 0 && t_ctr <= 0xFFFFFFFFll, "replace_known: t_ctr must be a 32-bit unsigned value");
  ReplaceP p = {};
  p.x = x; p.known = known; p.noise = noise; p.mask = token_mask; p.n = n; p.per_token = per_token;
  p.sa = sqrt_abar; p.sb = sqrt_one_minus_abar; p.seed = seed; p.t = t_ctr;
  return launch_grouped(replace_known_kernel, p, sample_keys, per_sample, stream, "replace_known_kernel launch");
}

int bg_replace_known_tab(float* x, const float* known, const uint8_t* token_mask, int64_t n, int64_t per_token,
                         uint64_t seed, const uint64_t* sample_keys, int64_t per_sample, const int64_t* t_cur,
                         const float* coef_table, const int32_t* step, void* stream) {
  BG_REQUIRE(x && known && token_mask && n > 0 && t_cur && coef_table && step, "replace_known_tab: bad arguments");
  BG_REQUIRE(per_token > 0 && n % per_token == 0, "replace_known_tab: n must be a positive multiple of per_token");
  BG_REQUIRE(!sample_keys || (per_sample > 0 && per_sample % per_token == 0 && n % per_sample == 0),
             "replace_known_tab: per_sample must be a positive multiple of per_token that divides n");
  ReplaceP p = {};
  p.x = x; p.known = known; p.mask = token_mask; p.n = n; p.per_token = per_token; p.seed = seed;
  p.coef = coef_table; p.step = step; p.t_cur = reinterpret_cast<const long long*>(t_cur);
  return launch_grouped(replace_known_kernel, p, sample_keys, per_sample, stream, "replace_known_kernel launch");
}

int bg_repaint_step(const float* eps_cond, const float* eps_uncond, float cfg_w, const float* x, float* out,
                    const float* known, const uint8_t* token_mask, int64_t per_token, const float* noise, uint64_t seed,
                    const uint64_t* sample_keys, int64_t per_sample, int64_t k, int64_t n, float sqrt_one_minus_abar,
                    float sqrt_abar, float sqrt_abar_prev, float c_dir, float sigma, float sqrt_one_minus_abar_prev,
                    float clip, void* stream) {
  BG_REQUIRE(eps_cond && x && out && n > 0, "repaint_step: bad arguments");
  BG_REQUIRE((known == nullptr) == (token_mask == nullptr), "repaint_step: give known and token_mask together or neither");
  BG_REQUIRE(!token_mask || (per_token > 0 && n % per_token == 0),
             "repaint_step: n must be a positive multiple of per_token");
  BG_REQUIRE(!sample_keys || (per_sample > 0 && n % per_sample == 0 && (!token_mask || per_sample % per_token == 0)),
             "repaint_step: per_sample must be a positive multiple of per_token that divides n");
  BG_REQUIRE(k >= 0 && k <= 0xFFFFFFFFll, "repaint_step: k must be a 32-bit unsigned value");
  BG_REQUIRE(sqrt_abar > 0.f, "repaint_step: sqrt_abar must be positive");
  RepaintP p = {};
  p.eps_c = eps_cond; p.eps_u = eps_uncond; p.x = x; p.out = out; p.known = known; p.mask = token_mask; p.noise = noise;
  p.n = n; p.per_token = per_token; p.w = cfg_w; p.sb = sqrt_one_minus_abar; p.sa = sqrt_abar; p.sa_prev = sqrt_abar_prev;
  p.c_dir = c_dir; p.sigma = sigma; p.sb_prev = sqrt_one_minus_abar_prev; p.clip = clip; p.seed = seed; p.k = k;
  return launch_grouped(repaint_step_kernel, p, sample_keys, per_sample, stream, "repaint_step_kernel launch");
}

int bg_repaint_step_tab(const float* eps_cond, const float* eps_uncond, float cfg_w, const float* x, float* out,
                        const float* known, const uint8_t* token_mask, int64_t per_token, uint64_t seed,
                        const uint64_t* sample_keys, int64_t per_sample, int64_t n, const float* coef_table,
                        const int32_t* step, float clip, void* stream) {
  BG_REQUIRE(eps_cond && x && out && n > 0 && coef_table && step, "repaint_step_tab: bad arguments");
  BG_REQUIRE((known == nullptr) == (token_mask == nullptr),
             "repaint_step_tab: give known and token_mask together or neither");
  BG_REQUIRE(!token_mask || (per_token > 0 && n % per_token == 0),
             "repaint_step_tab: n must be a positive multiple of per_token");
  BG_REQUIRE(!sample_keys || (per_sample > 0 && n % per_sample == 0 && (!token_mask || per_sample % per_token == 0)),
             "repaint_step_tab: per_sample must be a positive multiple of per_token that divides n");
  RepaintP p = {};
  p.eps_c = eps_cond; p.eps_u = eps_uncond; p.x = x; p.out = out; p.known = known; p.mask = token_mask; p.n = n;
  p.per_token = per_token; p.w = cfg_w; p.clip = clip; p.seed = seed; p.coef = coef_table; p.step = step;
  return launch_grouped(repaint_step_kernel, p, sample_keys, per_sample, stream, "repaint_step_kernel launch");
}

int bg_repaint_undo(float* x, int64_t n, int32_t n_trans, const float* coef, const float* noise, uint64_t seed,
                    const uint64_t* sample_keys, int64_t per_sample, int64_t k, void* stream) {
  BG_REQUIRE(x && coef && n > 0 && n_trans > 0, "repaint_undo: bad arguments");
  BG_REQUIRE(!sample_keys || (per_sample > 0 && n % per_sample == 0),
             "repaint_undo: n must be a positive multiple of per_sample");
  BG_REQUIRE(k >= 0 && (k + 1) * (int64_t)n_trans <= 0x100000000ll,
             "repaint_undo: the counter words k * n_trans + i must be 32-bit unsigned values");
  UndoP p = {};
  p.x = x; p.noise = noise; p.n = n; p.n_trans = n_trans; p.cf = coef; p.seed = seed; p.k = k;
  return launch_grouped(repaint_undo_kernel, p, sample_keys, per_sample, stream, "repaint_undo_kernel launch");
}

int bg_repaint_undo_tab(float* x, int64_t n, int32_t n_trans, uint64_t seed, const uint64_t* sample_keys,
                        int64_t per_sample, const float* coef_table, const int32_t* step, void* stream) {
  BG_REQUIRE(x && coef_table && step && n > 0 && n_trans > 0, "repaint_undo_tab: bad arguments");
  BG_REQUIRE(!sample_keys || (per_sample > 0 && n % per_sample == 0),
             "repaint_undo_tab: n must be a positive multiple of per_sample");
  UndoP p = {};
  p.x = x; p.n = n; p.n_trans = n_trans; p.seed = seed; p.coef = coef_table; p.step = step;
  return launch_grouped(repaint_undo_kernel, p, sample_keys, per_sample, stream, "repaint_undo_kernel launch");
}

int bg_slerp(const float* a, const float* b, const float* alpha, const uint8_t* token_mask, int64_t n_samples,
             int64_t per_sample, int64_t per_token, float* out, void* stream) {
  BG_REQUIRE(a && b && alpha && out, "slerp: a, b, alpha and out must not be NULL");
  BG_REQUIRE(n_samples > 0 && n_samples <= 0x7FFFFFFFll && per_sample > 0 && per_token > 0,
             "slerp: n_samples (at most 2^31 - 1), per_sample and per_token must be positive");
  BG_REQUIRE(per_sample % per_token == 0, "slerp: per_sample must be a multiple of per_token");
  SlerpP p;
  p.a = a; p.b = b; p.alpha = alpha; p.mask = token_mask; p.out = out; p.per_sample = per_sample; p.per_token = per_token;
  slerp_kernel<<<(unsigned)n_samples, kSlerpThreads, 0, reinterpret_cast<cudaStream_t>(stream)>>>(p);
  return check_launch("slerp_kernel launch");
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

int bg_cfg_combine(const float* eps_c, const float* eps_u, const int32_t* uncond_row, const float* w, int64_t n_samples,
                   int64_t n_uncond, int64_t per_sample, float* out, void* stream) {
  BG_REQUIRE(eps_c && uncond_row && w && out && (eps_u || n_uncond == 0), "cfg_combine: bad arguments");
  BG_REQUIRE(n_samples > 0 && per_sample > 0 && n_uncond >= 0, "cfg_combine: n_samples and per_sample must be positive, "
             "n_uncond non-negative");
  BG_REQUIRE(n_samples <= INT64_MAX / per_sample && n_uncond <= INT64_MAX / per_sample, "cfg_combine: sizes overflow");
  CfgP p;
  p.eps_c = eps_c; p.eps_u = eps_u; p.w = w; p.row = uncond_row; p.out = out;
  p.n_samples = n_samples; p.n_uncond = n_uncond; p.per_sample = per_sample;
  const auto a16 = [](const void* q) { return q == nullptr || (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
  p.vec = per_sample % 4 == 0 && a16(eps_c) && a16(eps_u) && a16(out);
  cfg_combine_kernel<<<grid_for(n_samples * ((per_sample + 3) / 4)), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(p);
  return check_launch("cfg_combine_kernel launch");
}

int bg_axpby(const float* x, float a, const float* y, float b, float* out, int64_t n, void* stream) {
  BG_REQUIRE(x && out && n > 0, "axpby: bad arguments");
  axpby_kernel<<<grid_for(n), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(x, a, y, b, out, n);
  return check_launch("axpby_kernel launch");
}

}  // extern "C"
