/* brepgen_b200 -- C ABI of the H100-native BrepGen sampling path (libbrepgen_b200.so).
 *
 * The reference (samxuxiang/BrepGen) is pure Python and has NO FFI of its own: its boundary for this path is the
 * Python class surface  SurfPosNet/SurfZNet/EdgePosNet/EdgeZNet.forward (network.py:1107,1176,1257,1357),
 * AutoencoderKLFastDecode / AutoencoderKL1DFastDecode .forward (network.py:1013,846) and the diffusers
 * DDPMScheduler/PNDMScheduler .step used by sample.py:120-299.  brepgen_b200/{models,vae,schedulers}.py mirror that
 * surface and call the entry points below through ctypes (INTEGRATION.md shows the binding a maintainer adds).
 *
 * Conventions
 *   - every pointer is a DEVICE pointer owned by the caller unless stated otherwise; fp32 = float, masks = 1 byte
 *     per element (torch.bool), timesteps / labels = int64.
 *   - every call is stream-ordered on `stream` (a cudaStream_t passed as void*); no hidden device synchronisation,
 *     so the calls can be captured into CUDA graphs.
 *   - return value: 0 on success, negative BgStatus otherwise; bg_last_error() gives the message (thread-local).
 *   - no C++ exception crosses this boundary.
 */
#ifndef BREPGEN_B200_H_
#define BREPGEN_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum {
  BG_STATUS_OK = 0,
  BG_STATUS_BAD_ARG = -1,
  BG_STATUS_UNSUPPORTED_ARCH = -2,   /* not an sm_90 (H100) device */
  BG_STATUS_CUDA = -3,
  BG_STATUS_WORKSPACE = -4,          /* workspace too small */
  BG_STATUS_MISSING_WEIGHT = -5
} BgStatus;

int bg_version(void);
const char* bg_last_error(void);
/* number of CUDA kernels this library has launched so far in this process (bench.py's gpu_launches) */
uint64_t bg_launch_count(void);
/* 0 if the current device is sm_90 (H100); BG_STATUS_UNSUPPORTED_ARCH otherwise */
int bg_check_device(void);

/* ---------------------------------------------------------------------------------------------------------------
 * Denoisers.  Replaces  <Net>(use_cf).load_state_dict(...).to(device).eval()  +  <Net>.forward(...)
 *   kind 0 SurfPosNet  network.py:1066-1126      kind 1 SurfZNet   network.py:1129-1200
 *   kind 2 EdgePosNet  network.py:1203-1286      kind 3 EdgeZNet   network.py:1289-1393
 * ------------------------------------------------------------------------------------------------------------- */
typedef struct BgDenoiser BgDenoiser;

typedef struct {
  const char* name;      /* state-dict key, e.g. "net.layers.0.self_attn.in_proj_weight" */
  const float* data;     /* device fp32, contiguous */
  int64_t numel;
} BgNamedTensor;

/* Packs the checkpoint (fp16 copies of the GEMM weights, fp32 norms/biases, the 1000-row time-embedding table).
 * `sincos` may be NULL (table built on device) or a device fp32 [1000][768] copy of network.py:1043 sincos_embedding
 * for t = 0..999.  The weights may be freed after the call returns AND `stream` has been synchronised.
 * precision: 0 = plain fp16 tensor-core operands (error ~1e-3 of the fp32 reference, like the reference's own fp16
 *            autocast path); 1 (default) = the value rows of in_proj and out_proj as fp16 hi+lo pairs and a compensated
 *            fc_out tail (error ~5e-4; the q / k rows only perturb the softmax logits, 1.5e-5, and stay single);
 *            2 = all four encoder weight matrices as hi+lo pairs.  All modes accumulate in fp32 and keep
 *            the residual stream, LayerNorm, softmax statistics and the scheduler in fp32. */
int bg_denoiser_create(int kind, int use_cf, int precision, const BgNamedTensor* weights, int n_weights,
                       const float* sincos, void* stream, BgDenoiser** out);
void bg_denoiser_destroy(BgDenoiser* m);

typedef struct {
  int B, S, E;                 /* batch, faces, edges per face (E = 0 for the surface nets) */
  const float* x;              /* noisy input: surfPos (B,S,6) | surfZ (B,S,48) | edgePos (B,S,E,6) | edge (B,S,E,18) */
  const int64_t* timesteps;    /* n_timesteps entries (1, or B) */
  int n_timesteps;
  const float* surfPos;        /* (B,S,6)    kinds 1,2,3 */
  const float* surfZ;          /* (B,S,48)   kinds 2,3   */
  const float* edgePos;        /* (B,S,E,6)  kind 3      */
  const uint8_t* mask;         /* kind 1,2: (B,S) face mask; kind 3: (B,S,E) edge mask; nonzero = padded; may be NULL */
  const int64_t* class_label;  /* (B,1) when created with use_cf, else NULL */
  float* out;                  /* prediction, same shape as x, fp32 */
  int compact;                 /* != 0 and a mask is given: mask-aware token compaction -- the valid tokens of every sample
                                * are gathered before the encoder (embeds, LayerNorms and GEMMs run on sum(valid) rows,
                                * attention on ceil(valid / 128) tiles per sample) and the head scatters back; outputs of
                                * padded tokens are 0.  Result-preserving for the valid tokens: padded keys are never
                                * attended to (network.py:1268,1387-1390) and padded outputs are discarded downstream
                                * (sample.py:245,284). */
} BgDenoiserArgs;

size_t bg_denoiser_workspace_bytes(const BgDenoiser* m, int B, int S, int E);
int bg_denoiser_forward(BgDenoiser* m, const BgDenoiserArgs* args, void* workspace, size_t workspace_bytes,
                        void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * VAE decoders.  Replace AutoencoderKLFastDecode.forward (network.py:1013-1040; kind 0: z (N,3,4,4) -> (N,3,32,32)) and
 * AutoencoderKL1DFastDecode.forward (network.py:846-858; kind 1: z (N,3,4) -> (N,3,32)) for the configurations of
 * sample.py:72-97.  `weights`: the `decoder.*` and `post_quant_conv.*` entries of the checkpoint (extra keys ignored).
 * ------------------------------------------------------------------------------------------------------------- */
typedef struct BgVae BgVae;
/* kind: 0 surface decoder, 1 edge decoder, 2 surface encoder, 3 edge encoder */
int bg_vae_create(int kind, const BgNamedTensor* weights, int n_weights, void* stream, BgVae** out);
/* bg_vae_create with the number of product terms of the compensated fp16 GEMMs: 0 = the default of the kind (3; 2 for the
 * edge decoder), 3 = A_hi W_hi + A_lo W_hi + A_hi W_lo, 2 = A_hi W_hi + A_hi W_lo (a third less GEMM work, larger error) */
int bg_vae_create_ex(int kind, int terms, const BgNamedTensor* weights, int n_weights, void* stream, BgVae** out);
void bg_vae_destroy(BgVae* m);
size_t bg_vae_workspace_bytes(const BgVae* m, int N);
int bg_vae_decode(BgVae* m, const float* z, int N, float* out, void* workspace, size_t workspace_bytes, void* stream);
/* surface decoder with a latent of hw x hw (1..4) positions -> (N,3,8hw,8hw); bg_vae_decode == hw 4 */
int bg_vae_decode_hw(BgVae* m, const float* z, int N, int hw, float* out, void* workspace, size_t workspace_bytes,
                     void* stream);
/* Encoders (BASELINE config 1 round trip; SURVEY 8a row 17): kind 2 = AutoencoderKLFastEncode.forward network.py:927-945,
 * x (N,3,hw,hw), hw in {8,16,24,32} -> latent mode (N,3,hw/8,hw/8); kind 3 = AutoencoderKL1DFastEncode.forward
 * network.py:745-783, x (N,3,32) -> (N,3,4).  `weights`: `encoder.*` and `quant_conv.*`. */
int bg_vae_encode(BgVae* m, const float* x, int N, int hw, float* out, void* workspace, size_t workspace_bytes,
                  void* stream);
/* The full auto-encoders (diffusers AutoencoderKL, trainer.py:20-30, and the reference's AutoencoderKL1D, network.py:316-687):
 * the encoder's posterior, diffusers' DiagonalGaussianDistribution over moments = quant_conv(encoder(x)), P latent positions
 * per sample (hw/8 x hw/8 surface, 4 edge).
 * encode_moments: kind 2 / 3 handle, x as bg_vae_encode -> moments (N,6,P) fp32, raw, mean = channels 0-2, logvar = 3-5;
 *                 the mean half equals bg_vae_encode's output bit for bit.  Workspace: bg_vae_workspace_bytes.
 * posterior:      caller moments (N,6,P) -> z (N,3,P) = mean + exp(0.5 clamp(logvar, -30, 20)) * noise (noise (N,3,P),
 *                 NULL: z = mean) and kl (N) = 0.5 sum_{c,p} (mean^2 + var - 1 - logvar), var = exp(clamped logvar), summed
 *                 in a fixed order (deterministic).  deterministic != 0: std = var = 0, so z = mean and kl = 0.  z / kl may
 *                 be NULL.
 * reconstruct:    encoder -> posterior -> decoder -> per-sample MSE in one stream-ordered call (no host synchronisation,
 *                 graph-capturable): enc a kind 2 / 3 handle, dec the decoder of the same family (kind enc - 2), x (N,3,hw,hw)
 *                 with hw in {8,16,24,32} or (N,3,32); dec_out has the shape of x; mse (N) = mean over C*H*W of
 *                 (dec_out - x)^2.  noise, moments, z, kl, mse may be NULL (noise NULL: the decoder reads the mode).
 *                 Workspace: bg_vae_reconstruct_workspace_bytes(enc, dec, N). */
int bg_vae_encode_moments(BgVae* m, const float* x, int N, int hw, float* moments, void* workspace, size_t workspace_bytes,
                          void* stream);
int bg_vae_posterior(const float* moments, const float* noise, int N, int P, int deterministic, float* z, float* kl,
                     void* stream);
size_t bg_vae_reconstruct_workspace_bytes(const BgVae* enc, const BgVae* dec, int N);
int bg_vae_reconstruct(BgVae* enc, BgVae* dec, const float* x, int N, int hw, const float* noise, float* moments, float* z,
                       float* kl, float* dec_out, float* mse, void* workspace, size_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Scheduler updates.  Replace diffusers DDPMScheduler.step / PNDMScheduler.step as called at
 * sample.py:137,153,202,222,236,282 (arithmetic: SURVEY.md Appendix A.3/A.4).  Scalars are computed by the host-side
 * scheduler object from its alphas_cumprod table exactly as diffusers does.
 * ------------------------------------------------------------------------------------------------------------- */
/* eps = eps_cond if eps_uncond == NULL else eps_cond*(1+w) - eps_uncond*w            (CFG, sample.py:134)
 * x0  = clamp((x - sqrt_one_minus_abar*eps) / sqrt_abar, -clip, clip)  (clip <= 0: no clamp)
 * out = c_x0*x0 + c_x*x + sigma*noise
 * noise (only read when sigma != 0): the explicit tensor if not NULL; else, when sample_keys != NULL, the per-sample
 * streams below at timestep t (domain 0), over n / per_sample samples of per_sample elements; else the batch Philox
 * stream (seed, offset).  Keyed: per_sample <= 0 or n not a multiple of per_sample is BG_STATUS_BAD_ARG, as are NULL
 * pointers, sqrt_abar <= 0 and t outside 32 bits; nothing is launched then.  The keyed step is bit-identical to the step
 * fed the tensor bg_randn_keyed(..., 0, t, ...) writes. */
int bg_ddpm_step(const float* eps_cond, const float* eps_uncond, float cfg_w, const float* x, float* out,
                 const float* noise, uint64_t seed, uint64_t offset, const uint64_t* sample_keys, int64_t per_sample,
                 int64_t t, int64_t n, float sqrt_one_minus_abar, float sqrt_abar, float clip, float c_x0, float c_x,
                 float sigma, void* stream);
/* The same update in table-driven form for CUDA-graph capture of a whole denoising loop (SURVEY.md 7.2 step 4): no
 * step-specific value is a kernel argument.  coef_table[k][5] = (sqrt(1-abar_t), sqrt(abar_t), c_x0, c_x, sigma) of step k
 * (device, built once per loop from the scheduler's host tables); *step (device int32) = the current step index;
 * batch-stream counter offset0 + k * offset_stride, or, when sample_keys != NULL, the per-sample streams at the timestep
 * *t_cur (t_cur may be NULL only without keys).  Bit-identical to bg_ddpm_step with the same coefficients and noise.
 * Replaces the loop body sample.py:145-153. */
int bg_ddpm_step_tab(const float* eps_cond, const float* eps_uncond, float cfg_w, const float* x, float* out, uint64_t seed,
                     uint64_t offset0, uint64_t offset_stride, const uint64_t* sample_keys, int64_t per_sample,
                     const int64_t* t_cur, int64_t n, const float* coef_table, const int32_t* step, float clip,
                     void* stream);
/* k = ++(*step) (clamped to n_steps - 1);  *t_cur = timesteps[k].  One tiny kernel at the top of every captured step: the
 * denoiser forward reads its timestep from t_cur (device int64), bg_ddpm_step_tab reads k. */
int bg_step_advance(const int64_t* timesteps, int n_steps, int32_t* step, int64_t* t_cur, void* stream);
/* Per-sample noise streams (opt-in; without sample_keys the steps draw the batch-wide (seed, offset) stream).
 * sample_keys: device uint64 [n_samples], one Philox4x32-10 key per sample.  Element j of sample b is normal (j % 4) of the block with key
 * sample_keys[b] and counter (j / 4 as 64 bits, t, domain), Box-Muller as bg_ddpm_step; a block of 4 never straddles two
 * samples.  domain 0 = DDPM step noise at timestep t, domain 1 = initial noise (t = 0), domain 2 = known-token
 * replacement noise (bg_replace_known; t = the counter word t_ctr), domain 3 = RePaint step noise (bg_repaint_step; t = the
 * list entry k), domain 4 = RePaint undo noise (bg_repaint_undo; t = k * n_trans + i).  A sample's noise is therefore a
 * function of its key alone, whatever the batch size, its position in the batch or the rank that runs it.
 * bg_randn_keyed: NULL sample_keys, n_samples <= 0 or per_sample <= 0: BG_STATUS_BAD_ARG, nothing is launched. */
/* out[b * per_sample + j] = normal j of sample b  (n_samples * per_sample fp32) */
int bg_randn_keyed(const uint64_t* sample_keys, int64_t n_samples, int64_t per_sample, int32_t domain, int64_t t, float* out,
                   void* stream);
/* DDIM step (diffusers DDIMScheduler.step, prediction_type "epsilon"), fp32 in diffusers' order of operations:
 * eps   = eps_cond if eps_uncond == NULL else eps_cond*(1+w) - eps_uncond*w            (CFG, as bg_ddpm_step)
 * x0    = clamp((x - sqrt_one_minus_abar*eps) / sqrt_abar, -clip, clip)  (clip <= 0: no clamp)
 * e_dir = eps, or (x - sqrt_abar*x0) / sqrt_one_minus_abar if use_clipped_eps (use_clipped_model_output)
 * out   = sqrt_abar_prev*x0 + c_dir*e_dir + sigma*noise;   sigma = eta*sqrt((1-abar_prev)/(1-abar_t)*(1-abar_t/abar_prev)),
 *         c_dir = sqrt(1 - abar_prev - sigma^2), computed by the host scheduler.
 * noise (only read when sigma != 0): the explicit tensor if not NULL; else, when sample_keys != NULL, the per-sample
 * streams at timestep t (domain 0; the same normals bg_ddpm_step draws at t); else the batch Philox stream (seed, offset)
 * of bg_ddpm_step.  Keyed: per_sample <= 0 or n not a multiple of per_sample is
 * BG_STATUS_BAD_ARG, as are NULL pointers, sqrt_abar <= 0 and t outside 32 bits; nothing is launched then.
 * The inverse step (DDIM inversion, diffusers DDIMInverseScheduler.step from level t - ratio up to t) is this same call with
 * (sqrt_one_minus_abar, sqrt_abar) of level t - ratio, sqrt_abar_prev = sqrt(abar_t), c_dir = sqrt(1 - abar_t), sigma = 0
 * and use_clipped_eps = 0. */
int bg_ddim_step(const float* eps_cond, const float* eps_uncond, float cfg_w, const float* x, float* out,
                 const float* noise, uint64_t seed, uint64_t offset, const uint64_t* sample_keys, int64_t per_sample,
                 int64_t t, int64_t n, float sqrt_one_minus_abar, float sqrt_abar, float sqrt_abar_prev, float c_dir,
                 float sigma, float clip, int32_t use_clipped_eps, void* stream);
/* table-driven form for graph capture: coef_table[k][5] = (sqrt(1-abar_t), sqrt(abar_t), sqrt(abar_prev), c_dir, sigma)
 * of step k = *step (bg_step_advance), batch-stream counter offset0 + k * offset_stride, or, when sample_keys != NULL, the
 * per-sample streams at the timestep *t_cur (t_cur may be NULL only without keys).  Bit-identical to bg_ddim_step with the
 * same coefficients and noise. */
int bg_ddim_step_tab(const float* eps_cond, const float* eps_uncond, float cfg_w, const float* x, float* out, uint64_t seed,
                     uint64_t offset0, uint64_t offset_stride, const uint64_t* sample_keys, int64_t per_sample,
                     const int64_t* t_cur, int64_t n, const float* coef_table, const int32_t* step, float clip,
                     int32_t use_clipped_eps, void* stream);
/* DPM-Solver++ multistep step (diffusers DPMSolverMultistepScheduler, prediction_type "epsilon", solver_type "midpoint",
 * algorithm_type "dpmsolver++" or "sde-dpmsolver++"), fp32 with every operation rounded in diffusers' order:
 * eps = eps_cond if eps_uncond == NULL else eps_cond*(1+w) - eps_uncond*w            (CFG, as bg_ddpm_step)
 * x0  = clamp((x - sigma_s*eps) / alpha_s, -clip, clip)   (clip <= 0: no clamp; the data prediction)
 * D1  = (x0 - hist) * inv_r0;   hist = x0                  (hist holds the previous step's x0; updated in place)
 * out = c_x*x + c_0*x0 + c_1*D1 + c_z*noise
 * With h = lambda_t - lambda_s (lambda = log alpha - log sigma): ODE c_x = sigma_t/sigma_s, c_0 = -alpha_t(e^-h - 1),
 * c_1 = c_0/2 (second order) or 0 (first order), c_z = 0; SDE c_x = sigma_t/sigma_s e^-h, c_0 = alpha_t(1 - e^-2h),
 * c_1 = c_0/2 or 0, c_z = sigma_t sqrt(1 - e^-2h).  Computed by the host scheduler.  c_1 == 0 never reads hist, and
 * hist == NULL (allowed only then) skips the store.  out may alias x; hist must alias neither.  noise (only read when
 * c_z != 0): as bg_ddim_step (explicit tensor, else the per-sample streams at domain 0 and timestep t, else the batch
 * stream (seed, offset)).  BG_STATUS_BAD_ARG, launching nothing: NULL pointers, hist == NULL with c_1 != 0,
 * alpha_s <= 0, t outside 32 bits, keyed with per_sample <= 0 or n not a multiple of per_sample. */
int bg_dpm_step(const float* eps_cond, const float* eps_uncond, float cfg_w, const float* x, float* out, float* hist,
                const float* noise, uint64_t seed, uint64_t offset, const uint64_t* sample_keys, int64_t per_sample,
                int64_t t, int64_t n, float alpha_s, float sigma_s, float c_x, float c_0, float c_1, float inv_r0, float c_z,
                float clip, void* stream);
/* table-driven form for graph capture: coef_table[k][7] = (alpha_s, sigma_s, c_x, c_0, c_1, inv_r0, c_z) of step
 * k = *step (bg_step_advance), batch-stream counter offset0 + k * offset_stride, or, when sample_keys != NULL, the
 * per-sample streams at the timestep *t_cur (t_cur may be NULL only without keys).  hist must not be NULL.
 * Bit-identical to bg_dpm_step with the same coefficients and noise. */
int bg_dpm_step_tab(const float* eps_cond, const float* eps_uncond, float cfg_w, const float* x, float* out, float* hist,
                    uint64_t seed, uint64_t offset0, uint64_t offset_stride, const uint64_t* sample_keys, int64_t per_sample,
                    const int64_t* t_cur, int64_t n, const float* coef_table, const int32_t* step, float clip, void* stream);
/* UniPC multistep step (diffusers UniPCMultistepScheduler, predict_x0, prediction_type "epsilon", solver_type "bh1" or
 * "bh2"): the corrector UniC of the previous step's output and the predictor UniP of this one, fp32 with every operation
 * rounded in diffusers' order.  One row of BG_UNIPC_ROW floats, computed by the host scheduler:
 *   [0] alpha_s  [1] sigma_s  [2] corrector order c (0 = none, 1..3)  [3] predictor order p (1..3)
 *   [4] slot_new  [5..7] slots of the x0 of 1, 2, 3 steps back        (small integers stored as floats)
 *   [8..15]  corrector cc_x, cc_m0, cc_B, r_1, r_2, rho_1, rho_2, rho_t
 *   [16..22] predictor cp_x, cp_m0, cp_B, r_1, r_2, rho_1, rho_2     [23] unused
 * Per element, with eps the CFG combine of bg_dpm_step and m_i = hist[slot of i steps back] (slot s = elements s*n ..):
 *   x0  = clamp((x - sigma_s*eps) / alpha_s, -clip, clip)           (clip <= 0: no clamp)
 *   xc  = cc_x*last - cc_m0*m_1 - cc_B*(sum_{i<c} rho_i*(m_{i+1} - m_1)/r_i + rho_t*(x0 - m_1))   if c > 0, else x
 *   last = xc;  hist[slot_new] = x0
 *   out = cp_x*xc - cp_m0*x0 - cp_B*sum_{i<p} rho_i*(m_i - x0)/r_i
 * hist is a ring of n_slots slots of n elements; last and hist are read and written in place, out may alias x, and last /
 * hist alias nothing else.  last == NULL (allowed only with c = 0) skips its store.  per_sample groups the elements as
 * in the keyed steps; the step draws no noise.  BG_STATUS_BAD_ARG, launching nothing: NULL pointers, n <= 0, per_sample
 * <= 0 or not dividing n, n_slots outside 1-3, alpha_s <= 0, c outside 0-3 or p outside 1-3, c > 0 without last, a slot
 * the step uses outside [0, n_slots). */
#define BG_UNIPC_ROW 24
int bg_unipc_step(const float* eps_cond, const float* eps_uncond, float cfg_w, const float* x, float* out, float* last,
                  float* hist, int32_t n_slots, int64_t per_sample, int64_t n, const float* coef, float clip,
                  void* stream);
/* table-driven form for graph capture: the row coef_table[BG_UNIPC_ROW * k .. ] of step k = *step (bg_step_advance), as
 * written by the host scheduler's coefficient_table (rows are not validated on the device).  last must not be NULL.
 * Bit-identical to bg_unipc_step with the same row. */
int bg_unipc_step_tab(const float* eps_cond, const float* eps_uncond, float cfg_w, const float* x, float* out, float* last,
                      float* hist, int64_t per_sample, int64_t n, const float* coef_table, const int32_t* step, float clip,
                      void* stream);
/* Known-token replacement (B-rep completion; runs after the step kernel, in place on x).  x is n fp32 elements in tokens
 * of per_token consecutive elements; token_mask holds one byte per token (n / per_token).  For every element of a token
 * whose byte is non-zero:  x[i] = sqrt_abar*known[i] + sqrt_one_minus_abar*z  (fmaf(sa, known, sb*z); sa*known when
 * sb == 0, so a last step with abar_prev = 1 ends at known bit for bit).  Every other element is neither read nor written.
 * z: the explicit `noise` tensor if not NULL; else, when sample_keys != NULL, normal (j % 4) of the per-sample stream of
 * sample b = i / per_sample at counter (j / 4, t_ctr, domain 2), j = i % per_sample (bg_randn_keyed(domain 2, t_ctr));
 * else the batch key `seed`, the whole tensor counted as one sample: counter (i / 4, t_ctr, 2).  The batch form draws
 * from its own key and domain, so it neither reads nor advances the (seed, offset) stream of the step kernels.
 * t_ctr: the timestep t of the step just taken, or t_first + 1 for the replacement before a stage's first step.
 * NULL x / known / token_mask, n <= 0, per_token <= 0, n not a multiple of per_token, (keyed) per_sample not a positive
 * multiple of per_token or not dividing n, t_ctr outside 32 bits: BG_STATUS_BAD_ARG, nothing is launched. */
int bg_replace_known(float* x, const float* known, const uint8_t* token_mask, int64_t n, int64_t per_token,
                     const float* noise, uint64_t seed, const uint64_t* sample_keys, int64_t per_sample, int64_t t_ctr,
                     float sqrt_abar, float sqrt_one_minus_abar, void* stream);
/* table-driven form for graph capture: coef_table[k][2] = (sqrt(abar_prev), sqrt(1-abar_prev)) of step k = *step
 * (bg_step_advance) and t_ctr = *t_cur; no explicit noise.  Bit-identical to bg_replace_known with the same coefficients,
 * t_ctr and keys or seed.  NULL t_cur / coef_table / step are BG_STATUS_BAD_ARG too. */
int bg_replace_known_tab(float* x, const float* known, const uint8_t* token_mask, int64_t n, int64_t per_token,
                         uint64_t seed, const uint64_t* sample_keys, int64_t per_sample, const int64_t* t_cur,
                         const float* coef_table, const int32_t* step, void* stream);
/* Start of a varied stage (B-rep variations, SDEdit: diffusers' img2img add_noise on a gathered, scaled source).  out holds
 * n_tokens tokens of dim fp32 values; for every element i of output token g = i / dim:
 *   out[i] = sqrt_abar*(scale*src[index[g] * dim + i % dim]) + sqrt_one_minus_abar*z[i]
 * every product and the sum rounded on its own (__fmul_rn / __fadd_rn: the fp32 torch expression of add_noise on the
 * gathered tensor, bit for bit).  index (int32, one per output token) holds flat source-token indices into src
 * (n_src_tokens tokens of dim values); index == -1: out = z (no source, pure noise); any other index outside
 * [0, n_src_tokens): the token is NaN.  z: the explicit `noise` tensor, or, when sample_keys != NULL, normal (e % 4) of
 * the per-sample stream of sample b = g / tokens_per_sample at counter (e / 4, t, domain), e = the element's index within
 * its sample (bg_randn_keyed's normals).  Exactly one of noise and sample_keys.  BG_STATUS_BAD_ARG, launching nothing:
 * NULL src / index / out, n_src_tokens, n_tokens or dim <= 0, both or neither noise source, (keyed) tokens_per_sample not
 * a positive divisor of n_tokens, domain or t outside 32 bits. */
int bg_add_noise_gather(const float* src, int64_t n_src_tokens, const int32_t* index, int64_t n_tokens, int32_t dim,
                        float scale, float sqrt_abar, float sqrt_one_minus_abar, const float* noise,
                        const uint64_t* sample_keys, int64_t tokens_per_sample, int32_t domain, int64_t t, float* out,
                        void* stream);
/* RePaint step (diffusers RePaintScheduler.step, prediction_type "epsilon"; inpainting with resampling).  Every element
 * of a token whose token_mask byte is zero gets the bg_ddim_step update, written with its expressions (bit-identical to
 * bg_ddim_step with use_clipped_eps = 0 for the same noise):
 *   out = sqrt_abar_prev*x0 + c_dir*eps + sigma*z,   x0 = clamp((x - sqrt_one_minus_abar*eps) / sqrt_abar, -clip, clip)
 * (eps with the CFG combine of bg_ddpm_step); every element of a token whose byte is set gets the known part
 *   out = sqrt_abar_prev*known + sqrt_one_minus_abar_prev*z   (fmaf; sqrt_abar_prev*known when the second is 0)
 * with the SAME z.  Tokens are per_token consecutive elements.  known == NULL and token_mask == NULL: nothing known.
 * z (drawn only when sigma != 0 or the group of 4 holds a known element): the explicit `noise` tensor if not NULL; else,
 * when sample_keys != NULL, the per-sample streams at counter (j / 4, k, 3) (bg_randn_keyed(domain 3, k)), k = the entry's
 * index in the stage's RePaint timestep list; else the batch key `seed`, the whole tensor counted as one sample.
 * out may alias x.  BG_STATUS_BAD_ARG, launching nothing: NULL pointers, known without token_mask or the reverse,
 * n not a multiple of per_token, (keyed) per_sample not a positive multiple of per_token dividing n, sqrt_abar <= 0,
 * k outside 32 bits. */
int bg_repaint_step(const float* eps_cond, const float* eps_uncond, float cfg_w, const float* x, float* out,
                    const float* known, const uint8_t* token_mask, int64_t per_token, const float* noise, uint64_t seed,
                    const uint64_t* sample_keys, int64_t per_sample, int64_t k, int64_t n, float sqrt_one_minus_abar,
                    float sqrt_abar, float sqrt_abar_prev, float c_dir, float sigma, float sqrt_one_minus_abar_prev,
                    float clip, void* stream);
/* table-driven form for graph capture: coef_table[k][6] = (sqrt(1-abar_t), sqrt(abar_t), sqrt(abar_prev), c_dir, sigma,
 * sqrt(1-abar_prev)) and the counter word k = *step (bg_step_advance over the whole RePaint list, so step and undo entries
 * share the counter); no explicit noise.  Bit-identical to bg_repaint_step with the same coefficients, k and keys or seed. */
int bg_repaint_step_tab(const float* eps_cond, const float* eps_uncond, float cfg_w, const float* x, float* out,
                        const float* known, const uint8_t* token_mask, int64_t per_token, uint64_t seed,
                        const uint64_t* sample_keys, int64_t per_sample, int64_t n, const float* coef_table,
                        const int32_t* step, float clip, void* stream);
/* RePaint undo (diffusers RePaintScheduler.undo_step), in place: for i = 0..n_trans-1,
 *   x = coef[2i]*x + coef[2i+1]*z_i        (coef[2i], coef[2i+1] = sqrt(1-beta), sqrt(beta) of transition i, device fp32)
 * each product and the sum rounded on their own (the fp32 torch chain); x is read and written once.  z_i: the explicit
 * `noise` tensor (n_trans, n) if not NULL; else, when sample_keys != NULL, the per-sample streams at counter
 * (j / 4, k * n_trans + i, 4); else the batch key `seed`, the whole tensor counted as one sample.  BG_STATUS_BAD_ARG,
 * launching nothing: NULL x / coef, n <= 0, n_trans <= 0, (keyed) per_sample not a positive divisor of n,
 * k < 0 or (k + 1) * n_trans > 2^32. */
int bg_repaint_undo(float* x, int64_t n, int32_t n_trans, const float* coef, const float* noise, uint64_t seed,
                    const uint64_t* sample_keys, int64_t per_sample, int64_t k, void* stream);
/* table-driven form: coef = coef_table + 2 * n_trans * k and the counter word k * n_trans + i, k = *step; no explicit
 * noise.  Bit-identical to bg_repaint_undo with the same coefficients, k and keys or seed. */
int bg_repaint_undo_tab(float* x, int64_t n, int32_t n_trans, uint64_t seed, const uint64_t* sample_keys,
                        int64_t per_sample, const float* coef_table, const int32_t* step, void* stream);
/* Spherical interpolation per sample (B-rep interpolation between two DDIM-inverted noises).  a, b, out: n_samples
 * samples of per_sample fp32 values; alpha: device fp32, one per sample; token_mask: one byte per token of per_token
 * consecutive values, nonzero = masked (NULL: none masked).  Per sample, a.b, |a|^2 and |b|^2 over the unmasked tokens
 * (fp64, one CTA per sample, a fixed reduction order: no atomics, independent of the batch), then
 *   out = sin((1-alpha) theta)/sin(theta) * a + sin(alpha theta)/sin(theta) * b,   theta = acos(clamp(cos, -1, 1)),
 * or the lerp (1-alpha) a + alpha b when |cos| > 0.9995 or a norm is zero, in fp64 rounded once to fp32.  alpha == 0
 * gives a and alpha == 1 gives b bit for bit; masked tokens are copied from a.  out may alias a.  No host
 * synchronisation (graph-capturable).  BG_STATUS_BAD_ARG, launching nothing: NULL a / b / alpha / out, n_samples,
 * per_sample or per_token <= 0, n_samples >= 2^31, per_sample not a multiple of per_token. */
int bg_slerp(const float* a, const float* b, const float* alpha, const uint8_t* token_mask, int64_t n_samples,
             int64_t per_sample, int64_t per_token, float* out, void* stream);
/* out = c_sample*x - c_eps*(w0*e0 + w1*e1 + w2*e2 + w3*e3)    (PNDM transfer + Adams-Bashforth / RK combination;
 * unused e_i may be NULL with w_i = 0) */
int bg_pndm_step(const float* x, float* out, int64_t n, float c_sample, float c_eps, const float* e0, float w0,
                 const float* e1, float w1, const float* e2, float w2, const float* e3, float w3, void* stream);
/* Per-sample classifier-free combine (mixed-class batches, a guidance scale per sample):
 *   out[b*per_sample + j] = uncond_row[b] < 0 ? eps_c[b*per_sample + j]
 *                         : eps_c[...]*(1 + w[b]) - eps_u[uncond_row[b]*per_sample + j]*w[b]
 * in fp32 with 1 + w[b], both products and the difference each rounded on their own (the torch expression
 * pc*(1 + w[:, None]) - pu[uncond_row]*w[:, None], bit for bit).  uncond_row (n_samples) int32 and w (n_samples) fp32
 * live on the device, so there is no host synchronisation and the call is graph-capturable.  out may alias eps_c; then
 * samples with uncond_row[b] == -1 are neither read nor written.  An entry outside [-1, n_uncond) writes NaN for its
 * sample.  eps_u may be NULL only when n_uncond == 0.  BG_STATUS_BAD_ARG, launching nothing: any other NULL pointer,
 * n_samples or per_sample <= 0, n_uncond < 0. */
int bg_cfg_combine(const float* eps_c, const float* eps_u, const int32_t* uncond_row, const float* w, int64_t n_samples,
                   int64_t n_uncond, int64_t per_sample, float* out, void* stream);
/* out = a*x + b*y  (y may be NULL); out = eps_cond*(1+w) - eps_uncond*w is bg_axpby(eps_c, 1+w, eps_u, -w) */
int bg_axpby(const float* x, float a, const float* y, float b, float* out, int64_t n, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Stage glue on the device (replaces the D2H -> numpy loops -> H2D round trips of sample.py:159-183 and :242-261).
 * Greedy first-seen duplicate removal under max-norm < threshold, also against the corner-swapped box.
 * ------------------------------------------------------------------------------------------------------------- */
/* surfPos (B,S,6) -> out_pos (B,S,6): np.round(.,4) survivors packed first, zero padded; out_mask (B,S): 1 = padded */
int bg_dedup_surfaces(const float* surfPos, int B, int S, float threshold, float* out_pos, uint8_t* out_mask, void* stream);
/* edgePos (B,S,E,6), surf_mask (B,S) -> edge_mask (B,S,E): 1 = padded face or duplicate edge; slot 0 of a valid face = 0 */
int bg_dedup_edges(const float* edgePos, const uint8_t* surf_mask, int B, int S, int E, float threshold,
                   uint8_t* edge_mask, void* stream);
/* bg_dedup_surfaces plus out_index (B,S): the input slot of each survivor, -1 past them (positions and mask are those of
 * bg_dedup_surfaces, bit for bit).  NULL out_index is BG_STATUS_BAD_ARG. */
int bg_dedup_surfaces_index(const float* surfPos, int B, int S, float threshold, float* out_pos, uint8_t* out_mask,
                            int32_t* out_index, void* stream);
/* The trainers' pad_repeat layout (utils.py:100-106) as a gather map, one warp per output row.  src_mask: n_src_rows rows
 * of in_slots bytes, 1 = padded (as surfMask / edgeM); row_map (int32 [rows], may be NULL = identity): the source row of
 * each output row, -1 = no source.  out_index (rows, out_slots) int32: the flat source-token index
 * (src_row * in_slots + slot) each output slot takes when the n valid slots of the source row, in slot order, are
 * repeated to out_slots.  Every slot of a row without a source or without a valid slot is -1; every slot of a row with
 * more valid slots than out_slots, or whose row_map entry is outside [-1, n_src_rows), is -2 (which bg_add_noise_gather
 * poisons).  BG_STATUS_BAD_ARG, launching nothing: NULL src_mask / out_index, rows or n_src_rows <= 0, in_slots outside
 * [1, 256], out_slots <= 0, rows > n_src_rows without a row map, n_src_rows * in_slots beyond 32 bits. */
int bg_fill_index(const uint8_t* src_mask, const int32_t* row_map, int64_t rows, int64_t n_src_rows, int32_t in_slots,
                  int32_t out_slots, int32_t* out_index, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Unit-level entry points (used by tests and the bench to check/time individual kernels through the C ABI).
 * ------------------------------------------------------------------------------------------------------------- */
/* out[M,N] = act(A[M,K] (fp16) * W[N,K]^T (fp16) + bias + rowvec[row/rows_per_vec] + resid) */
int bg_op_gemm_f16(const void* A, int lda, const void* W, int ldw, int M, int N, int K, void* out, int ldo, int out_f16,
                   int relu, const float* bias, const float* resid, int ldr, const float* rowvec, int rows_per_vec,
                   int ldv, void* stream);
/* bg_op_gemm_f16 with the modes the denoisers use (test entry point; every extra argument may be 0 / NULL):
 *   a_kwrap > 0: A has a_kwrap columns and is re-read cyclically along K (column k of the product reads A column
 *                k % a_kwrap): split-weight GEMMs [W_hi | W_lo] and the compensated [x_hi | x_lo | x_hi] x [W_hi | W_hi | W_lo]
 *   n_short, k_short: output column tiles below n_short (a multiple of 256) stop after the first k_short columns of K
 *   m_dev:   device int; only rows below min(M, *m_dev) are computed and written
 *   row_map: device int [M]; row r adds rowvec[row_map[r] / rows_per_vec] instead of rowvec[r / rows_per_vec] */
int bg_op_gemm_f16_ex(const void* A, int lda, const void* W, int ldw, int M, int N, int K, void* out, int ldo, int out_f16,
                      int relu, const float* bias, const float* resid, int ldr, const float* rowvec, int rows_per_vec,
                      int ldv, int a_kwrap, int n_short, int k_short, const int* m_dev, const int* row_map, void* stream);
/* Implicit-GEMM convolution (stride 1, zero "same" padding: kw / 2 columns, (taps / kw) / 2 rows), as the VAEs run it
 * (test entry point).  x: channels-last fp16 image (N, H, W, planes * C) with a pitch of ldc elements per pixel; planes = 2
 * ([hi | lo]) with lo_plane, else 1.  w: fp16 [Cout][terms * taps * C], k = (term, tap, channel), tap = ky * kw + kx.
 * terms 1: x_hi w_0;  2: x_hi (w_0 + w_1);  3 with lo_plane: x_hi w_0 + x_lo w_1 + x_hi w_2.
 * out (fp32, pitch ldo) [N * H * W][Cout] = conv + bias (+ resid, pitch ldr; may alias out).  1-D: H = 1, kw = taps.
 * Shapes: C and Cout multiples of 64 / 128, W * H divides 128 or is a multiple of it. */
int bg_op_conv_f16(const void* x, int ldc, const void* w, int Cout, int N, int H, int W, int C, int taps, int kw,
                   int lo_plane, int terms, float* out, int ldo, const float* bias, const float* resid, int ldr,
                   void* stream);
/* qkv fp16 [B*L][2304] -> out fp16 [B*L][768]; key_mask (B,L) or NULL; use_block_list: skip fully padded key blocks
 * (needs scratch_int of B*(5*ceil(L/128)+1) ints: block list, counts and the invalid-key bit words) */
int bg_op_attention(const void* qkv, void* out, int B, int L, const uint8_t* key_mask, int use_block_list,
                    int* scratch_int, void* stream);
/* variable-length mode, as the token-compacted denoiser forwards call it: qkv [B*L][2304] and out [B*L][768] as above,
 * sample b owns rows [seq_row0[b], seq_row0[b] + seq_len[b]) of both, all of them valid (device int32 [B]);
 * L >= every seq_len[b]; rows outside every sample are not written */
int bg_op_attention_varlen(const void* qkv, void* out, int B, int L, const int* seq_row0, const int* seq_len,
                           void* stream);
int bg_op_layernorm_f16(const float* x, int ldx, const float* gamma, const float* beta, void* y, int ldy, int rows,
                        int act, void* stream);
/* bg_op_layernorm_f16 plus the split the compensated fc_out reads (test entry point): lo_offset > 0 also writes
 * fp16(value - fp16(value)) at y[row][lo_offset + c]; rows_dev (device int, may be NULL): only min(rows, *rows_dev) rows */
int bg_op_layernorm_f16_ex(const float* x, int ldx, const float* gamma, const float* beta, void* y, int ldy, int rows,
                           int act, int lo_offset, const int* rows_dev, void* stream);
int bg_op_cast_f16(const float* x, void* y, int64_t n, void* stream);
/* The denoisers' CUDA-core ends (test entry points), with token compaction's rows_dev (device int: only
 * min(rows, *rows_dev) rows) and row_map (device int [rows]), both may be NULL.
 * embed_in:     y[r] (fp16, pitch ldy) = SiLU(LayerNorm(x[row_map[r]][0:d_in] W0t + b0)) (eps 1e-5); W0t [d_in][768]
 * ln_silu_head: out[row_map[r]][0:d_out] = SiLU(LayerNorm(x[r][0:768])) W^T + bias (fp32); W [d_out][768], d_out <= 64
 * compact:      mask (B, L), nonzero = padded -> seq_len[b] valid tokens, seq_row0[b] = exclusive prefix sum,
 *               *m_valid = total, row_map[seq_row0[b] + i] = b * L + (token of the i-th valid one of sample b) */
int bg_op_embed_in(const float* x, int ldx, int d_in, const float* W0t, const float* b0, const float* gamma,
                   const float* beta, void* y, int ldy, int rows, const int* rows_dev, const int* row_map, void* stream);
int bg_op_ln_silu_head(const float* x, int ldx, const float* gamma, const float* beta, const float* W, const float* bias,
                       float* out, int d_out, int rows, const int* rows_dev, const int* row_map, void* stream);
int bg_op_compact(const uint8_t* mask, int B, int L, int* seq_len, int* seq_row0, int* m_valid, int* row_map,
                  void* stream);
/* The VAEs' CUDA-core kernels through the networks' own launch code (test entry points).  Activations are channels-last
 * fp32; "[hi | lo]" is an fp16 pair per value, hi = fp16(v), lo = fp16(v - hi), stored as the two halves of each row.
 * groupnorm:        x (N, P, C) -> act(GroupNorm(x) * gamma + beta) (+ resid, which may alias out32) into out32 (N, P, C)
 *                   and / or out16 (N, P, [C hi | C lo]); act 0 none, 1 SiLU, 2 GELU (erf); C <= 1024, C / G a power of
 *                   two up to 32 or a multiple of 32
 * vae_attention:    qkv (N*T, [q | k | v]) fp16, 512 channels in Hh heads -> out (N*T, [512 hi | 512 lo]) =
 *                   softmax(q k^T * scale) v per head; T * T * Hh <= 256
 * cubic1d:          diffusers cubic Upsample1d (up: (N, L, C) -> (N, 2L, C)) / Downsample1d ((N, L, C) -> (N, L / 2, C))
 *                   with the 8-tap kernel8 and reflect padding
 * cast_split:       x (rows, C) -> (rows, [C hi | C lo])
 * upsample2x_split: nearest 2x, x (N, H, W, C) -> (N, 2H, 2W, [C hi | C lo])
 * postquant:        1x1 convolution 3 -> 3, z (N, 3, P) -> (N, P, [3 hi | 3 lo]) = w z + b, w [3][3]
 * im2col:           in (N, H, W, C) fp16 (pitch ldin per pixel) -> A (N * H/stride * W/stride, Kpad) (pitch ldA) with
 *                   k = (ky * kw + kx) * C + c, zero for k >= kh * kw * C; stride 1: "same" zero padding, stride 2: zero
 *                   padding on the right / bottom only (diffusers Downsample2D(padding=0)) */
int bg_op_groupnorm(const float* x, int N, int P, int C, int G, float eps, const float* gamma, const float* beta, int act,
                    const float* resid, float* out32, void* out16, void* stream);
int bg_op_vae_attention(const void* qkv, void* out, int N, int T, int Hh, float scale, void* stream);
int bg_op_cubic1d(const float* x, float* y, int N, int L, int C, const float* kernel8, int up, void* stream);
int bg_op_cast_split(const float* x, void* y, int64_t rows, int C, void* stream);
int bg_op_upsample2x_split(const float* x, void* y, int N, int H, int W, int C, void* stream);
int bg_op_postquant(const float* z, const float* w, const float* b, void* y, int N, int P, void* stream);
int bg_op_im2col(const void* in, int ldin, void* A, int ldA, int N, int H, int W, int C, int kh, int kw, int stride,
                 int Kpad, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Post-decode geometry glue (SURVEY.md 8(f) row 3): the numeric cores of the per-CAD post-processing between the VAE
 * decoders and OpenCASCADE.  The list / set bookkeeping around them stays on the host (brepgen_b200/postprocess.py, same
 * function names and return values as utils.py); construct_brep (utils.py:819) is out of scope.  All pointers are device
 * pointers; fp32 / int32.
 * ------------------------------------------------------------------------------------------------------------- */
/* sample.py:316-329 (+ utils.py:48-59): out[e][0|1][3] = edge_ncs[e][0|31] * (bsize / 2) + bcenter of the edge box
 * edge_pos[e][6] * pos_scale (bsize = largest extent) */
int bg_edge_endpoints(const float* edge_ncs, const float* edge_pos, float pos_scale, int64_t n_edges, float* out, void* stream);
/* nn[i] = index of the nearest point of ANOTHER group inside the same segment [seg_off[s], seg_off[s+1]) (lowest index on
 * ties, -1 if none): utils.py:403-421 (edge2loop: group = edge, segment = face) and :505-524 (group = face, segment = CAD) */
int bg_nn_exclude(const float* pts, const int32_t* group, const int32_t* seg_off, int n_seg, int32_t* nn, void* stream);
/* out[i][j] = |pts_i - pts_j| < threshold (n x n): utils.py:556-561 */
int bg_pairs_within(const float* pts, int n, float threshold, uint8_t* out, void* stream);
/* out[i][j] = i != j && set(adj_i) == set(adj_j) && mean|z_i - z_j| < threshold (n x n): utils.py:607-619 */
int bg_edge_pair_match(const int32_t* edge_vertex_adj, const float* z, int z_dim, int n, float threshold, uint8_t* out,
                       void* stream);
/* utils.py:692-728: fit every decoded edge curve edge_ncs[e][32][3] to its two vertices vertex_se[e][2][3] */
int bg_edge_fit(const float* edge_ncs, const float* vertex_se, int n_edges, float* edge_wcs, void* stream);
/* utils.py:732-752: initial surface grids surf_wcs[f][32*32][3]; face f owns the edges adj[adj_off[f] .. adj_off[f+1]) */
int bg_surf_init(const float* surf_ncs, const float* surf_pos, const float* edge_wcs, const int32_t* adj_off, const int32_t* adj,
                 int n_faces, float* surf_wcs, void* stream);
/* utils.py:756-770: `iters` AdamW steps on one translation per face minimising the wire -> surface Chamfer distance, all
 * faces and all iterations in ONE launch; inv_nface[f] = 1 / (number of faces of f's CAD) (the loss is a mean over the CAD's
 * faces).  surf_out = surf_init + the offset before the last step (what the reference returns); offset_out may be NULL. */
int bg_surf_offset_opt(const float* surf_init, const float* edge_wcs, const int32_t* adj_off, const int32_t* adj,
                       const float* inv_nface, int n_faces, int max_edges_per_face, int iters, float lr, float beta1, float beta2,
                       float eps, float weight_decay, float* surf_out, float* offset_out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* BREPGEN_B200_H_ */
