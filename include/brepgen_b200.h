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

/* ---------------------------------------------------------------------------------------------------------------
 * Scheduler updates.  Replace diffusers DDPMScheduler.step / PNDMScheduler.step as called at
 * sample.py:137,153,202,222,236,282 (arithmetic: SURVEY.md Appendix A.3/A.4).  Scalars are computed by the host-side
 * scheduler object from its alphas_cumprod table exactly as diffusers does.
 * ------------------------------------------------------------------------------------------------------------- */
/* eps = eps_cond if eps_uncond == NULL else eps_cond*(1+w) - eps_uncond*w            (CFG, sample.py:134)
 * x0  = clamp((x - sqrt_one_minus_abar*eps) / sqrt_abar, -clip, clip)  (clip <= 0: no clamp)
 * out = c_x0*x0 + c_x*x + sigma*noise;   noise: explicit tensor, or Philox N(0,1) from (seed, offset) if NULL & sigma>0 */
int bg_ddpm_step(const float* eps_cond, const float* eps_uncond, float cfg_w, const float* x, float* out,
                 const float* noise, uint64_t seed, uint64_t offset, int64_t n, float sqrt_one_minus_abar,
                 float sqrt_abar, float clip, float c_x0, float c_x, float sigma, void* stream);
/* The same update in table-driven form for CUDA-graph capture of a whole denoising loop (SURVEY.md 7.2 step 4): no
 * step-specific value is a kernel argument.  coef_table[k][5] = (sqrt(1-abar_t), sqrt(abar_t), c_x0, c_x, sigma) of step k
 * (device, built once per loop from the scheduler's host tables); *step (device int32) = the current step index;
 * in-kernel Philox noise with counter offset0 + k * offset_stride.  Replaces the loop body sample.py:145-153. */
int bg_ddpm_step_tab(const float* eps_cond, const float* eps_uncond, float cfg_w, const float* x, float* out, uint64_t seed,
                     uint64_t offset0, uint64_t offset_stride, int64_t n, const float* coef_table, const int32_t* step,
                     float clip, void* stream);
/* k = ++(*step) (clamped to n_steps - 1);  *t_cur = timesteps[k].  One tiny kernel at the top of every captured step: the
 * denoiser forward reads its timestep from t_cur (device int64), bg_ddpm_step_tab reads k. */
int bg_step_advance(const int64_t* timesteps, int n_steps, int32_t* step, int64_t* t_cur, void* stream);
/* out = c_sample*x - c_eps*(w0*e0 + w1*e1 + w2*e2 + w3*e3)    (PNDM transfer + Adams-Bashforth / RK combination;
 * unused e_i may be NULL with w_i = 0) */
int bg_pndm_step(const float* x, float* out, int64_t n, float c_sample, float c_eps, const float* e0, float w0,
                 const float* e1, float w1, const float* e2, float w2, const float* e3, float w3, void* stream);
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

/* ---------------------------------------------------------------------------------------------------------------
 * Unit-level entry points (used by tests and the bench to check/time individual kernels through the C ABI).
 * ------------------------------------------------------------------------------------------------------------- */
/* out[M,N] = act(A[M,K] (fp16) * W[N,K]^T (fp16) + bias + rowvec[row/rows_per_vec] + resid) */
int bg_op_gemm_f16(const void* A, int lda, const void* W, int ldw, int M, int N, int K, void* out, int ldo, int out_f16,
                   int relu, const float* bias, const float* resid, int ldr, const float* rowvec, int rows_per_vec,
                   int ldv, void* stream);
/* qkv fp16 [B*L][2304] -> out fp16 [B*L][768]; key_mask (B,L) or NULL; use_block_list: skip fully padded key blocks
 * (needs scratch_int of B*(5*ceil(L/128)+1) ints: block list, counts and the invalid-key bit words) */
int bg_op_attention(const void* qkv, void* out, int B, int L, const uint8_t* key_mask, int use_block_list,
                    int* scratch_int, void* stream);
int bg_op_layernorm_f16(const float* x, int ldx, const float* gamma, const float* beta, void* y, int ldy, int rows,
                        int act, void* stream);
int bg_op_cast_f16(const float* x, void* y, int64_t n, void* stream);

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
