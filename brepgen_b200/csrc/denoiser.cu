// Denoiser handle: packs a reference checkpoint once, then runs a whole forward (embed -> 12 pre-norm encoder layers ->
// final LayerNorm -> fc_out) as a fixed sequence of stream-ordered kernels.
//
// Mirrors network.py: SurfPosNet.forward :1107-1126, SurfZNet.forward :1176-1200,
// EdgePosNet.forward :1257-1286, EdgeZNet.forward :1357-1393; encoder = nn.TransformerEncoder(12 x
// TransformerEncoderLayer(d=768, nhead=12, ff=1024, norm_first=True), LayerNorm) built at :1076-1078 etc.
//
// Work the reference recomputes every step and we do not: the time-embedding MLP depends only on t -> a 1000 x 768
// table built at create(); the several per-token embed MLPs of one net are fused into ONE GEMM by concatenating their
// hidden activations along K (sum of products == product of concatenation).
#include <string>

#include "../../include/brepgen_b200.h"
#include "bg_internal.h"

namespace bg {

namespace {

constexpr int D = 768, FF = 1024, NLAYER = 12, NCLASS = 11, NT_TABLE = 1000;

struct EmbedDef {
  const char* name;
  int d_in;
  int level;   // 0 = per token of the sequence, 1 = per face (edge nets only)
  int src;     // 0 x, 1 surfPos, 2 surfZ, 3 edgePos, 4 x[..., :12], 5 x[..., 12:]
};

struct KindDef {
  int n_embed;
  EmbedDef e[5];
  int d_out;
  int x_width;
};

const KindDef KINDS[4] = {
    {1, {{"p_embed", 6, 0, 0}}, 6, 6},
    {2, {{"z_embed", 48, 0, 0}, {"p_embed", 6, 0, 1}}, 48, 48},
    {3, {{"surfz_embed", 48, 1, 2}, {"surfp_embed", 6, 1, 1}, {"edgep_embed", 6, 0, 0}}, 6, 6},
    {5, {{"surfz_embed", 48, 1, 2}, {"surfp_embed", 6, 1, 1}, {"edgep_embed", 6, 0, 3}, {"edgez_embed", 12, 0, 4},
         {"vertp_fc", 6, 0, 5}}, 18, 18},
};

struct LayerW {
  // [N][k*] fp16; k* = K (single) or 2K ([W_hi | W_lo], split-weight GEMM).  in_proj is ONE operand [2304][kqkv]: at
  // precision 1 only the v rows (>= qk_rows) carry a lo half (their rounding error is 4.8e-4 of the output; the q|k rows only
  // perturb the softmax logits: 1.5e-5) and the GEMM stops at K = 768 for the q|k column tiles (GemmEpilogue::n_short)
  __half *wqkv, *wo, *w1, *w2;
  int kqkv, qk_short, ko, k1, k2;
  float *bqkv, *bo, *b1, *b2, *ln1g, *ln1b, *ln2g, *ln2b;
};

struct EmbedW {
  float *w0t, *b0, *lng, *lnb;
};

__global__ void transpose_kernel(const float* __restrict__ w, float* __restrict__ wt, int rows, int cols) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;   // over rows*cols of the output [cols][rows]
  if (i < rows * cols) {
    const int c = i / rows, r = i % rows;
    wt[i] = w[(size_t)r * cols + c];
  }
}
// wcat[n, col0 + k] = fp16(w[n, k]);  w: [768][768]
__global__ void pack_cat_kernel(const float* __restrict__ w, __half* __restrict__ wcat, int ldcat, int col0) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < D * D) {
    const int n = i / D, k = i % D;
    wcat[(size_t)n * ldcat + col0 + k] = __float2half_rn(w[i]);
  }
}
// dst[n, col0 + k] = hi or lo part of w[n, k]:  hi = fp16(w), lo = fp16(w - float(hi))  (lo is ~2^-11 |w|; fp16
// subnormals keep it to ~1 % which is all the compensation needs)
__global__ void pack_split_kernel(const float* __restrict__ w, __half* __restrict__ dst, int N, int K, int ld, int col0,
                                  int part) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < (size_t)N * K) {
    const int n = (int)(i / K), k = (int)(i % K);
    const float v = w[i];
    const __half hi = __float2half_rn(v);
    dst[(size_t)n * ld + col0 + k] = part == 0 ? hi : __float2half_rn(v - __half2float(hi));
  }
}
__global__ void add_vec_kernel(float* __restrict__ acc, const float* __restrict__ v, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) acc[i] += v[i];
}
// fp32 row-by-row MLP used once at create():  out[t] = W3 silu(LN(W0 in[t] + b0)) + b3   (768 -> 768 -> 768)
__global__ void __launch_bounds__(256) mlp_table_kernel(const float* __restrict__ in, const float* __restrict__ w0,
                                                        const float* __restrict__ b0, const float* __restrict__ g,
                                                        const float* __restrict__ b, const float* __restrict__ w3,
                                                        const float* __restrict__ b3, float* __restrict__ out) {
  __shared__ float sx[D];
  __shared__ float sh[D];
  __shared__ float red[2];
  const int t = blockIdx.x;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int i = threadIdx.x; i < D; i += blockDim.x) sx[i] = in[(size_t)t * D + i];
  __syncthreads();
  for (int o = warp; o < D; o += 8) {
    float acc = 0.f;
    for (int k = lane; k < D; k += 32) acc = fmaf(sx[k], w0[(size_t)o * D + k], acc);
    for (int s = 16; s > 0; s >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, s);
    if (lane == 0) sh[o] = acc + b0[o];
  }
  __syncthreads();
  if (warp == 0) {
    float s = 0.f;
    for (int k = lane; k < D; k += 32) s += sh[k];
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const float mean = s / D;
    float q = 0.f;
    for (int k = lane; k < D; k += 32) q += (sh[k] - mean) * (sh[k] - mean);
    for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
    if (lane == 0) { red[0] = mean; red[1] = rsqrtf(q / D + 1e-5f); }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < D; i += blockDim.x) {
    const float y = (sh[i] - red[0]) * red[1] * g[i] + b[i];
    sx[i] = y / (1.f + expf(-y));
  }
  __syncthreads();
  for (int o = warp; o < D; o += 8) {
    float acc = 0.f;
    for (int k = lane; k < D; k += 32) acc = fmaf(sx[k], w3[(size_t)o * D + k], acc);
    for (int s = 16; s > 0; s >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, s);
    if (lane == 0) out[(size_t)t * D + o] = acc + b3[o];
  }
}

}  // namespace

}  // namespace bg

using namespace bg;

struct BgDenoiser {
  int kind = 0, use_cf = 0;
  int precision = 1;           // 0: plain fp16 operands; 1: + split V / out-proj weights + compensated fc_out; 2: all split
  char* arena = nullptr;       // one device allocation holding every packed tensor
  size_t arena_bytes = 0;
  LayerW layer[NLAYER];
  float *normg = nullptr, *normb = nullptr;
  EmbedW embed[5];
  __half* wcat_tok = nullptr;   // [768][n_tok*768]  second Linear of the per-token embeds, concatenated along K
  float* bcat_tok = nullptr;    // [768] summed biases
  int n_tok = 0;
  __half* wcat_face = nullptr;  // same for the per-face embeds (edge nets)
  float* bcat_face = nullptr;
  int n_face = 0;
  __half* fc0w = nullptr;       // fc_out.0
  float *fc0b = nullptr, *fclng = nullptr, *fclnb = nullptr, *fc3w = nullptr, *fc3b = nullptr;
  float* time_table = nullptr;  // [1000][768]
  float* class_table = nullptr; // [11][768]
};

namespace {

struct DPacker : Packer {
  using Packer::Packer;
  __half* cast_f16(const std::string& name, int64_t numel) {
    const float* src = find(name, numel);
    __half* dst = take<__half>(numel);
    if (!dry && src && !err) err = launch_cast_f32_to_f16(st, src, dst, (size_t)numel);
    return dst;
  }
  // [N][K] fp32 -> fp16 [N][K] (split == 0) or [N][2K] = [W_hi | W_lo]; returns the packed K through *k_out
  __half* pack_weight(const std::string& name, int N, int K, bool split, int* k_out) {
    const float* src = find(name, (int64_t)N * K);
    const int kp = split ? 2 * K : K;
    *k_out = kp;
    __half* dst = take<__half>((size_t)N * kp);
    if (!dry && src && !err) {
      const unsigned blocks = (unsigned)(((size_t)N * K + 255) / 256);
      pack_split_kernel<<<blocks, 256, 0, st>>>(src, dst, N, K, kp, 0, 0);
      if (split) pack_split_kernel<<<blocks, 256, 0, st>>>(src, dst, N, K, kp, K, 1);
      err = check_launch("pack_split_kernel");
    }
    return dst;
  }
};

int pack(BgDenoiser* m, DPacker& pk, const float* sincos) {
  const KindDef& kd = KINDS[m->kind];
  for (int i = 0; i < NLAYER; ++i) {
    const std::string p = "net.layers." + std::to_string(i) + ".";
    LayerW& L = m->layer[i];
    const bool s_attn = m->precision >= 1, s_ff = m->precision >= 2;
    if (s_attn && !s_ff) {      // precision 1: [q|k rows: W_hi, unused] / [v rows: W_hi | W_lo]
      const float* src = pk.find(p + "self_attn.in_proj_weight", (int64_t)3 * D * D);
      L.kqkv = 2 * D;
      L.qk_short = 1;
      L.wqkv = pk.take<__half>((size_t)3 * D * 2 * D);
      if (!pk.dry && src && !pk.err) {
        pk.err = check_cuda(cudaMemsetAsync(L.wqkv, 0, (size_t)3 * D * 2 * D * sizeof(__half), pk.st), "memset");
        const unsigned bqk = (unsigned)(((size_t)2 * D * D + 255) / 256), bv = (unsigned)(((size_t)D * D + 255) / 256);
        pack_split_kernel<<<bqk, 256, 0, pk.st>>>(src, L.wqkv, 2 * D, D, 2 * D, 0, 0);
        pack_split_kernel<<<bv, 256, 0, pk.st>>>(src + (size_t)2 * D * D, L.wqkv + (size_t)2 * D * 2 * D, D, D, 2 * D, 0, 0);
        pack_split_kernel<<<bv, 256, 0, pk.st>>>(src + (size_t)2 * D * D, L.wqkv + (size_t)2 * D * 2 * D, D, D, 2 * D, D, 1);
        if (!pk.err) pk.err = check_launch("pack in_proj");
      }
    } else {
      L.qk_short = 0;
      L.wqkv = pk.pack_weight(p + "self_attn.in_proj_weight", 3 * D, D, s_ff, &L.kqkv);
    }
    L.bqkv = pk.copy_f32(p + "self_attn.in_proj_bias", 3 * D);
    L.wo = pk.pack_weight(p + "self_attn.out_proj.weight", D, D, s_attn, &L.ko);
    L.bo = pk.copy_f32(p + "self_attn.out_proj.bias", D);
    L.w1 = pk.pack_weight(p + "linear1.weight", FF, D, s_ff, &L.k1);
    L.b1 = pk.copy_f32(p + "linear1.bias", FF);
    L.w2 = pk.pack_weight(p + "linear2.weight", D, FF, s_ff, &L.k2);
    L.b2 = pk.copy_f32(p + "linear2.bias", D);
    L.ln1g = pk.copy_f32(p + "norm1.weight", D);
    L.ln1b = pk.copy_f32(p + "norm1.bias", D);
    L.ln2g = pk.copy_f32(p + "norm2.weight", D);
    L.ln2b = pk.copy_f32(p + "norm2.bias", D);
  }
  m->normg = pk.copy_f32("net.norm.weight", D);
  m->normb = pk.copy_f32("net.norm.bias", D);

  m->n_tok = m->n_face = 0;
  for (int i = 0; i < kd.n_embed; ++i) (kd.e[i].level == 0 ? m->n_tok : m->n_face)++;
  m->wcat_tok = pk.take<__half>((size_t)D * m->n_tok * D);
  m->bcat_tok = pk.take<float>(D);
  if (m->n_face) {
    m->wcat_face = pk.take<__half>((size_t)D * m->n_face * D);
    m->bcat_face = pk.take<float>(D);
  }
  if (!pk.dry && !pk.err) {
    pk.err = check_cuda(cudaMemsetAsync(m->bcat_tok, 0, D * sizeof(float), pk.st), "memset");
    if (m->n_face && !pk.err) pk.err = check_cuda(cudaMemsetAsync(m->bcat_face, 0, D * sizeof(float), pk.st), "memset");
  }
  int i_tok = 0, i_face = 0;
  for (int i = 0; i < kd.n_embed; ++i) {
    const EmbedDef& e = kd.e[i];
    const std::string p = std::string(e.name) + ".";
    EmbedW& W = m->embed[i];
    const float* w0 = pk.find(p + "0.weight", (int64_t)D * e.d_in);
    W.w0t = pk.take<float>((size_t)D * e.d_in);
    W.b0 = pk.copy_f32(p + "0.bias", D);
    W.lng = pk.copy_f32(p + "1.weight", D);
    W.lnb = pk.copy_f32(p + "1.bias", D);
    const float* w3 = pk.find(p + "3.weight", (int64_t)D * D);
    const float* b3 = pk.find(p + "3.bias", D);
    if (!pk.dry && !pk.err) {
      const int n = D * e.d_in;
      transpose_kernel<<<(n + 255) / 256, 256, 0, pk.st>>>(w0, W.w0t, D, e.d_in);
      const bool tok = e.level == 0;
      const int slot = tok ? i_tok : i_face;
      pack_cat_kernel<<<(D * D + 255) / 256, 256, 0, pk.st>>>(w3, tok ? m->wcat_tok : m->wcat_face,
                                                               (tok ? m->n_tok : m->n_face) * D, slot * D);
      add_vec_kernel<<<(D + 255) / 256, 256, 0, pk.st>>>(tok ? m->bcat_tok : m->bcat_face, b3, D);
      pk.err = check_launch("pack embed");
    }
    (e.level == 0 ? i_tok : i_face)++;
  }
  if (m->precision >= 1) {
    // compensated product: [x_hi | x_lo | x_hi] * [W_hi | W_hi | W_lo]^T  (drops only the lo*lo term, ~2^-22)
    const float* src = pk.find("fc_out.0.weight", 1LL * D * D);
    m->fc0w = pk.take<__half>((size_t)D * 3 * D);
    if (!pk.dry && src && !pk.err) {
      const unsigned blocks = (D * D + 255) / 256;
      pack_split_kernel<<<blocks, 256, 0, pk.st>>>(src, m->fc0w, D, D, 3 * D, 0, 0);
      pack_split_kernel<<<blocks, 256, 0, pk.st>>>(src, m->fc0w, D, D, 3 * D, D, 0);
      pack_split_kernel<<<blocks, 256, 0, pk.st>>>(src, m->fc0w, D, D, 3 * D, 2 * D, 1);
      pk.err = check_launch("pack fc_out.0");
    }
  } else {
    m->fc0w = pk.cast_f16("fc_out.0.weight", 1LL * D * D);
  }
  m->fc0b = pk.copy_f32("fc_out.0.bias", D);
  m->fclng = pk.copy_f32("fc_out.1.weight", D);
  m->fclnb = pk.copy_f32("fc_out.1.bias", D);
  m->fc3w = pk.copy_f32("fc_out.3.weight", (int64_t)kd.d_out * D);
  m->fc3b = pk.copy_f32("fc_out.3.bias", kd.d_out);

  m->time_table = pk.take<float>((size_t)NT_TABLE * D);
  float* sincos_buf = pk.take<float>((size_t)NT_TABLE * D);
  const float* tw0 = pk.find("time_embed.0.weight", 1LL * D * D);
  const float* tb0 = pk.find("time_embed.0.bias", D);
  const float* tg = pk.find("time_embed.1.weight", D);
  const float* tb = pk.find("time_embed.1.bias", D);
  const float* tw3 = pk.find("time_embed.3.weight", 1LL * D * D);
  const float* tb3 = pk.find("time_embed.3.bias", D);
  if (!pk.dry && !pk.err) {
    const float* sc = sincos;
    if (!sc) {
      pk.err = launch_sincos_table(pk.st, sincos_buf, NT_TABLE);
      sc = sincos_buf;
    }
    if (!pk.err) {
      mlp_table_kernel<<<NT_TABLE, 256, 0, pk.st>>>(sc, tw0, tb0, tg, tb, tw3, tb3, m->time_table);
      pk.err = check_launch("time table");
    }
  }
  if (m->use_cf) m->class_table = pk.copy_f32("class_embed.embed.weight", (int64_t)NCLASS * D);
  return pk.err;
}

struct Workspace {
  float *X, *cond, *condface;
  __half *Xn, *QKV, *AO, *Hff, *Hface;
  uint8_t* mask;
  int *blk_list, *blk_count;
  uint32_t* blk_words;
  int *row_map, *seq_len, *seq_row0, *m_valid;   // token compaction
  size_t bytes;
};

Workspace carve(char* base, int kind, int B, int S, int E) {
  const size_t L = (kind >= 2) ? (size_t)S * E : (size_t)S;
  const size_t M = (size_t)B * L;
  const size_t nkb = (L + 127) / 128;
  size_t off = 0;
  auto take = [&](size_t bytes) {
    char* p = base ? base + off : nullptr;
    off += align_up(bytes, 1024);
    return p;
  };
  Workspace w;
  w.X = reinterpret_cast<float*>(take(M * D * 4));
  w.Xn = reinterpret_cast<__half*>(take(M * D * 2));
  w.QKV = reinterpret_cast<__half*>(take(M * 3 * D * 2));
  w.AO = reinterpret_cast<__half*>(take(M * D * 2));
  w.Hff = reinterpret_cast<__half*>(take(M * FF * 2));
  w.cond = reinterpret_cast<float*>(take((size_t)B * D * 4));
  w.condface = reinterpret_cast<float*>(take(kind >= 2 ? (size_t)B * S * D * 4 : 0));
  w.Hface = reinterpret_cast<__half*>(take(kind >= 2 ? (size_t)B * S * 2 * D * 2 : 0));
  w.mask = reinterpret_cast<uint8_t*>(take(M));
  w.blk_list = reinterpret_cast<int*>(take((size_t)B * nkb * 4));
  w.blk_count = reinterpret_cast<int*>(take((size_t)B * 4));
  w.blk_words = reinterpret_cast<uint32_t*>(take((size_t)B * nkb * 16));
  w.row_map = reinterpret_cast<int*>(take(M * 4));
  w.seq_len = reinterpret_cast<int*>(take((size_t)B * 4));
  w.seq_row0 = reinterpret_cast<int*>(take((size_t)B * 4));
  w.m_valid = reinterpret_cast<int*>(take(4));
  w.bytes = off;
  return w;
}

}  // namespace

extern "C" {

int bg_denoiser_create(int kind, int use_cf, int precision, const BgNamedTensor* weights, int n_weights,
                       const float* sincos, void* stream, BgDenoiser** out) {
  BG_REQUIRE(kind >= 0 && kind < 4 && weights && n_weights > 0 && out, "denoiser_create: bad arguments");
  BG_REQUIRE(precision >= 0 && precision <= 2, "denoiser_create: precision must be 0, 1 or 2");
  BG_TRY(bg_check_device());
  BgDenoiser* m = new BgDenoiser();
  m->kind = kind;
  m->use_cf = use_cf ? 1 : 0;
  m->precision = precision;
  DPacker pk(weights, n_weights, stream);
  const int s = pack_arena(pk, [&] { return pack(m, pk, sincos); }, &m->arena, &m->arena_bytes);
  if (s != 0) {
    bg_denoiser_destroy(m);
    return s;
  }
  *out = m;
  return BG_OK;
}

void bg_denoiser_destroy(BgDenoiser* m) {
  if (!m) return;
  if (m->arena) cudaFree(m->arena);
  delete m;
}

size_t bg_denoiser_workspace_bytes(const BgDenoiser* m, int B, int S, int E) {
  if (!m || B <= 0 || S <= 0 || (m->kind >= 2 && E <= 0)) return 0;
  return carve(nullptr, m->kind, B, S, E).bytes + 1024;
}

int bg_denoiser_forward(BgDenoiser* m, const BgDenoiserArgs* a, void* workspace, size_t workspace_bytes, void* stream) {
  BG_REQUIRE(m && a && workspace, "denoiser_forward: null argument");
  const int kind = m->kind;
  const KindDef& kd = KINDS[kind];
  const bool edge = kind >= 2;
  BG_REQUIRE(a->B > 0 && a->S > 0 && (!edge || a->E > 0), "denoiser_forward: bad shape");
  BG_REQUIRE(a->x && a->out && a->timesteps, "denoiser_forward: x / out / timesteps missing");
  BG_REQUIRE(kind < 1 || a->surfPos, "denoiser_forward: surfPos missing");
  BG_REQUIRE(kind < 2 || a->surfZ, "denoiser_forward: surfZ missing");
  BG_REQUIRE(kind < 3 || a->edgePos, "denoiser_forward: edgePos missing");
  BG_REQUIRE(!m->use_cf || a->class_label, "denoiser_forward: class_label missing for a use_cf model");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int B = a->B, S = a->S, E = edge ? a->E : 1;
  const int L = S * E, M = B * L, BS = B * S;

  char* base;
  BG_TRY(align_workspace(workspace, workspace_bytes, carve(nullptr, kind, B, S, E).bytes, "denoiser_forward", &base));
  const Workspace w = carve(base, kind, B, S, E);

  // 1. conditioning vector per sample: time table row (+ class embedding)
  BG_TRY(launch_cond(st, m->time_table, a->timesteps, a->n_timesteps, m->use_cf ? m->class_table : nullptr,
                     a->class_label, w.cond, B));

  // key-padding mask (face mask repeated over edges for EdgePosNet, network.py:1268); with compaction the valid tokens are
  // gathered: everything below runs on *m_valid rows (device-side count, no host synchronisation)
  const uint8_t* kmask = nullptr;
  if (kind >= 1 && a->mask) {
    if (kind == 2) {
      BG_TRY(launch_mask_expand(st, a->mask, w.mask, BS, E));
      kmask = w.mask;
    } else {
      kmask = a->mask;
    }
  }
  const bool compact = a->compact != 0 && kmask != nullptr;
  const int* m_dev = nullptr;
  const int* row_map = nullptr;
  if (compact) {
    BG_TRY(launch_compact(st, kmask, B, L, w.seq_len, w.seq_row0, w.m_valid, w.row_map));
    m_dev = w.m_valid;
    row_map = w.row_map;
  }

  // 2. embeddings -> X
  const float* srcs[6] = {a->x, a->surfPos, a->surfZ, a->edgePos, a->x, a->x ? a->x + 12 : nullptr};
  const int src_ld[6] = {kd.x_width, 6, 48, 6, 18, 18};
  int i_tok = 0, i_face = 0;
  __half* Htok = w.QKV;   // [M][n_tok*768] aliases the (not yet used) QKV buffer
  for (int i = 0; i < kd.n_embed; ++i) {
    const EmbedDef& e = kd.e[i];
    const EmbedW& W = m->embed[i];
    if (e.level == 1) {
      BG_TRY(launch_embed_in(st, srcs[e.src], src_ld[e.src], e.d_in, W.w0t, W.b0, W.lng, W.lnb, w.Hface + i_face * D,
                             m->n_face * D, BS));
      ++i_face;
    } else {
      BG_TRY(launch_embed_in(st, srcs[e.src], src_ld[e.src], e.d_in, W.w0t, W.b0, W.lng, W.lnb, Htok + i_tok * D,
                             m->n_tok * D, M, m_dev, row_map));
      ++i_tok;
    }
  }
  const float* tokvec = w.cond;
  int tok_rpv = L;
  if (edge) {
    GemmEpilogue ep;
    ep.out = w.condface; ep.ldo = D; ep.out_f16 = 0; ep.bias = m->bcat_face;
    ep.rowvec = w.cond; ep.rows_per_vec = S; ep.ldv = D;
    BG_TRY(launch_gemm_f16(st, w.Hface, m->n_face * D, m->wcat_face, m->n_face * D, BS, D, m->n_face * D, ep));
    tokvec = w.condface;
    tok_rpv = E;
  }
  {
    GemmEpilogue ep;
    ep.out = w.X; ep.ldo = D; ep.out_f16 = 0; ep.bias = m->bcat_tok;
    ep.rowvec = tokvec; ep.rows_per_vec = tok_rpv; ep.ldv = D;
    ep.m_dev = m_dev; ep.row_map = row_map;       // compaction: row r carries source token row_map[r]
    BG_TRY(launch_gemm_f16(st, Htok, m->n_tok * D, m->wcat_tok, m->n_tok * D, M, D, m->n_tok * D, ep));
  }

  // 3. valid key-block list (dense layout only: after compaction every key of a sample's rows is valid)
  if (kmask && !compact) BG_TRY(launch_build_block_list(st, kmask, B, L, w.blk_list, w.blk_count, w.blk_words));
  // compaction: the last sample's final key tile reads up to 127 rows past the last valid token; the QKV GEMMs never write
  // them, so clear them once (the embed stage above used this buffer as scratch)
  if (compact) BG_TRY(launch_zero_rows_f16(st, w.QKV, 3 * D, 3 * D, w.m_valid, 128, M));

  // 4. encoder
  for (int i = 0; i < NLAYER; ++i) {
    const LayerW& Lw = m->layer[i];
    BG_TRY(launch_layernorm_f16(st, w.X, D, Lw.ln1g, Lw.ln1b, w.Xn, D, M, 0, 0, m_dev));
    {
      GemmEpilogue ep;
      ep.m_dev = m_dev;
      ep.out = w.QKV; ep.ldo = 3 * D; ep.out_f16 = 1; ep.bias = Lw.bqkv;
      // one GEMM for q | k | v (Xn is read once): at precision 1 the q|k column tiles stop after the hi half of K
      ep.a_kwrap = Lw.kqkv > D ? D : 0;
      if (Lw.qk_short) { ep.n_short = 2 * D; ep.k_short = D; }
      BG_TRY(launch_gemm_f16(st, w.Xn, D, Lw.wqkv, Lw.kqkv, M, 3 * D, Lw.kqkv, ep));
    }
    {
      AttnArgs at;
      at.qkv = w.QKV; at.out = w.AO; at.ldo = D; at.B = B; at.L = L;
      if (compact) {
        at.seq_row0 = w.seq_row0; at.seq_len = w.seq_len;
      } else {
        at.key_mask = kmask;
        at.blk_list = kmask ? w.blk_list : nullptr;
        at.blk_count = kmask ? w.blk_count : nullptr;
        at.blk_words = kmask ? w.blk_words : nullptr;
      }
      BG_TRY(launch_attention(st, at));
    }
    {
      GemmEpilogue ep;
      ep.m_dev = m_dev;
      ep.out = w.X; ep.ldo = D; ep.out_f16 = 0; ep.bias = Lw.bo; ep.resid = w.X; ep.ldr = D;
      ep.a_kwrap = Lw.ko > D ? D : 0;
      BG_TRY(launch_gemm_f16(st, w.AO, D, Lw.wo, Lw.ko, M, D, Lw.ko, ep));
    }
    BG_TRY(launch_layernorm_f16(st, w.X, D, Lw.ln2g, Lw.ln2b, w.Xn, D, M, 0, 0, m_dev));
    {
      GemmEpilogue ep;
      ep.m_dev = m_dev;
      ep.out = w.Hff; ep.ldo = FF; ep.out_f16 = 1; ep.relu = 1; ep.bias = Lw.b1;
      ep.a_kwrap = Lw.k1 > D ? D : 0;
      BG_TRY(launch_gemm_f16(st, w.Xn, D, Lw.w1, Lw.k1, M, FF, Lw.k1, ep));
    }
    {
      GemmEpilogue ep;
      ep.m_dev = m_dev;
      ep.out = w.X; ep.ldo = D; ep.out_f16 = 0; ep.bias = Lw.b2; ep.resid = w.X; ep.ldr = D;
      ep.a_kwrap = Lw.k2 > FF ? FF : 0;
      BG_TRY(launch_gemm_f16(st, w.Hff, FF, Lw.w2, Lw.k2, M, D, Lw.k2, ep));
    }
  }

  // 5. final norm + fc_out (Linear -> LN -> SiLU -> Linear(768, d_out)); this tail feeds the output directly, so at
  //    precision >= 1 it runs as a compensated fp16 product (hi/lo activations x hi/lo weights) and an fp32 head.
  {
    GemmEpilogue ep;
    ep.m_dev = m_dev;
    ep.out = w.X; ep.ldo = D; ep.out_f16 = 0; ep.bias = m->fc0b;
    if (m->precision >= 1) {
      __half* A3 = w.QKV;   // [M][2304] scratch: cols 0..767 hi, 768..1535 lo (the third K block wraps back to hi)
      BG_TRY(launch_layernorm_f16(st, w.X, D, m->normg, m->normb, A3, 3 * D, M, 0, D, m_dev));
      ep.a_kwrap = 2 * D;
      BG_TRY(launch_gemm_f16(st, A3, 3 * D, m->fc0w, 3 * D, M, D, 3 * D, ep));
    } else {
      BG_TRY(launch_layernorm_f16(st, w.X, D, m->normg, m->normb, w.Xn, D, M, 0, 0, m_dev));
      BG_TRY(launch_gemm_f16(st, w.Xn, D, m->fc0w, D, M, D, D, ep));
    }
  }
  if (compact) BG_CUDA(cudaMemsetAsync(a->out, 0, (size_t)M * kd.d_out * sizeof(float), st));   // padded tokens: 0
  BG_TRY(launch_ln_silu_head(st, w.X, D, m->fclng, m->fclnb, m->fc3w, m->fc3b, a->out, kd.d_out, M, m_dev, row_map));
  return BG_OK;
}

}  // extern "C"
