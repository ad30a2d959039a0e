// Internal (C++) interface between the translation units of libbrepgen_b200.so. Not part of the C ABI.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include <functional>
#include <map>
#include <string>

#include "../../include/brepgen_b200.h"

namespace bg {

// ---- error plumbing (no C++ exception crosses the C ABI) ----
enum Status : int {
  BG_OK = 0,
  BG_ERR_BAD_ARG = -1,
  BG_ERR_UNSUPPORTED_ARCH = -2,
  BG_ERR_CUDA = -3,
  BG_ERR_WORKSPACE = -4,
  BG_ERR_MISSING_WEIGHT = -5,
};
int set_error(int code, const std::string& msg);
int check_cuda(cudaError_t e, const char* what);
int check_launch(const char* what);          // cudaGetLastError() after a kernel launch; counts the launch
unsigned long long launch_count();
#define BG_CUDA(x)                                              \
  do {                                                          \
    int _s = ::bg::check_cuda((x), #x);                         \
    if (_s != 0) return _s;                                     \
  } while (0)
#define BG_TRY(x)                    \
  do {                               \
    int _s = (x);                    \
    if (_s != 0) return _s;          \
  } while (0)
#define BG_REQUIRE(cond, msg)                                                           \
  do {                                                                                  \
    if (!(cond)) return ::bg::set_error(::bg::BG_ERR_BAD_ARG, std::string(msg) + " [" #cond "]"); \
  } while (0)

int num_sms();   // of the current device (cached per device)
// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) once per (kernel, device)
int ensure_dynamic_smem(const void* func, int bytes);

inline size_t align_up(size_t x, size_t a = 256) { return (x + a - 1) / a * a; }

// Start of the caller's workspace rounded up to 1 KB (the bg_*_workspace_bytes sizes include that slack) in *base;
// BG_ERR_WORKSPACE when `need` bytes from there do not fit in `bytes`.
int align_workspace(void* ws, size_t bytes, size_t need, const char* what, char** base);

// ---- weight packing: named fp32 device tensors in, one device arena out ----
// A pack function runs twice over the same Packer: a dry pass (take() returns null, nothing is read) that only sizes the
// arena, then a pass that fills it.  The first error is kept in `err` (and bg_last_error).
struct Packer {
  std::map<std::string, const BgNamedTensor*> by_name;
  char* base = nullptr;
  size_t off = 0;
  bool dry = true;
  cudaStream_t st = nullptr;
  int err = 0;

  Packer(const BgNamedTensor* weights, int n, void* stream);
  const float* find(const std::string& name, int64_t numel);   // null (and err set) when missing or of the wrong size
  template <class T>
  T* take(size_t n) {
    T* p = dry ? nullptr : reinterpret_cast<T*>(base + off);
    off += align_up(n * sizeof(T));
    return p;
  }
  float* copy_f32(const std::string& name, int64_t numel);
  float* zeros(int64_t numel);
};
// pass 1 (size), cudaMalloc of *arena, pass 2 (fill); on error the arena is freed and *arena is null
int pack_arena(Packer& pk, const std::function<int()>& pack, char** arena, size_t* arena_bytes);

// ---- TMA descriptor creation (driver entry point resolved at run time; no link dependency on libcuda) ----
// 2-D fp16 row-major [rows][cols] with row pitch ld (elements); box = {box_cols(=64), box_rows}; SWIZZLE_128B.
int make_tmap_2d_f16(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows,
                     uint32_t box_cols = 64);
// 2-D fp32 row-major [rows][cols], row pitch ld (elements); box = {box_cols (<= 32: 128-byte swizzle span), box_rows}
int make_tmap_2d_f32(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows,
                     uint32_t box_cols);

// 4-D fp16 channels-last activation [n][h][w][c] (c contiguous, pitch ldc elements per pixel); box = {64 channels, box_w,
// box_h, box_n}; SWIZZLE_128B; out-of-range coordinates (the zero padding of a convolution) are filled with zeros
int make_tmap_4d_f16(CUtensorMap* out, const void* base, uint64_t C, uint64_t W, uint64_t H, uint64_t N, uint64_t ldc,
                     uint32_t box_w, uint32_t box_h, uint32_t box_n);

// Implicit-GEMM convolution (stride 1, "same" zero padding) over a channels-last activation [n][H][W][planes * C] fp16:
// row m of the GEMM is output pixel m (n, y, x order), its K axis runs over (term, tap, channel): the A tile of k-block
// (term, tap, 64-channel chunk) is the TMA box {64 channels, W, box_h, box_n} of the input shifted by the tap's offset, so
// the im2col matrix exists only as shared-memory tiles (VAE decoders: network.py:1013-1040, 846-858).
struct ConvGeom {
  int taps = 0;            // 0: plain GEMM.  kh * kw
  int kw = 1;              // taps per kernel row (1-D convolutions: kw = taps, H = 1)
  int C = 0;               // channels per plane (multiple of 64)
  int W = 0, H = 1, N = 0; // image extents and number of images;  W * H divides 128 or is a multiple of 128
  int lo_plane = 0;        // 1: A is [hi | lo] (pitch 2C) and the middle term of a 3-term product reads the lo plane
  int terms = 1;           // K = terms * taps * C: [A_hi W_hi (+ A_lo W_hi) + A_hi W_lo]
};

// ---- wgmma GEMM:  out[M,N] = epilogue( A[M,K] (fp16, pitch lda) * W[N,K]^T (fp16, pitch ldw) ) ----
struct GemmEpilogue {
  void* out = nullptr;           // fp16 or fp32, pitch ldo (elements)
  int ldo = 0;
  int out_f16 = 1;
  int relu = 0;
  const float* bias = nullptr;   // [N]
  const float* resid = nullptr;  // fp32 [M, ldr] added (may alias out when out is fp32)
  int ldr = 0;
  const float* rowvec = nullptr; // fp32 [(M / rows_per_vec), ldv]: row r adds rowvec[r / rows_per_vec]
  int rows_per_vec = 1;
  int ldv = 0;
  int a_kwrap = 0;               // >0: A has a_kwrap columns and is reused cyclically along K (split-weight GEMM)
  int n_short = 0, k_short = 0;  // column tiles below n_short (a multiple of 256) use only the first k_short columns of K
  const int* m_dev = nullptr;    // optional device int: only min(M, *m_dev) rows are computed (token compaction)
  const int* row_map = nullptr;  // optional: rowvec is indexed with row_map[row] / rows_per_vec instead of row / rows_per_vec
  ConvGeom conv;                 // conv.taps > 0: A is a channels-last image and the GEMM is an implicit convolution
};
int launch_gemm_f16(cudaStream_t st, const __half* A, int lda, const __half* W, int ldw, int M, int N, int K,
                    const GemmEpilogue& ep);

// ---- wgmma flash attention over packed QKV [B*L, 2304] fp16 (q | k | v, head h at +64h) ----
struct AttnArgs {
  const __half* qkv = nullptr;      // [B*L, 3*768]
  __half* out = nullptr;            // [B*L, ldo] head h at column 64h
  int ldo = 768;
  int B = 0, L = 0;
  const uint8_t* key_mask = nullptr;   // [B, L] nonzero = padded key (ignored), or null
  const int* blk_list = nullptr;       // [B, nkb] key blocks (of 128) with >=1 valid key, or null = all
  const int* blk_count = nullptr;      // [B]
  const uint32_t* blk_words = nullptr; // [B, nkb, 4] invalid-key bit words in LIST order (launch_build_block_list), or null
  // variable-length mode (token compaction): sample b owns rows [seq_row0[b], seq_row0[b] + seq_len[b]) of qkv / out, all of
  // them valid; L = the maximum length (grid size); key_mask / blk_* must be null
  const int* seq_row0 = nullptr;
  const int* seq_len = nullptr;
};
constexpr int ATTN_MAX_L = 8192;   // longest sequence launch_attention takes (64 key blocks of mask words in shared memory)
int launch_attention(cudaStream_t st, const AttnArgs& a);
// builds blk_list/blk_count from key_mask ([B,L]); nkb = ceil(L/128)
int launch_build_block_list(cudaStream_t st, const uint8_t* key_mask, int B, int L, int* blk_list, int* blk_count,
                            uint32_t* blk_words = nullptr);

// ---- CUDA-core kernels (HBM-bound glue) ----
// y[row, 0:768] (fp16, pitch ldy) = act(LayerNorm(x[row, 0:768]) * g + b); act: 0 none, 1 SiLU.   eps = 1e-5
// lo_offset > 0: additionally writes the fp16 rounding residual (value - fp16(value)) at y[row, lo_offset + c]
// rows_dev (optional): device int, the kernel processes min(rows, *rows_dev) rows (token compaction)
int launch_layernorm_f16(cudaStream_t st, const float* x, int ldx, const float* g, const float* b, __half* y, int ldy,
                         int rows, int act, int lo_offset = 0, const int* rows_dev = nullptr);
// y (fp16, pitch ldy) = SiLU(LayerNorm(x[row,0:d_in] * W0^T + b0)); W0t is [d_in][768] fp32 (transposed Linear weight)
// row_map (optional): output row r reads input row row_map[r] (gather of the valid tokens)
int launch_embed_in(cudaStream_t st, const float* x, int ldx, int d_in, const float* W0t, const float* b0, const float* g,
                    const float* b, __half* y, int ldy, int rows, const int* rows_dev = nullptr, const int* row_map = nullptr);
// out[row, 0:d_out] (fp32) = SiLU(LayerNorm(x[row, 0:768])) * W^T + bias, all fp32;  W [d_out][768], d_out <= 64
// row_map (optional): input row r is written to output row row_map[r] (scatter back to the padded layout)
int launch_ln_silu_head(cudaStream_t st, const float* x, int ldx, const float* g, const float* b, const float* W,
                        const float* bias, float* out, int d_out, int rows, const int* rows_dev = nullptr,
                        const int* row_map = nullptr);
// valid-token compaction of a [B, L] key-padding mask: seq_len[b], seq_row0[b] (exclusive prefix), *m_valid (total) and
// row_map[compact row] = b * L + token
int launch_zero_rows_f16(cudaStream_t st, __half* y, int ld, int cols, const int* row0_dev, int nrows, int max_rows);
int launch_compact(cudaStream_t st, const uint8_t* mask, int B, int L, int* seq_len, int* seq_row0, int* m_valid, int* row_map);
// cond[b, :] = time_table[t_b, :] + (class_table ? class_table[label_b, :] : 0);  t: int64 [n_t] (n_t = 1 or B)
int launch_cond(cudaStream_t st, const float* time_table, const int64_t* t, int n_t, const float* class_table,
                const int64_t* label, float* cond, int B);
// sincos rows for t = 0..n-1:  out[t, :] = [cos(t f) | sin(t f)], f_i = exp(-ln(1e4) i / 384)   (fp32, 768 wide)
int launch_sincos_table(cudaStream_t st, float* out, int n);
int launch_cast_f32_to_f16(cudaStream_t st, const float* x, __half* y, size_t n);
int launch_mask_expand(cudaStream_t st, const uint8_t* face_mask, uint8_t* edge_mask, int BS, int E);

}  // namespace bg
