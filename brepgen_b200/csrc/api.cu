// C ABI: version / error / device check and the unit-level entry points declared in include/brepgen_b200.h.
#include "../../include/brepgen_b200.h"
#include "bg_internal.h"

namespace bg {
const char* last_error_cstr();
}
using namespace bg;

extern "C" {

int bg_version(void) { return 100; }   // 0.1.0

const char* bg_last_error(void) { return last_error_cstr(); }

uint64_t bg_launch_count(void) { return launch_count(); }

int bg_check_device(void) {
  int dev = 0, major = 0, minor = 0;
  BG_CUDA(cudaGetDevice(&dev));
  BG_CUDA(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev));
  BG_CUDA(cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev));
  if (major != 9 || minor != 0)
    return set_error(BG_ERR_UNSUPPORTED_ARCH, "brepgen_b200 kernels are built for sm_90a (H100) only; device is sm_" +
                                                  std::to_string(major) + std::to_string(minor));
  return BG_OK;
}

int bg_op_gemm_f16(const void* A, int lda, const void* W, int ldw, int M, int N, int K, void* out, int ldo, int out_f16,
                   int relu, const float* bias, const float* resid, int ldr, const float* rowvec, int rows_per_vec,
                   int ldv, void* stream) {
  BG_TRY(bg_check_device());
  GemmEpilogue ep;
  ep.out = out; ep.ldo = ldo; ep.out_f16 = out_f16; ep.relu = relu; ep.bias = bias;
  ep.resid = resid; ep.ldr = ldr; ep.rowvec = rowvec; ep.rows_per_vec = rows_per_vec; ep.ldv = ldv;
  return launch_gemm_f16(reinterpret_cast<cudaStream_t>(stream), reinterpret_cast<const __half*>(A), lda,
                         reinterpret_cast<const __half*>(W), ldw, M, N, K, ep);
}

int bg_op_gemm_f16_ex(const void* A, int lda, const void* W, int ldw, int M, int N, int K, void* out, int ldo, int out_f16,
                      int relu, const float* bias, const float* resid, int ldr, const float* rowvec, int rows_per_vec,
                      int ldv, int a_kwrap, int n_short, int k_short, const int* m_dev, const int* row_map, void* stream) {
  BG_TRY(bg_check_device());
  GemmEpilogue ep;
  ep.out = out; ep.ldo = ldo; ep.out_f16 = out_f16; ep.relu = relu; ep.bias = bias;
  ep.resid = resid; ep.ldr = ldr; ep.rowvec = rowvec; ep.rows_per_vec = rows_per_vec; ep.ldv = ldv;
  ep.a_kwrap = a_kwrap; ep.n_short = n_short; ep.k_short = k_short; ep.m_dev = m_dev; ep.row_map = row_map;
  return launch_gemm_f16(reinterpret_cast<cudaStream_t>(stream), reinterpret_cast<const __half*>(A), lda,
                         reinterpret_cast<const __half*>(W), ldw, M, N, K, ep);
}

int bg_op_conv_f16(const void* x, int ldc, const void* w, int Cout, int N, int H, int W, int C, int taps, int kw,
                   int lo_plane, int terms, float* out, int ldo, const float* bias, const float* resid, int ldr,
                   void* stream) {
  BG_TRY(bg_check_device());
  BG_REQUIRE(terms >= 1 && terms <= 3, "conv: terms must be 1, 2 or 3");
  ConvGeom g;
  g.taps = taps; g.kw = kw; g.C = C; g.W = W; g.H = H; g.N = N; g.lo_plane = lo_plane; g.terms = terms;
  GemmEpilogue ep;
  ep.out = out; ep.ldo = ldo; ep.out_f16 = 0; ep.bias = bias; ep.resid = resid; ep.ldr = ldr;
  ep.conv = g;
  const int K = terms * taps * C;
  return launch_gemm_f16(reinterpret_cast<cudaStream_t>(stream), reinterpret_cast<const __half*>(x), ldc,
                         reinterpret_cast<const __half*>(w), K, N * H * W, Cout, K, ep);
}

int bg_op_attention(const void* qkv, void* out, int B, int L, const uint8_t* key_mask, int use_block_list,
                    int* scratch_int, void* stream) {
  BG_TRY(bg_check_device());
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  AttnArgs a;
  a.qkv = reinterpret_cast<const __half*>(qkv);
  a.out = reinterpret_cast<__half*>(out);
  a.ldo = 768; a.B = B; a.L = L; a.key_mask = key_mask;
  // checked before the block list is built, so that a rejected call launches nothing
  BG_REQUIRE(L <= ATTN_MAX_L, "attention: sequence longer than 8192 tokens is not supported");
  if (use_block_list && key_mask) {
    BG_REQUIRE(scratch_int != nullptr, "attention: block list needs scratch_int");
    const int nkb = (L + 127) / 128;
    a.blk_list = scratch_int;
    a.blk_count = scratch_int + (size_t)B * nkb;
    uint32_t* words = reinterpret_cast<uint32_t*>(scratch_int + (size_t)B * (nkb + 1));
    a.blk_words = words;
    BG_TRY(launch_build_block_list(st, key_mask, B, L, scratch_int, scratch_int + (size_t)B * nkb, words));
  }
  return launch_attention(st, a);
}

int bg_op_attention_varlen(const void* qkv, void* out, int B, int L, const int* seq_row0, const int* seq_len,
                           void* stream) {
  BG_TRY(bg_check_device());
  BG_REQUIRE(seq_row0 && seq_len, "attention: variable-length mode needs seq_row0 and seq_len");
  AttnArgs a;
  a.qkv = reinterpret_cast<const __half*>(qkv);
  a.out = reinterpret_cast<__half*>(out);
  a.ldo = 768; a.B = B; a.L = L;
  a.seq_row0 = seq_row0; a.seq_len = seq_len;
  return launch_attention(reinterpret_cast<cudaStream_t>(stream), a);
}

int bg_op_layernorm_f16(const float* x, int ldx, const float* gamma, const float* beta, void* y, int ldy, int rows,
                        int act, void* stream) {
  return launch_layernorm_f16(reinterpret_cast<cudaStream_t>(stream), x, ldx, gamma, beta, reinterpret_cast<__half*>(y),
                              ldy, rows, act);
}

int bg_op_layernorm_f16_ex(const float* x, int ldx, const float* gamma, const float* beta, void* y, int ldy, int rows,
                           int act, int lo_offset, const int* rows_dev, void* stream) {
  return launch_layernorm_f16(reinterpret_cast<cudaStream_t>(stream), x, ldx, gamma, beta, reinterpret_cast<__half*>(y),
                              ldy, rows, act, lo_offset, rows_dev);
}

int bg_op_cast_f16(const float* x, void* y, int64_t n, void* stream) {
  return launch_cast_f32_to_f16(reinterpret_cast<cudaStream_t>(stream), x, reinterpret_cast<__half*>(y), (size_t)n);
}

int bg_op_embed_in(const float* x, int ldx, int d_in, const float* W0t, const float* b0, const float* gamma,
                   const float* beta, void* y, int ldy, int rows, const int* rows_dev, const int* row_map, void* stream) {
  BG_TRY(bg_check_device());
  return launch_embed_in(reinterpret_cast<cudaStream_t>(stream), x, ldx, d_in, W0t, b0, gamma, beta,
                         reinterpret_cast<__half*>(y), ldy, rows, rows_dev, row_map);
}

int bg_op_ln_silu_head(const float* x, int ldx, const float* gamma, const float* beta, const float* W, const float* bias,
                       float* out, int d_out, int rows, const int* rows_dev, const int* row_map, void* stream) {
  BG_TRY(bg_check_device());
  return launch_ln_silu_head(reinterpret_cast<cudaStream_t>(stream), x, ldx, gamma, beta, W, bias, out, d_out, rows,
                             rows_dev, row_map);
}

int bg_op_compact(const uint8_t* mask, int B, int L, int* seq_len, int* seq_row0, int* m_valid, int* row_map,
                  void* stream) {
  BG_TRY(bg_check_device());
  return launch_compact(reinterpret_cast<cudaStream_t>(stream), mask, B, L, seq_len, seq_row0, m_valid, row_map);
}

}  // extern "C"
