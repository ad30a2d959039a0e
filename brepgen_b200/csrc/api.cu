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

int bg_op_attention(const void* qkv, void* out, int B, int L, const uint8_t* key_mask, int use_block_list,
                    int* scratch_int, void* stream) {
  BG_TRY(bg_check_device());
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  AttnArgs a;
  a.qkv = reinterpret_cast<const __half*>(qkv);
  a.out = reinterpret_cast<__half*>(out);
  a.ldo = 768; a.B = B; a.L = L; a.key_mask = key_mask;
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

int bg_op_layernorm_f16(const float* x, int ldx, const float* gamma, const float* beta, void* y, int ldy, int rows,
                        int act, void* stream) {
  return launch_layernorm_f16(reinterpret_cast<cudaStream_t>(stream), x, ldx, gamma, beta, reinterpret_cast<__half*>(y),
                              ldy, rows, act);
}

int bg_op_cast_f16(const float* x, void* y, int64_t n, void* stream) {
  return launch_cast_f32_to_f16(reinterpret_cast<cudaStream_t>(stream), x, reinterpret_cast<__half*>(y), (size_t)n);
}

}  // extern "C"
