// Error plumbing, device queries and TMA descriptor creation shared by all translation units.
#include <map>
#include <mutex>
#include <utility>

#include "bg_internal.h"

namespace bg {

static thread_local std::string g_last_error;

int set_error(int code, const std::string& msg) {
  g_last_error = msg;
  return code;
}
const char* last_error_cstr() { return g_last_error.c_str(); }

int check_cuda(cudaError_t e, const char* what) {
  if (e == cudaSuccess) return BG_OK;
  return set_error(BG_ERR_CUDA, std::string(what) + ": " + cudaGetErrorName(e) + " (" + cudaGetErrorString(e) + ")");
}

static unsigned long long g_launches = 0;   // kernels launched by this library (host-side counter, single host thread)
int check_launch(const char* what) {
  ++g_launches;
  return check_cuda(cudaGetLastError(), what);
}
unsigned long long launch_count() { return g_launches; }

// Per-DEVICE caches: one process may drive several GPUs (models.py / vae.py switch devices with torch.cuda.device), and both
// the SM count and cudaFuncAttributeMaxDynamicSharedMemorySize are per device / context.
static constexpr int MAX_DEV = 64;

int num_sms() {
  static int cached[MAX_DEV] = {0};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= MAX_DEV) return 132;
  if (cached[dev] == 0) {
    int n = 0;
    cached[dev] = (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && n > 0) ? n : 132;
  }
  return cached[dev];
}

int ensure_dynamic_smem(const void* func, int bytes) {
  static std::mutex mu;
  static std::map<std::pair<const void*, int>, int> done;   // (kernel, device) -> configured bytes
  int dev = 0;
  BG_CUDA(cudaGetDevice(&dev));
  std::lock_guard<std::mutex> lock(mu);
  auto it = done.find({func, dev});
  if (it != done.end() && it->second >= bytes) return BG_OK;
  BG_CUDA(cudaFuncSetAttribute(func, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
  done[{func, dev}] = bytes;
  return BG_OK;
}

int align_workspace(void* ws, size_t bytes, size_t need, const char* what, char** base) {
  *base = reinterpret_cast<char*>((reinterpret_cast<uintptr_t>(ws) + 1023) & ~uintptr_t(1023));
  if (need + (size_t)(*base - reinterpret_cast<char*>(ws)) > bytes)
    return set_error(BG_ERR_WORKSPACE, std::string(what) + ": workspace too small");
  return BG_OK;
}

Packer::Packer(const BgNamedTensor* weights, int n, void* stream) : st(reinterpret_cast<cudaStream_t>(stream)) {
  for (int i = 0; i < n; ++i) by_name[weights[i].name] = &weights[i];
}

const float* Packer::find(const std::string& name, int64_t numel) {
  auto it = by_name.find(name);
  if (it == by_name.end()) {
    if (!err) err = set_error(BG_ERR_MISSING_WEIGHT, "missing weight: " + name);
    return nullptr;
  }
  if (it->second->numel != numel) {
    if (!err) err = set_error(BG_ERR_BAD_ARG, "weight " + name + " has " + std::to_string(it->second->numel) +
                                                  " elements, expected " + std::to_string(numel));
    return nullptr;
  }
  return it->second->data;
}

float* Packer::copy_f32(const std::string& name, int64_t numel) {
  const float* src = find(name, numel);
  float* dst = take<float>(numel);
  if (!dry && src && !err)
    err = check_cuda(cudaMemcpyAsync(dst, src, numel * sizeof(float), cudaMemcpyDeviceToDevice, st), "copy weight");
  return dst;
}

float* Packer::zeros(int64_t numel) {
  float* dst = take<float>(numel);
  if (!dry && !err) err = check_cuda(cudaMemsetAsync(dst, 0, numel * sizeof(float), st), "memset");
  return dst;
}

int pack_arena(Packer& pk, const std::function<int()>& pack, char** arena, size_t* arena_bytes) {
  pk.dry = true;
  pk.off = 0;
  int s = pack();
  if (s == 0) {
    *arena_bytes = pk.off;
    s = check_cuda(cudaMalloc(reinterpret_cast<void**>(arena), *arena_bytes), "cudaMalloc(weights)");
  }
  if (s == 0) {
    pk.dry = false;
    pk.base = *arena;
    pk.off = 0;
    s = pack();
  }
  if (s != 0 && *arena) {
    cudaFree(*arena);
    *arena = nullptr;
  }
  return s;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

static int encode(CUtensorMap* out, const void* base, uint32_t rank, const cuuint64_t* dims, const cuuint64_t* strides,
                  const cuuint32_t* box, CUtensorMapDataType dtype = CU_TENSOR_MAP_DATA_TYPE_FLOAT16) {
  EncodeTiledFn fn = encode_fn();
  if (!fn) return set_error(BG_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available (no CUDA driver?)");
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = fn(out, dtype, rank, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return set_error(BG_ERR_CUDA, "cuTensorMapEncodeTiled failed with CUresult " + std::to_string((int)r));
  return BG_OK;
}

int make_tmap_2d_f16(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows,
                     uint32_t box_cols) {
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {ld * 2};
  cuuint32_t box[2] = {box_cols, box_rows};
  return encode(out, base, 2, dims, strides, box);
}

int make_tmap_4d_f16(CUtensorMap* out, const void* base, uint64_t C, uint64_t W, uint64_t H, uint64_t N, uint64_t ldc,
                     uint32_t box_w, uint32_t box_h, uint32_t box_n) {
  cuuint64_t dims[4] = {C, W, H, N};
  cuuint64_t strides[3] = {ldc * 2, W * ldc * 2, H * W * ldc * 2};
  cuuint32_t box[4] = {64, box_w, box_h, box_n};
  return encode(out, base, 4, dims, strides, box);
}

int make_tmap_2d_f32(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows,
                     uint32_t box_cols) {
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {ld * 4};
  cuuint32_t box[2] = {box_cols, box_rows};
  return encode(out, base, 2, dims, strides, box, CU_TENSOR_MAP_DATA_TYPE_FLOAT32);
}

}  // namespace bg
