#include "host_util.h"

#include <cstdarg>
#include <mutex>
#include <utility>
#include <vector>

namespace stb {

std::string& last_error_string() {
  static thread_local std::string s;
  return s;
}

int set_error(int code, const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  last_error_string() = buf;
  return code;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    // resolved through the runtime so that libcuda.so is not a link-time dependency of the library
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

int make_tmap_bf16_3d(CUtensorMap* out, const void* base, uint64_t d0, uint64_t d1, uint64_t d2, uint64_t stride1,
                      uint64_t stride2, uint32_t b0, uint32_t b1, uint32_t b2) {
  EncodeTiledFn fn = get_encode_fn();
  STB_CHECK(fn != nullptr, STB_ERR_CUDA, "cuTensorMapEncodeTiled not available from the driver");
  STB_CHECK((reinterpret_cast<uintptr_t>(base) & 127) == 0, STB_ERR_INVALID, "TMA base %p not 128B aligned", base);
  STB_CHECK(stride1 % 16 == 0 && stride2 % 16 == 0, STB_ERR_INVALID, "TMA strides must be multiples of 16 bytes");
  cuuint64_t dims[3] = {d0, d1, d2};
  cuuint64_t strides[2] = {stride1, stride2};
  cuuint32_t box[3] = {b0, b1, b2};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  STB_CHECK(r == CUDA_SUCCESS, STB_ERR_CUDA,
            "cuTensorMapEncodeTiled failed (%d): dims=(%llu,%llu,%llu) strides=(%llu,%llu) box=(%u,%u,%u)", (int)r,
            (unsigned long long)d0, (unsigned long long)d1, (unsigned long long)d2, (unsigned long long)stride1,
            (unsigned long long)stride2, b0, b1, b2);
  return STB_OK;
}

int make_tmap_f32_2d(CUtensorMap* out, const void* base, uint64_t cols, uint64_t rows, uint32_t box_cols,
                     uint32_t box_rows) {
  EncodeTiledFn fn = get_encode_fn();
  STB_CHECK(fn != nullptr, STB_ERR_CUDA, "cuTensorMapEncodeTiled not available from the driver");
  STB_CHECK((reinterpret_cast<uintptr_t>(base) & 127) == 0, STB_ERR_INVALID, "TMA base %p not 128B aligned", base);
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {cols * 4};
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  STB_CHECK(r == CUDA_SUCCESS, STB_ERR_CUDA, "cuTensorMapEncodeTiled(f32 2d) failed (%d): %llux%llu box %ux%u", (int)r,
            (unsigned long long)rows, (unsigned long long)cols, box_rows, box_cols);
  return STB_OK;
}

int make_tmap_f16_2d(CUtensorMap* out, const void* base, uint64_t cols, uint64_t rows, uint32_t box_cols,
                     uint32_t box_rows) {
  EncodeTiledFn fn = get_encode_fn();
  STB_CHECK(fn != nullptr, STB_ERR_CUDA, "cuTensorMapEncodeTiled not available from the driver");
  STB_CHECK((reinterpret_cast<uintptr_t>(base) & 127) == 0, STB_ERR_INVALID, "TMA base %p not 128B aligned", base);
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {cols * 2};
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  STB_CHECK(r == CUDA_SUCCESS, STB_ERR_CUDA, "cuTensorMapEncodeTiled(f16 2d) failed (%d): %llux%llu box %ux%u", (int)r,
            (unsigned long long)rows, (unsigned long long)cols, box_rows, box_cols);
  return STB_OK;
}

int ensure_dynamic_smem(const void* func, int bytes) {
  static std::mutex mu;
  static std::vector<std::pair<const void*, int>> done;  // (kernel, device)
  int dev = 0;
  STB_CUDA_CHECK(cudaGetDevice(&dev));
  std::lock_guard<std::mutex> lock(mu);
  for (const auto& d : done)
    if (d.first == func && d.second == dev) return STB_OK;
  STB_CUDA_CHECK(cudaFuncSetAttribute(func, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
  done.emplace_back(func, dev);
  return STB_OK;
}

int num_sms() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 132;
  }
  return n;
}

}  // namespace stb
