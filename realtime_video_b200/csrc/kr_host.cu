// kr_host.cu — host-side utilities: error string, device query, TMA descriptor encode.
#include "kr_common.cuh"
#include "kr_ops.h"

#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <mutex>

namespace kr {

static thread_local char g_last_error[512] = "";

void set_last_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_last_error, sizeof(g_last_error), fmt, ap);
  va_end(ap);
}
const char* last_error() { return g_last_error; }

int sm_count() {
  static int cached = 0;
  if (cached == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 132;
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0)
      return 132;
    cached = n;
  }
  return cached;
}

// cuTensorMapEncodeTiled is a driver API; resolve it at run time so the library
// neither links libcuda nor needs it to be present when only loaded for symbol checks.
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, []() {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres);
    if (e == cudaSuccess && qres == cudaDriverEntryPointSuccess) fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

int make_tmap_nd(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                 const uint64_t* strides_bytes, const uint32_t* box, bool is_bf16, int swizzle_bytes) {
  EncodeTiledFn fn = get_encode_fn();
  if (fn == nullptr) {
    set_last_error("cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)");
    return KR_ERR_NO_DEVICE;
  }
  if (rank < 1 || rank > 5) {
    set_last_error("tensor map rank %d out of range", rank);
    return KR_ERR_INVALID_ARG;
  }
  cuuint64_t gdim[5];
  cuuint64_t gstride[4];
  cuuint32_t bdim[5];
  cuuint32_t estride[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bdim[i] = box[i];
    estride[i] = 1;
    if (i > 0) gstride[i - 1] = strides_bytes[i - 1];
  }
  CUresult r = fn(out, is_bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16,
                  static_cast<cuuint32_t>(rank), const_cast<void*>(base), gdim, gstride, bdim,
                  estride, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  swizzle_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B
                  : swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B
                  : swizzle_bytes == 32 ? CU_TENSOR_MAP_SWIZZLE_32B : CU_TENSOR_MAP_SWIZZLE_NONE,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error("cuTensorMapEncodeTiled failed (CUresult %d) rank=%d dims=[%llu,%llu,...] "
                   "box=[%u,%u,...] base=%p",
                   static_cast<int>(r), rank, (unsigned long long)dims[0],
                   (unsigned long long)(rank > 1 ? dims[1] : 0), box[0], rank > 1 ? box[1] : 0, base);
    return KR_ERR_TENSORMAP;
  }
  return KR_OK;
}

// byte tensors (FP8 operands): dims / box innermost first, strides in bytes for dims 1..rank-1
int make_tmap_u8(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                 const uint32_t* box, int swizzle_bytes) {
  EncodeTiledFn fn = get_encode_fn();
  if (fn == nullptr) {
    set_last_error("cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)");
    return KR_ERR_NO_DEVICE;
  }
  if (rank < 1 || rank > 5) {
    set_last_error("tensor map rank %d out of range", rank);
    return KR_ERR_INVALID_ARG;
  }
  cuuint64_t gdim[5];
  cuuint64_t gstride[4];
  cuuint32_t bdim[5];
  cuuint32_t estride[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bdim[i] = box[i];
    estride[i] = 1;
    if (i > 0) gstride[i - 1] = strides_bytes[i - 1];
  }
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_UINT8, static_cast<cuuint32_t>(rank), const_cast<void*>(base), gdim,
                  gstride, bdim, estride, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  swizzle_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error("cuTensorMapEncodeTiled (u8) failed (CUresult %d) dims=[%llu,%llu] box=[%u,%u] base=%p",
                   static_cast<int>(r), (unsigned long long)dims[0], (unsigned long long)(rank > 1 ? dims[1] : 0),
                   box[0], rank > 1 ? box[1] : 0, base);
    return KR_ERR_TENSORMAP;
  }
  return KR_OK;
}

int make_tmap_2d(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols,
                 uint64_t row_pitch_elems, uint32_t box_rows, uint32_t box_cols, bool is_bf16) {
  uint64_t dims[2] = {cols, rows};
  uint64_t strides[1] = {row_pitch_elems * 2};
  uint32_t box[2] = {box_cols, box_rows};
  return make_tmap_nd(out, base, 2, dims, strides, box, is_bf16, 128);
}

}  // namespace kr
