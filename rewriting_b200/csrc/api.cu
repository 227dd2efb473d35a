// api.cu — the library-level part of the extern "C" boundary declared in
// include/rewriting_b200.h (version, last error, device), and the host-side utilities the kernel
// translation units share: the error state, check_cuda, the SM count and the TMA descriptor
// encoders.  Every other entry point is defined beside the kernel it launches.
#include <cstdarg>
#include <cstdio>
#include <mutex>

#include "../../include/rewriting_b200.h"
#include "rw_common.cuh"

namespace rw {

static thread_local char g_err[512] = "";

void set_last_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int check_cuda(cudaError_t e, const char* what) {
  if (e == cudaSuccess) return RW_OK;
  set_last_error("%s: %s (%s)", what, cudaGetErrorName(e), cudaGetErrorString(e));
  return RW_ERR_CUDA;
}

int device_sm_count() {
  static int cached[64] = {0};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
  if (cached[dev] == 0) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0)
      n = 132;
    cached[dev] = n;
  }
  return cached[dev];
}

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                    const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                    const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode_fn() {
  static PFN_encodeTiled fn = nullptr;
  static std::once_flag once;
  std::call_once(once, []() {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q);
    if (e == cudaSuccess && q == cudaDriverEntryPointSuccess) fn = reinterpret_cast<PFN_encodeTiled>(p);
  });
  return fn;
}

int make_tmap_2d_bf16(CUtensorMap* out, const void* base, uint64_t inner, uint64_t outer,
                      uint64_t row_stride_bytes, uint32_t box_inner, uint32_t box_outer) {
  PFN_encodeTiled fn = get_encode_fn();
  if (!fn) {
    set_last_error("cuTensorMapEncodeTiled not available from the driver");
    return RW_ERR_NO_DRIVER_SYMBOL;
  }
  if ((reinterpret_cast<uintptr_t>(base) & 0xF) != 0 || (row_stride_bytes & 0xF) != 0) {
    set_last_error("TMA operand must be 16-byte aligned (ptr=%p stride=%llu)", base,
                   (unsigned long long)row_stride_bytes);
    return RW_ERR_BAD_ARG;
  }
  cuuint64_t gdim[2] = {inner, outer};
  cuuint64_t gstr[1] = {row_stride_bytes};
  cuuint32_t box[2] = {box_inner, box_outer};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), gdim, gstr,
                  box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error("cuTensorMapEncodeTiled failed: CUresult %d (inner=%llu outer=%llu box=%ux%u)",
                   (int)r, (unsigned long long)inner, (unsigned long long)outer, box_inner,
                   box_outer);
    return RW_ERR_CUDA;
  }
  return RW_OK;
}

// general form: rank <= 5, element strides (a stride s on dimension d loads every s-th element
// of the box extent box[d]), swizzle 0 = none, 1 = 32 B, 2 = 128 B, 3 = 64 B
int make_tmap_nd_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                      const uint64_t* strides_bytes, const uint32_t* box, const uint32_t* estrides,
                      int swizzle) {
  PFN_encodeTiled fn = get_encode_fn();
  if (!fn) {
    set_last_error("cuTensorMapEncodeTiled not available from the driver");
    return RW_ERR_NO_DRIVER_SYMBOL;
  }
  if (rank < 2 || rank > 5 || (reinterpret_cast<uintptr_t>(base) & 0xF) != 0) {
    set_last_error("TMA operand: rank %d, ptr %p (must be rank 2..5, 16-byte aligned)", rank, base);
    return RW_ERR_BAD_ARG;
  }
  cuuint64_t gdim[5], gstr[4];
  cuuint32_t bx[5], es[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bx[i] = box[i];
    es[i] = estrides ? estrides[i] : 1u;
    if (i + 1 < rank) gstr[i] = strides_bytes[i];
  }
  const CUtensorMapSwizzle sw = swizzle == 2   ? CU_TENSOR_MAP_SWIZZLE_128B
                                : swizzle == 3 ? CU_TENSOR_MAP_SWIZZLE_64B
                                : swizzle == 1 ? CU_TENSOR_MAP_SWIZZLE_32B
                                               : CU_TENSOR_MAP_SWIZZLE_NONE;
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, static_cast<cuuint32_t>(rank),
                  const_cast<void*>(base), gdim, gstr, bx, es, CU_TENSOR_MAP_INTERLEAVE_NONE, sw,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error("cuTensorMapEncodeTiled(rank %d) failed: CUresult %d (dim0 %llu dim1 %llu box %u %u)",
                   rank, (int)r, (unsigned long long)dims[0], (unsigned long long)dims[1], box[0],
                   box[1]);
    return RW_ERR_CUDA;
  }
  return RW_OK;
}

}  // namespace rw

using namespace rw;

extern "C" {

int rw_version(void) { return 100; }
const char* rw_last_error(void) { return g_err; }
int rw_set_device(int device) { return check_cuda(cudaSetDevice(device), "cudaSetDevice"); }
int rw_device_sm_count(void) { return device_sm_count(); }

}  // extern "C"
