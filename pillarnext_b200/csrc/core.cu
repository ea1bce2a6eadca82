// core.cu -- error reporting, version and TMA descriptor encoding for libpnx (C-ABI, see include/pnx.h).
#include <stdarg.h>
#include <string.h>

#include "pnx_common.cuh"

static thread_local char g_err[512] = "";

void pnx_set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

extern "C" const char* pnx_last_error(void) { return g_err; }
extern "C" int pnx_abi_version(void) { return 1; }

// number of SMs of the current device (used by the host side to size persistent grids)
extern "C" int pnx_sm_count(void) {
  int dev = 0, n = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return -1;
  if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return -1;
  return n;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (fn) return fn;
  void* p = nullptr;
  cudaDriverEntryPointQueryResult q;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess ||
      q != cudaDriverEntryPointSuccess)
    return nullptr;
  fn = (EncodeTiledFn)p;
  return fn;
}

int pnx_encode_tmap_2d_bf16(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols,
                            uint64_t row_stride_bytes, uint32_t box_rows, uint32_t box_cols) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) {
    pnx_set_error("cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)");
    return PNX_ERR_CUDA;
  }
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {row_stride_bytes};
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    pnx_set_error("cuTensorMapEncodeTiled failed: CUresult %d (rows=%llu cols=%llu box=%ux%u)", (int)r,
                  (unsigned long long)rows, (unsigned long long)cols, box_rows, box_cols);
    return PNX_ERR_CUDA;
  }
  return PNX_OK;
}

int pnx_encode_tmap_4d_bf16(CUtensorMap* out, const void* base, const uint64_t dims[4], const uint64_t strides_bytes[3],
                            const uint32_t box[4]) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) {
    pnx_set_error("cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)");
    return PNX_ERR_CUDA;
  }
  cuuint64_t d[4] = {dims[0], dims[1], dims[2], dims[3]};
  cuuint64_t st[3] = {strides_bytes[0], strides_bytes[1], strides_bytes[2]};
  cuuint32_t bx[4] = {box[0], box[1], box[2], box[3]};
  cuuint32_t es[4] = {1, 1, 1, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(base), d, st, bx, es,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    pnx_set_error("cuTensorMapEncodeTiled(4d) failed: CUresult %d", (int)r);
    return PNX_ERR_CUDA;
  }
  return PNX_OK;
}
