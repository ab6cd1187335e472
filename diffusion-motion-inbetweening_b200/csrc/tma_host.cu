// Host-side TMA descriptor construction + the library's last-error string.
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <mutex>

#include "kernels.h"

namespace cmdi {

namespace {
thread_local char g_last_error[1024] = "";

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

PFN_encodeTiled get_encode_fn() {
  static PFN_encodeTiled fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    // resolved from the driver at run time: the library itself does not link libcuda
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres);
    if (e == cudaSuccess && qres == cudaDriverEntryPointSuccess) fn = reinterpret_cast<PFN_encodeTiled>(ptr);
  });
  return fn;
}
}  // namespace

void set_last_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_last_error, sizeof(g_last_error), fmt, ap);
  va_end(ap);
}

const char* get_last_error() { return g_last_error; }

int make_tmap_2d(CUtensorMap* out, const void* base, int elem_bytes, uint64_t rows, uint64_t cols, uint64_t ld,
                 uint32_t box_cols, uint32_t box_rows);

int make_tmap_bf16_2d(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_cols,
                      uint32_t box_rows) {
  return make_tmap_2d(out, base, 2, rows, cols, ld, box_cols, box_rows);
}

// elem_bytes: 2 (bf16) or 4 (fp32); the box is one swizzle row wide: 128 bytes (SWIZZLE_128B) or 64 bytes (SWIZZLE_64B)
int make_tmap_2d(CUtensorMap* out, const void* base, int elem_bytes, uint64_t rows, uint64_t cols, uint64_t ld,
                 uint32_t box_cols, uint32_t box_rows) {
  PFN_encodeTiled fn = get_encode_fn();
  if (!fn) {
    set_last_error("cuTensorMapEncodeTiled not available from the driver");
    return 1;
  }
  if ((ld * elem_bytes) % 16 != 0 || (reinterpret_cast<uintptr_t>(base) % 16) != 0 || (box_cols * elem_bytes != 128 && box_cols * elem_bytes != 64) ||
      box_rows > 256 || (elem_bytes != 2 && elem_bytes != 4)) {
    set_last_error("make_tmap_2d: bad geometry (ld=%llu box=%ux%u)", (unsigned long long)ld, box_cols, box_rows);
    return 1;
  }
  cuuint64_t gdim[2] = {cols, rows};
  cuuint64_t gstride[1] = {ld * (uint64_t)elem_bytes};  // bytes, dim 1
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(out, elem_bytes == 2 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<void*>(base), gdim, gstride, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, box_cols * elem_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error("cuTensorMapEncodeTiled failed: CUresult %d (rows=%llu cols=%llu ld=%llu box=%ux%u)", (int)r,
                   (unsigned long long)rows, (unsigned long long)cols, (unsigned long long)ld, box_cols, box_rows);
    return 1;
  }
  return 0;
}

}  // namespace cmdi

#include "../../include/condmdi_b200.h"

extern "C" const char* cmdi_last_error(void) { return cmdi::get_last_error(); }
extern "C" const char* cmdi_version(void) { return "condmdi_b200 0.1 (sm_90a: wgmma + TMA)"; }
