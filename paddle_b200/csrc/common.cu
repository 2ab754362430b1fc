#include "include/b200_common.cuh"
#include "include/b200_ops.h"
#include <stdio.h>
#include <string.h>

namespace b200 {
static thread_local char g_err[512] = {0};
static thread_local char g_err_out[512] = {0};
void set_last_error(const char* file, int line, const char* msg) {
  if (g_err[0] == 0) snprintf(g_err, sizeof(g_err), "%s:%d: %s", file, line, msg);
}
const char* take_last_error() {
  memcpy(g_err_out, g_err, sizeof(g_err));
  g_err[0] = 0;
  return g_err_out;
}

bool encode_tensor_map(CUtensorMap* out, CUtensorMapDataType type, int rank, const void* ptr, const uint64_t* dims,
                       const uint64_t* byte_strides, const uint32_t* box, const char* what) {
  bind_primary_context();
  // resolved through the runtime: the extension does not link libcuda
  static const auto encode = []() -> decltype(&cuTensorMapEncodeTiled) {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess)
      return nullptr;
    return reinterpret_cast<decltype(&cuTensorMapEncodeTiled)>(fn);
  }();
  char msg[160];
  if (!encode) {
    snprintf(msg, sizeof(msg), "%s: cuTensorMapEncodeTiled unavailable", what);
    set_last_error(__FILE__, __LINE__, msg);
    return false;
  }
  const uint32_t elem_strides[5] = {1, 1, 1, 1, 1};
  const CUresult r = encode(out, type, (uint32_t)rank, const_cast<void*>(ptr), dims, byte_strides, box, elem_strides,
                            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    snprintf(msg, sizeof(msg), "%s: cuTensorMapEncodeTiled failed (CUresult %d)", what, (int)r);
    set_last_error(__FILE__, __LINE__, msg);
    return false;
  }
  return true;
}
}  // namespace b200
