// fvb_host.cuh -- host-side helpers shared by the C-ABI entry points: error codes,
// cuTensorMapEncodeTiled lookup (through cudaGetDriverEntryPoint so the library has no
// link-time dependency on libcuda and loads on a GPU-less box), launch checks.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <mutex>

#include "../../include/fvb200.h"

namespace fvb {

extern thread_local char g_last_error[512];

inline int set_error(int code, const char* fmt, const char* a = "", long long b = 0, long long c = 0) {
  snprintf(g_last_error, sizeof(g_last_error), fmt, a ? a : "", b, c);
  return code;
}

#define FVB_CHECK_ARG(cond, msg)                                                    \
  do {                                                                              \
    if (!(cond)) return ::fvb::set_error(FVB_ERR_INVALID_ARG, "invalid argument: %s", msg); \
  } while (0)

#define FVB_CHECK_CUDA(expr)                                                                   \
  do {                                                                                         \
    cudaError_t _e = (expr);                                                                   \
    if (_e != cudaSuccess)                                                                     \
      return ::fvb::set_error(FVB_ERR_CUDA, "CUDA error: %s", cudaGetErrorString(_e));   \
  } while (0)

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                  CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                  CUtensorMapFloatOOBfill);

inline EncodeTiledFn get_encode_tiled() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, []() {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

// Tensor map of rank `rank` (<= 5) over elements of type `dtype`. dims/strides innermost first; strides[0] is implied
// (one element) and strides[i] (bytes) must be multiples of 16. 128B swizzle by default, zero OOB fill.
inline int make_tmap(CUtensorMap* out, CUtensorMapDataType dtype, const void* base, int rank, const uint64_t* dims,
                     const uint64_t* strides_bytes, const uint32_t* box,
                     CUtensorMapSwizzle swz = CU_TENSOR_MAP_SWIZZLE_128B) {
  EncodeTiledFn enc = get_encode_tiled();
  if (!enc) return set_error(FVB_ERR_NO_DEVICE, "cuTensorMapEncodeTiled unavailable (no CUDA driver)%s");
  cuuint64_t gdim[5], gstr[4];
  cuuint32_t bdim[5], estr[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bdim[i] = box[i];
    estr[i] = 1;
    if (i > 0) gstr[i - 1] = strides_bytes[i];
  }
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0)
    return set_error(FVB_ERR_INVALID_ARG, "tensor base not 16B aligned%s");
  CUresult r = enc(out, dtype, (cuuint32_t)rank, const_cast<void*>(base), gdim,
                   gstr, bdim, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return set_error(FVB_ERR_CUDA, "cuTensorMapEncodeTiled failed (%s) code %lld", "", (long long)r);
  return FVB_OK;
}

// bf16 tensor map (strides[0] implied: 2 bytes)
inline int make_tmap_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                          const uint64_t* strides_bytes, const uint32_t* box,
                          CUtensorMapSwizzle swz = CU_TENSOR_MAP_SWIZZLE_128B) {
  return make_tmap(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, base, rank, dims, strides_bytes, box, swz);
}

// one-byte tensor map (fp8 e4m3 operands; strides[0] implied: 1 byte)
inline int make_tmap_u8(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                        const uint64_t* strides_bytes, const uint32_t* box,
                        CUtensorMapSwizzle swz = CU_TENSOR_MAP_SWIZZLE_128B) {
  return make_tmap(out, CU_TENSOR_MAP_DATA_TYPE_UINT8, base, rank, dims, strides_bytes, box, swz);
}

// Tensor map of one bf16 operand of the head_dim-128 attention kernels: [B][H][S][128] addressed through (b, s, h) element
// strides, 64-row x 64-channel boxes (one 128B-swizzled half of a 64 x 128 tile).
inline int make_qkv_tmap(CUtensorMap* tm, const void* base, int64_t S, int64_t H, int64_t B, int64_t stride_s,
                         int64_t stride_h, int64_t stride_b) {
  uint64_t dims[4] = {128, (uint64_t)S, (uint64_t)H, (uint64_t)B};
  uint64_t str[4] = {2, (uint64_t)stride_s * 2, (uint64_t)stride_h * 2, (uint64_t)stride_b * 2};
  uint32_t box[4] = {64, 64, 1, 1};
  return make_tmap_bf16(tm, base, 4, dims, str, box);
}

inline int sm_count() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 132;  // H100 SXM
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
  }
  return n;
}

}  // namespace fvb
