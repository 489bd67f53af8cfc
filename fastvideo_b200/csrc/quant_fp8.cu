// quant_fp8.cu -- row-wise e4m3 quantisation (the activation / weight side of fvb_linear_fp8).
//   amax = max_k |x[r, k]| (fp32, exact for bf16), inv = 448 / amax, q = e4m3_satfinite_rn(x * inv), scale = amax / 448;
//   amax == 0: scale = 1 and q = 0.
// And row-wise int8 quantisation (the activation side of fvb_linear_w8a8_sp), the same rule with 127 and rint:
//   inv = 127 / amax, q = clamp(rint(x * inv), -127, 127), scale = amax / 127. Its rows may be read in K segments.
// One CTA per row. Each thread keeps its 16-byte vectors of the row in registers between the amax pass and the quantise
// pass, so the row is read from HBM once; rows longer than the register cache re-read the rest (from L2).
#include <cuda_fp8.h>

#include "fvb_host.cuh"
#include "fvb_ptx.cuh"

namespace fvb {

constexpr int QUANT_THREADS = 128;

FVB_DEVICE float amax8(const uint4& v, float m) {
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 f = __bfloat1622float2(h[i]);
    m = fmaxf(m, fmaxf(fabsf(f.x), fabsf(f.y)));
  }
  return m;
}

// 8 bf16 -> 8 e4m3 bytes (little-endian: element 0 in the lowest byte)
FVB_DEVICE uint2 quant8(const uint4& v, float inv) {
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&v);
  uint32_t w[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const float2 a = __bfloat1622float2(h[2 * i]), b = __bfloat1622float2(h[2 * i + 1]);
    const uint32_t lo = __nv_cvt_float2_to_fp8x2(make_float2(__fmul_rn(a.x, inv), __fmul_rn(a.y, inv)), __NV_SATFINITE, __NV_E4M3);
    const uint32_t hi = __nv_cvt_float2_to_fp8x2(make_float2(__fmul_rn(b.x, inv), __fmul_rn(b.y, inv)), __NV_SATFINITE, __NV_E4M3);
    w[i] = lo | (hi << 16);
  }
  return make_uint2(w[0], w[1]);
}

template <int NV>  // 16-byte vectors cached per thread
__global__ void __launch_bounds__(QUANT_THREADS)
quantize_fp8_rows_kernel(const __nv_bfloat16* __restrict__ x, int64_t ldx, int K, uint8_t* __restrict__ q, int64_t ldq,
                         float* __restrict__ scale) {
  const int64_t row = blockIdx.x;
  const uint4* xr = reinterpret_cast<const uint4*>(x + row * ldx);
  uint2* qr = reinterpret_cast<uint2*>(q + row * ldq);
  const int nvec = K / 8;
  uint4 v[NV];
  float m = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int idx = threadIdx.x + i * QUANT_THREADS;
    if (idx < nvec) {
      v[i] = __ldg(xr + idx);
      m = amax8(v[i], m);
    }
  }
  for (int idx = threadIdx.x + NV * QUANT_THREADS; idx < nvec; idx += QUANT_THREADS) m = amax8(__ldg(xr + idx), m);

  __shared__ float red[QUANT_THREADS / 32];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  m = red[0];
#pragma unroll
  for (int i = 1; i < QUANT_THREADS / 32; ++i) m = fmaxf(m, red[i]);

  if (m == 0.f) {
    if (threadIdx.x == 0) scale[row] = 1.f;
    for (int idx = threadIdx.x; idx < nvec; idx += QUANT_THREADS) qr[idx] = make_uint2(0u, 0u);
    return;
  }
  const float inv = __fdiv_rn(448.f, m);
  if (threadIdx.x == 0) scale[row] = __fdiv_rn(m, 448.f);
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int idx = threadIdx.x + i * QUANT_THREADS;
    if (idx < nvec) qr[idx] = quant8(v[i], inv);
  }
  for (int idx = threadIdx.x + NV * QUANT_THREADS; idx < nvec; idx += QUANT_THREADS) qr[idx] = quant8(__ldg(xr + idx), inv);
}

// 8 bf16 -> 8 int8 (element 0 in the lowest byte): clamp(rint(x * inv), -127, 127), rint half-to-even
FVB_DEVICE uint2 quant8_i8(const uint4& v, float inv) {
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&v);
  uint32_t w[2] = {0u, 0u};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 a = __bfloat1622float2(h[i]);
    const int q0 = min(max(__float2int_rn(__fmul_rn(a.x, inv)), -127), 127);
    const int q1 = min(max(__float2int_rn(__fmul_rn(a.y, inv)), -127), 127);
    w[i >> 1] |= ((uint32_t(q0) & 0xFFu) | ((uint32_t(q1) & 0xFFu) << 8)) << (16 * (i & 1));
  }
  return make_uint2(w[0], w[1]);
}

// Row r's logical element k lives at x + r * ldx + (k / seg_len) * seg_stride + k % seg_len (seg_len = K: a plain row).
// Vector idx (8 elements) never straddles a segment: seg_len is a multiple of 8.
template <int NV>  // 16-byte vectors cached per thread
__global__ void __launch_bounds__(QUANT_THREADS)
quantize_int8_rows_kernel(const __nv_bfloat16* __restrict__ x, int64_t ldx, int seg_len, int64_t seg_stride, int K,
                          int8_t* __restrict__ q, int64_t ldq, float* __restrict__ scale) {
  const int64_t row = blockIdx.x;
  const __nv_bfloat16* xr = x + row * ldx;
  uint2* qr = reinterpret_cast<uint2*>(q + row * ldq);
  const int nvec = K / 8;
  const int seg_vec = seg_len / 8;
  auto load = [&](int idx) {
    const int sg = idx / seg_vec;
    return __ldg(reinterpret_cast<const uint4*>(xr + sg * seg_stride) + (idx - sg * seg_vec));
  };
  uint4 v[NV];
  float m = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int idx = threadIdx.x + i * QUANT_THREADS;
    if (idx < nvec) {
      v[i] = load(idx);
      m = amax8(v[i], m);
    }
  }
  for (int idx = threadIdx.x + NV * QUANT_THREADS; idx < nvec; idx += QUANT_THREADS) m = amax8(load(idx), m);

  __shared__ float red[QUANT_THREADS / 32];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  m = red[0];
#pragma unroll
  for (int i = 1; i < QUANT_THREADS / 32; ++i) m = fmaxf(m, red[i]);

  if (m == 0.f) {
    if (threadIdx.x == 0) scale[row] = 1.f;
    for (int idx = threadIdx.x; idx < nvec; idx += QUANT_THREADS) qr[idx] = make_uint2(0u, 0u);
    return;
  }
  const float inv = __fdiv_rn(127.f, m);
  if (threadIdx.x == 0) scale[row] = __fdiv_rn(m, 127.f);
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int idx = threadIdx.x + i * QUANT_THREADS;
    if (idx < nvec) qr[idx] = quant8_i8(v[i], inv);
  }
  for (int idx = threadIdx.x + NV * QUANT_THREADS; idx < nvec; idx += QUANT_THREADS) qr[idx] = quant8_i8(load(idx), inv);
}

}  // namespace fvb

using namespace fvb;

extern "C" int fvb_quantize_fp8_rows(const void* x, int64_t ldx, int M, int K, void* q, int64_t ldq, float* scale,
                                     void* stream) {
  FVB_CHECK_ARG(x && q && scale, "null pointer");
  FVB_CHECK_ARG(M > 0 && K > 0, "empty problem");
  FVB_CHECK_ARG(K % 8 == 0, "K must be a multiple of 8");
  FVB_CHECK_ARG(ldx % 8 == 0 && ldx >= K, "ldx must be a multiple of 8 (16-byte rows) and >= K");
  FVB_CHECK_ARG(ldq % 8 == 0 && ldq >= K, "ldq must be a multiple of 8 and >= K");
  FVB_CHECK_ARG((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(q) & 7) == 0,
                "x must be 16-byte and q 8-byte aligned");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const auto* xb = reinterpret_cast<const __nv_bfloat16*>(x);
  auto* qb = reinterpret_cast<uint8_t*>(q);
  const int nvec = K / 8;
  if (nvec <= 4 * QUANT_THREADS)
    quantize_fp8_rows_kernel<4><<<M, QUANT_THREADS, 0, st>>>(xb, ldx, K, qb, ldq, scale);
  else if (nvec <= 8 * QUANT_THREADS)
    quantize_fp8_rows_kernel<8><<<M, QUANT_THREADS, 0, st>>>(xb, ldx, K, qb, ldq, scale);
  else
    quantize_fp8_rows_kernel<16><<<M, QUANT_THREADS, 0, st>>>(xb, ldx, K, qb, ldq, scale);
  FVB_CHECK_CUDA(cudaGetLastError());
  return FVB_OK;
}

extern "C" int fvb_quantize_int8_rows(const void* x, int64_t ldx, int x_seg_len, int64_t x_seg_stride, int M, int K, void* q,
                                      int64_t ldq, float* scale, void* stream) {
  FVB_CHECK_ARG(x && q && scale, "null pointer");
  FVB_CHECK_ARG(M > 0 && K > 0, "empty problem");
  FVB_CHECK_ARG(K % 8 == 0, "K must be a multiple of 8");
  if (x_seg_len <= 0 || x_seg_len >= K) {
    x_seg_len = K;
    x_seg_stride = 0;
  }
  FVB_CHECK_ARG(x_seg_len % 8 == 0 && K % x_seg_len == 0 && x_seg_stride % 8 == 0,
                "bad segmentation (x_seg_len a multiple of 8 dividing K, x_seg_stride a multiple of 8)");
  FVB_CHECK_ARG(ldx % 8 == 0 && ldx >= x_seg_len, "ldx must be a multiple of 8 (16-byte rows) and cover a segment");
  FVB_CHECK_ARG(ldq % 8 == 0 && ldq >= K, "ldq must be a multiple of 8 and >= K");
  FVB_CHECK_ARG((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(q) & 7) == 0,
                "x must be 16-byte and q 8-byte aligned");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const auto* xb = reinterpret_cast<const __nv_bfloat16*>(x);
  auto* qb = reinterpret_cast<int8_t*>(q);
  const int nvec = K / 8;
  if (nvec <= 4 * QUANT_THREADS)
    quantize_int8_rows_kernel<4><<<M, QUANT_THREADS, 0, st>>>(xb, ldx, x_seg_len, x_seg_stride, K, qb, ldq, scale);
  else if (nvec <= 8 * QUANT_THREADS)
    quantize_int8_rows_kernel<8><<<M, QUANT_THREADS, 0, st>>>(xb, ldx, x_seg_len, x_seg_stride, K, qb, ldq, scale);
  else
    quantize_int8_rows_kernel<16><<<M, QUANT_THREADS, 0, st>>>(xb, ldx, x_seg_len, x_seg_stride, K, qb, ldq, scale);
  FVB_CHECK_CUDA(cudaGetLastError());
  return FVB_OK;
}
