// vae_ops.cu -- bandwidth-bound pieces of the Wan VAE decoder on channels-last frames [pixels][C]:
//   fvb_rmsnorm_silu_cl   WanRMS_norm (F.normalize * sqrt(C) * gamma) [+ SiLU]   (wanvae.py:210-233, 414-446)
//   fvb_rmsnorm_silu_cl_e4m3  the same, written as e4m3 with a static per-tensor scale (input of an FP8 convolution)
//   fvb_upsample2x_cl     nearest-exact 2x spatial upsample                        (wanvae.py:236-248, 272-281)
//   fvb_transpose_bf16    [R, C] -> [C, R]                                         (V^T for the mid-block attention)
//   fvb_softmax_rows_f32  fp32 scores -> bf16 probabilities, rows of any length    (SDPA of WanAttentionBlock, wanvae.py:495)
//   fvb_clamp_to_nchw     channels-last bf16 -> clamp(-1,1) fp32 NCTHW             (wanvae.py:1210-1211)
#include <cuda_fp8.h>

#include "fvb_host.cuh"
#include "fvb_ptx.cuh"

namespace fvb {

// one warp per pixel; y = x / max(||x||_2, 1e-12) * sqrt(C) * gamma (+ beta), optional SiLU; fp32 math, bf16 out
// E4M3: out holds e4m3 bytes, q = e4m3_satfinite_rn(y * qscale) (no beta)
template <bool E4M3>
__global__ void __launch_bounds__(256) rmsnorm_silu_cl_kernel(const __nv_bfloat16* __restrict__ x, int64_t ldx,
                                                              const float* __restrict__ gamma, const float* __restrict__ beta,
                                                              void* __restrict__ out, int64_t ldo, int64_t npix,
                                                              int C, int apply_silu, float qscale) {
  const int64_t pix = int64_t(blockIdx.x) * 8 + (threadIdx.x >> 5);
  if (pix >= npix) return;
  const int lane = threadIdx.x & 31;
  const int nch = C >> 3;
  const __nv_bfloat16* xr = x + pix * ldx;
  float ss = 0.f;
  for (int ch = lane; ch < nch; ch += 32) {
    const uint4 u = reinterpret_cast<const uint4*>(xr)[ch];
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 f = __bfloat1622float2(h[i]);
      ss += f.x * f.x + f.y * f.y;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  const float denom = fmaxf(sqrtf(ss), 1e-12f);
  const float scale = sqrtf(float(C));
  __nv_bfloat16* orow = static_cast<__nv_bfloat16*>(out) + pix * ldo;
  uint8_t* qrow = static_cast<uint8_t*>(out) + pix * ldo;
  for (int ch = lane; ch < nch; ch += 32) {
    const uint4 u = reinterpret_cast<const uint4*>(xr)[ch];
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
    float y[8];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 f = __bfloat1622float2(h[i]);
      y[2 * i] = f.x;
      y[2 * i + 1] = f.y;
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      float v = __fmul_rn(__fmul_rn(__fdiv_rn(y[i], denom), scale), __ldg(gamma + ch * 8 + i));
      if (!E4M3 && beta) v = __fadd_rn(v, __ldg(beta + ch * 8 + i));
      if (apply_silu) v = __fdividef(v, 1.0f + __expf(-v));
      y[i] = v;
    }
    if constexpr (E4M3) {
      uint32_t w[2];
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const uint32_t lo = __nv_cvt_float2_to_fp8x2(make_float2(__fmul_rn(y[4 * i], qscale), __fmul_rn(y[4 * i + 1], qscale)),
                                                     __NV_SATFINITE, __NV_E4M3);
        const uint32_t hi = __nv_cvt_float2_to_fp8x2(make_float2(__fmul_rn(y[4 * i + 2], qscale), __fmul_rn(y[4 * i + 3], qscale)),
                                                     __NV_SATFINITE, __NV_E4M3);
        w[i] = lo | (hi << 16);
      }
      reinterpret_cast<uint2*>(qrow)[ch] = make_uint2(w[0], w[1]);
    } else {
      uint4 o;
      o.x = pack_bf16x2(y[0], y[1]);
      o.y = pack_bf16x2(y[2], y[3]);
      o.z = pack_bf16x2(y[4], y[5]);
      o.w = pack_bf16x2(y[6], y[7]);
      reinterpret_cast<uint4*>(orow)[ch] = o;
    }
  }
}

__global__ void upsample2x_cl_kernel(const uint4* __restrict__ in, uint4* __restrict__ out, int T, int H, int W, int C8) {
  const int64_t idx = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  const int64_t total = int64_t(T) * (2 * H) * (2 * W) * C8;
  if (idx >= total) return;
  const int c = int(idx % C8);
  int64_t r = idx / C8;
  const int x = int(r % (2 * W));
  r /= 2 * W;
  const int y = int(r % (2 * H));
  const int t = int(r / (2 * H));
  out[idx] = in[((int64_t(t) * H + (y >> 1)) * W + (x >> 1)) * C8 + c];
}

__global__ void transpose_bf16_kernel(const __nv_bfloat16* __restrict__ in, int64_t ldi, __nv_bfloat16* __restrict__ out,
                                      int64_t ldo, int R, int C) {
  __shared__ __nv_bfloat16 tile[32][33];
  const int r0 = blockIdx.y * 32, c0 = blockIdx.x * 32;
  for (int i = threadIdx.y; i < 32; i += 8) {
    const int r = r0 + i, c = c0 + threadIdx.x;
    tile[i][threadIdx.x] = (r < R && c < C) ? in[int64_t(r) * ldi + c] : __float2bfloat16(0.f);
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += 8) {
    const int c = c0 + i, r = r0 + threadIdx.x;
    if (c < C && r < R) out[int64_t(c) * ldo + r] = tile[threadIdx.x][i];
  }
}

// softmax over a row of fp32 logits (already scaled) -> bf16; 256 threads per row, three passes over global memory
__global__ void __launch_bounds__(256) softmax_rows_f32_kernel(const float* __restrict__ x, int64_t ldx,
                                                               __nv_bfloat16* __restrict__ out, int64_t ldo, int n) {
  __shared__ float red[8];
  const float* xr = x + int64_t(blockIdx.x) * ldx;
  float mx = -INFINITY;
  for (int i = threadIdx.x; i < n; i += 256) mx = fmaxf(mx, xr[i]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
  __syncthreads();
  mx = red[0];
#pragma unroll
  for (int i = 1; i < 8; ++i) mx = fmaxf(mx, red[i]);
  __syncthreads();
  float s = 0.f;
  for (int i = threadIdx.x; i < n; i += 256) s += __expf(xr[i] - mx);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  s = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) s += red[i];
  const float inv = 1.0f / s;
  __nv_bfloat16* orow = out + int64_t(blockIdx.x) * ldo;
  for (int i = threadIdx.x; i < n; i += 256) orow[i] = __float2bfloat16_rn(__expf(xr[i] - mx) * inv);
}

// channels-last bf16 [T][H][W][ld] (first C channels) -> fp32 [C][T][H][W], clamped to [-1, 1]
__global__ void clamp_to_nchw_kernel(const __nv_bfloat16* __restrict__ in, int64_t ld, float* __restrict__ out, int C,
                                     int64_t npix) {
  const int64_t idx = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= npix * C) return;
  const int64_t pix = idx % npix;
  const int c = int(idx / npix);
  const float v = __bfloat162float(in[pix * ld + c]);
  out[idx] = fminf(fmaxf(v, -1.0f), 1.0f);
}

}  // namespace fvb

using namespace fvb;

extern "C" int fvb_rmsnorm_silu_cl(const void* x, int64_t ldx, const float* gamma, const float* beta, void* out,
                                   int64_t ldo, int64_t npix, int C, int apply_silu, void* stream) {
  FVB_CHECK_ARG(x && gamma && out && npix > 0 && C > 0 && C % 8 == 0 && ldx % 8 == 0 && ldo % 8 == 0, "bad arguments");
  rmsnorm_silu_cl_kernel<false><<<(unsigned)((npix + 7) / 8), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const __nv_bfloat16*>(x), ldx, gamma, beta, out, ldo, npix, C, apply_silu, 0.f);
  FVB_CHECK_CUDA(cudaGetLastError());
  return FVB_OK;
}

extern "C" int fvb_rmsnorm_silu_cl_e4m3(const void* x, int64_t ldx, const float* gamma, void* out, int64_t ldo, int64_t npix,
                                        int C, int apply_silu, float bound, void* stream) {
  FVB_CHECK_ARG(x && gamma && out && npix > 0 && C > 0 && C % 8 == 0 && ldx % 8 == 0 && ldo % 8 == 0, "bad arguments");
  FVB_CHECK_ARG(bound >= 0.f, "bound must be >= 0");
  FVB_CHECK_ARG((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 7) == 0,
                "x must be 16-byte and out 8-byte aligned");
  const float qscale = bound > 0.f ? 448.0f / bound : 0.f;
  rmsnorm_silu_cl_kernel<true><<<(unsigned)((npix + 7) / 8), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const __nv_bfloat16*>(x), ldx, gamma, nullptr, out, ldo, npix, C, apply_silu, qscale);
  FVB_CHECK_CUDA(cudaGetLastError());
  return FVB_OK;
}

extern "C" int fvb_upsample2x_cl(const void* in, void* out, int T, int H, int W, int C, void* stream) {
  FVB_CHECK_ARG(in && out && T > 0 && H > 0 && W > 0 && C % 8 == 0, "bad arguments");
  const int64_t total = int64_t(T) * 2 * H * 2 * W * (C / 8);
  upsample2x_cl_kernel<<<(unsigned)((total + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const uint4*>(in), reinterpret_cast<uint4*>(out), T, H, W, C / 8);
  FVB_CHECK_CUDA(cudaGetLastError());
  return FVB_OK;
}

extern "C" int fvb_transpose_bf16(const void* in, int64_t ldi, void* out, int64_t ldo, int R, int C, void* stream) {
  FVB_CHECK_ARG(in && out && R > 0 && C > 0, "bad arguments");
  dim3 grid((C + 31) / 32, (R + 31) / 32), block(32, 8);
  transpose_bf16_kernel<<<grid, block, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const __nv_bfloat16*>(in), ldi, reinterpret_cast<__nv_bfloat16*>(out), ldo, R, C);
  FVB_CHECK_CUDA(cudaGetLastError());
  return FVB_OK;
}

extern "C" int fvb_softmax_rows_f32(const float* x, int64_t ldx, void* out, int64_t ldo, int64_t rows, int n, void* stream) {
  FVB_CHECK_ARG(x && out && rows > 0 && n > 0, "bad arguments");
  softmax_rows_f32_kernel<<<(unsigned)rows, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      x, ldx, reinterpret_cast<__nv_bfloat16*>(out), ldo, n);
  FVB_CHECK_CUDA(cudaGetLastError());
  return FVB_OK;
}

extern "C" int fvb_clamp_to_nchw(const void* in, int64_t ld, float* out, int C, int64_t npix, void* stream) {
  FVB_CHECK_ARG(in && out && C > 0 && npix > 0, "bad arguments");
  const int64_t total = npix * C;
  clamp_to_nchw_kernel<<<(unsigned)((total + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const __nv_bfloat16*>(in), ld, out, C, npix);
  FVB_CHECK_CUDA(cudaGetLastError());
  return FVB_OK;
}
