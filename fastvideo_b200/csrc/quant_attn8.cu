// quant_attn8.cu -- operand quantiser of the 8-bit attention (fvb_attention_8bit_quantize; arithmetic in include/fvb200.h).
//   1. kv_stats : per (b, h, 256-key chunk) and channel, the fp32 sum of k and the max |v| over the chunk (keys in order)
//   2. kv_finish: per (b, h) and channel, the chunk partials in chunk order -> k_mean = sum / Skv, v_scale = amax / 448
//   3. rows     : one warp per (token, head) row of 128: q, or k - k_mean, to int8 with one scale per row
//   4. v        : one thread per channel of a 64-key block: e4m3 of v * 448 / amax, transposed into the vt8 key-slot order
// No float atomics: every reduction has a fixed order, so the output is the same on every run.
#include <cuda_fp8.h>

#include "fvb_host.cuh"
#include "fvb_ptx.cuh"

namespace fvb {

constexpr int A8_D = 128;
constexpr int A8_CHUNK = 256;  // keys per kv_stats CTA
constexpr int A8_ROWS_PER_CTA = 8;

struct Bsh {
  int64_t b, s, h;
};

__global__ void __launch_bounds__(A8_D)
attn8_kv_stats_kernel(const __nv_bfloat16* __restrict__ k, Bsh ks, const __nv_bfloat16* __restrict__ v, Bsh vs, int H, int Skv,
                      int nchunk, float* __restrict__ ws_sum, float* __restrict__ ws_amax) {
  const int chunk = blockIdx.x, h = blockIdx.y, b = blockIdx.z, c = threadIdx.x;
  const int s0 = chunk * A8_CHUNK, s1 = min(Skv, s0 + A8_CHUNK);
  const __nv_bfloat16* kp = k + b * ks.b + h * ks.h + c;
  const __nv_bfloat16* vp = v + b * vs.b + h * vs.h + c;
  float sum = 0.f, amax = 0.f;
#pragma unroll 8
  for (int s = s0; s < s1; ++s) {
    sum = __fadd_rn(sum, __bfloat162float(kp[s * ks.s]));
    amax = fmaxf(amax, fabsf(__bfloat162float(vp[s * vs.s])));
  }
  const int64_t o = ((int64_t(b) * H + h) * nchunk + chunk) * A8_D + c;
  ws_sum[o] = sum;
  ws_amax[o] = amax;
}

__global__ void __launch_bounds__(A8_D)
attn8_kv_finish_kernel(const float* __restrict__ ws_sum, const float* __restrict__ ws_amax, int nchunk, int Skv,
                       float* __restrict__ k_mean, float* __restrict__ v_scale, float* __restrict__ v_inv) {
  const int64_t bh = blockIdx.x;
  const int c = threadIdx.x;
  float sum = 0.f, amax = 0.f;
  for (int i = 0; i < nchunk; ++i) {
    sum = __fadd_rn(sum, ws_sum[(bh * nchunk + i) * A8_D + c]);
    amax = fmaxf(amax, ws_amax[(bh * nchunk + i) * A8_D + c]);
  }
  k_mean[bh * A8_D + c] = __fdiv_rn(sum, float(Skv));
  v_scale[bh * A8_D + c] = amax > 0.f ? __fdiv_rn(amax, 448.f) : 1.f;
  v_inv[bh * A8_D + c] = amax > 0.f ? __fdiv_rn(448.f, amax) : 0.f;
}

// rows r = (b * H + h) * S + s; x8[r] int8 [128], scale[r]; mean (k only): fp32 [B, H, 128]
__global__ void __launch_bounds__(32 * A8_ROWS_PER_CTA)
attn8_rows_kernel(const __nv_bfloat16* __restrict__ x, Bsh xs, int H, int S, int64_t rows, const float* __restrict__ mean,
                  int8_t* __restrict__ x8, float* __restrict__ scale) {
  const int64_t r = int64_t(blockIdx.x) * A8_ROWS_PER_CTA + (threadIdx.x >> 5);
  if (r >= rows) return;
  const int lane = threadIdx.x & 31;
  const int s = int(r % S);
  const int64_t bh = r / S;
  const int h = int(bh % H), b = int(bh / H);
  const uint2 raw = *reinterpret_cast<const uint2*>(x + b * xs.b + s * xs.s + h * xs.h + 4 * lane);
  const __nv_bfloat162* hv = reinterpret_cast<const __nv_bfloat162*>(&raw);
  const float2 lo = __bfloat1622float2(hv[0]), hi = __bfloat1622float2(hv[1]);
  float f[4] = {lo.x, lo.y, hi.x, hi.y};
  if (mean != nullptr) {
    const float4 m = *reinterpret_cast<const float4*>(mean + bh * A8_D + 4 * lane);
    f[0] = __fsub_rn(f[0], m.x);
    f[1] = __fsub_rn(f[1], m.y);
    f[2] = __fsub_rn(f[2], m.z);
    f[3] = __fsub_rn(f[3], m.w);
  }
  float amax = fmaxf(fmaxf(fabsf(f[0]), fabsf(f[1])), fmaxf(fabsf(f[2]), fabsf(f[3])));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
  uint32_t packed = 0;
  if (amax > 0.f) {
    const float inv = __fdiv_rn(127.f, amax);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int q = min(127, max(-127, __float2int_rn(__fmul_rn(f[i], inv))));
      packed |= uint32_t(q & 0xFF) << (8 * i);
    }
  }
  reinterpret_cast<uint32_t*>(x8 + r * A8_D)[lane] = packed;
  if (lane == 0) scale[r] = amax > 0.f ? __fdiv_rn(amax, 127.f) : 1.f;
}

// vt8[b][h][kb][c][slot]: slot j of each 16-key group holds key 2 (j >> 2) + (j & 1) + 8 ((j >> 1) & 1) of the group
__global__ void __launch_bounds__(A8_D)
attn8_v_kernel(const __nv_bfloat16* __restrict__ v, Bsh vs, int H, int Skv, int nkb, const int32_t* __restrict__ kv_off,
               const int32_t* __restrict__ kv_len, const float* __restrict__ v_inv, uint8_t* __restrict__ vt8) {
  const int kb = blockIdx.x, h = blockIdx.y, b = blockIdx.z, c = threadIdx.x;
  int row0 = kv_off ? __ldg(kv_off + kb) : kb * 64;
  int vlen;
  if (kv_len) vlen = __ldg(kv_len + kb);
  else if (kv_off) vlen = min(64, __ldg(kv_off + kb + 1) - row0);
  else vlen = 64;
  vlen = min(vlen, max(0, Skv - row0));
  const int64_t bh = int64_t(b) * H + h;
  const float inv = v_inv[bh * A8_D + c];
  const __nv_bfloat16* vp = v + b * vs.b + h * vs.h + c;
  uint32_t w[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) {  // word i: slots 4 i .. 4 i + 3
    uint32_t word = 0;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int j = 4 * i + e;
      const int key = 16 * (j >> 4) + 2 * ((j & 15) >> 2) + (j & 1) + 8 * ((j >> 1) & 1);
      const float x = key < vlen ? __bfloat162float(vp[int64_t(row0 + key) * vs.s]) : 0.f;
      const uint32_t byte = inv > 0.f ? uint32_t(__nv_cvt_float_to_fp8(__fmul_rn(x, inv), __NV_SATFINITE, __NV_E4M3)) : 0u;
      word |= byte << (8 * e);
    }
    w[i] = word;
  }
  uint4* dst = reinterpret_cast<uint4*>(vt8 + ((bh * nkb + kb) * A8_D + c) * 64);
#pragma unroll
  for (int i = 0; i < 4; ++i) dst[i] = make_uint4(w[4 * i], w[4 * i + 1], w[4 * i + 2], w[4 * i + 3]);
}

static int64_t nchunks(int Skv) { return (int64_t(Skv) + A8_CHUNK - 1) / A8_CHUNK; }
static int64_t round256(int64_t n) { return (n + 255) / 256 * 256; }

}  // namespace fvb

using namespace fvb;

extern "C" int64_t fvb_attention_8bit_workspace_bytes(int B, int H, int Skv) {
  if (B <= 0 || H <= 0 || Skv <= 0) return 0;
  const int64_t bh = int64_t(B) * H;
  return 2 * round256(bh * nchunks(Skv) * A8_D * 4) + round256(bh * A8_D * 4);
}

extern "C" int fvb_attention_8bit_quantize(const void* q, const void* k, const void* v, const int64_t* q_strides,
                                           const int64_t* k_strides, const int64_t* v_strides, int B, int H, int Sq, int Skv,
                                           int head_dim, const int32_t* kv_off, const int32_t* kv_len, int nkb, void* q8,
                                           float* q_scale, void* k8, float* k_scale, float* k_mean, void* vt8, float* v_scale,
                                           void* workspace, int64_t workspace_bytes, void* stream) {
  FVB_CHECK_ARG(q && k && v && q_strides && k_strides && v_strides, "null pointer");
  FVB_CHECK_ARG(q8 && q_scale && k8 && k_scale && k_mean && vt8 && v_scale && workspace, "null pointer");
  FVB_CHECK_ARG(head_dim == A8_D, "head_dim must be 128");
  FVB_CHECK_ARG(B > 0 && H > 0 && Sq > 0 && Skv > 0 && nkb > 0, "empty problem");
  FVB_CHECK_ARG(H <= 65535 && B <= 65535, "too many heads / batches");
  if (kv_off == nullptr) FVB_CHECK_ARG(nkb == (Skv + 63) / 64, "without kv_off, nkb must be ceil(Skv / 64)");
  FVB_CHECK_ARG(workspace_bytes >= fvb_attention_8bit_workspace_bytes(B, H, Skv), "workspace too small");
  FVB_CHECK_ARG((reinterpret_cast<uintptr_t>(workspace) & 255) == 0, "workspace must be 256-byte aligned");
  for (int i = 0; i < 3; ++i)
    FVB_CHECK_ARG(q_strides[i] % 8 == 0 && k_strides[i] % 8 == 0 && v_strides[i] % 8 == 0, "strides must be multiples of 8 elements");
  FVB_CHECK_ARG(((reinterpret_cast<uintptr_t>(q) | reinterpret_cast<uintptr_t>(k) | reinterpret_cast<uintptr_t>(v)) & 15) == 0,
                "q, k, v must be 16-byte aligned");
  FVB_CHECK_ARG(((reinterpret_cast<uintptr_t>(q8) | reinterpret_cast<uintptr_t>(k8) | reinterpret_cast<uintptr_t>(vt8) |
                  reinterpret_cast<uintptr_t>(k_mean)) & 15) == 0,
                "q8, k8, vt8, k_mean must be 16-byte aligned");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const Bsh qs{q_strides[0], q_strides[1], q_strides[2]}, ks{k_strides[0], k_strides[1], k_strides[2]},
      vs{v_strides[0], v_strides[1], v_strides[2]};
  const auto* qb = reinterpret_cast<const __nv_bfloat16*>(q);
  const auto* kb = reinterpret_cast<const __nv_bfloat16*>(k);
  const auto* vb = reinterpret_cast<const __nv_bfloat16*>(v);
  const int64_t bh = int64_t(B) * H, nch = nchunks(Skv);
  float* ws_sum = reinterpret_cast<float*>(workspace);
  float* ws_amax = ws_sum + round256(bh * nch * A8_D * 4) / 4;
  float* v_inv = ws_amax + round256(bh * nch * A8_D * 4) / 4;

  attn8_kv_stats_kernel<<<dim3(unsigned(nch), unsigned(H), unsigned(B)), A8_D, 0, st>>>(kb, ks, vb, vs, H, Skv, int(nch),
                                                                                         ws_sum, ws_amax);
  FVB_CHECK_CUDA(cudaGetLastError());
  attn8_kv_finish_kernel<<<unsigned(bh), A8_D, 0, st>>>(ws_sum, ws_amax, int(nch), Skv, k_mean, v_scale, v_inv);
  FVB_CHECK_CUDA(cudaGetLastError());
  const int64_t qrows = bh * Sq, krows = bh * Skv;
  attn8_rows_kernel<<<unsigned((qrows + A8_ROWS_PER_CTA - 1) / A8_ROWS_PER_CTA), 32 * A8_ROWS_PER_CTA, 0, st>>>(
      qb, qs, H, Sq, qrows, nullptr, reinterpret_cast<int8_t*>(q8), q_scale);
  FVB_CHECK_CUDA(cudaGetLastError());
  attn8_rows_kernel<<<unsigned((krows + A8_ROWS_PER_CTA - 1) / A8_ROWS_PER_CTA), 32 * A8_ROWS_PER_CTA, 0, st>>>(
      kb, ks, H, Skv, krows, k_mean, reinterpret_cast<int8_t*>(k8), k_scale);
  FVB_CHECK_CUDA(cudaGetLastError());
  attn8_v_kernel<<<dim3(unsigned(nkb), unsigned(H), unsigned(B)), A8_D, 0, st>>>(vb, vs, H, Skv, nkb, kv_off, kv_len, v_inv,
                                                                                  reinterpret_cast<uint8_t*>(vt8));
  FVB_CHECK_CUDA(cudaGetLastError());
  return FVB_OK;
}
