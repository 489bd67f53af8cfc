// elementwise.cu -- HBM-bound row kernels of the Wan block: fp32 LayerNorm + AdaLN modulation,
// QK RMSNorm (across all heads) fused with 3D RoPE, VSA gate combine.
// Two families: warp-per-row kernels for the large activations (a warp owns whole rows, staged in shared memory
// by 1-D bulk copies one or more rows ahead; only warp shuffles synchronise) and block-per-row kernels (one CTA per
// token row, the row kept in registers between the statistics pass and the write) as the fallback for small inputs.
// Either way every tensor is read once and written once with 128-bit accesses.
//
// Rounding points mirror the reference's eager path exactly (they decide where bf16 rounding
// happens): fastvideo/models/dits/wanvideo.py:393,398-401,419-432, fastvideo/layers/layernorm.py:48-83,
// 115-125,159-213,216-273, fastvideo/layers/rotary_embedding.py:105-135.
#include <algorithm>
#include "fvb_host.cuh"
#include "fvb_ptx.cuh"

namespace fvb {

constexpr int EW_THREADS = 256;
constexpr int EW_MAX_CHUNKS = 4;  // 256 threads * 4 chunks * 8 elements = 8192 columns max

FVB_DEVICE float block_sum(float v, float* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();  // protect `red` from the previous use
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float t = (lane < EW_THREADS / 32) ? red[lane] : 0.f;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
  return t;
}

FVB_DEVICE void unpack8(const uint4& u, float* f) {
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float2 t = __bfloat1622float2(h[i]);
    f[2 * i] = t.x;
    f[2 * i + 1] = t.y;
  }
}
FVB_DEVICE uint4 pack8(const float* f) {
  uint4 u;
  u.x = pack_bf16x2(f[0], f[1]);
  u.y = pack_bf16x2(f[2], f[3]);
  u.z = pack_bf16x2(f[4], f[5]);
  u.w = pack_bf16x2(f[6], f[7]);
  return u;
}

// ------------------------------------------------------------------------------------------
// LayerNorm family.  IN_F32: input row is fp32 (the un-rounded gated residual) else bf16.
//   y_ln = (x - mean) * rstd [* w + b]                 (fp32, biased variance, eps inside sqrt)
//   ROUND_LN: y_ln is rounded to bf16 before modulation (the reference's FP32LayerNorm casts back to
//             the input dtype when the input is bf16: layernorm.py:117-125)
//   modulation (scale != NULL): y = y_ln * (1 + scale[c]) + shift[c]     (fp32 mul, then fp32 add)
//   out = bf16(y);  hidden_out (optional) = bf16(x)  -- the residual stream cast (wanvideo.py:421)
// ------------------------------------------------------------------------------------------
template <bool IN_F32, bool ROUND_LN, bool MOD_BF16 = false>
__global__ void __launch_bounds__(EW_THREADS) layernorm_kernel(const void* __restrict__ x_, int64_t ldx,
                                                               const float* __restrict__ w,
                                                               const float* __restrict__ b,
                                                               const float* __restrict__ scale,
                                                               const float* __restrict__ shift,
                                                               __nv_bfloat16* __restrict__ out, int64_t ldo,
                                                               __nv_bfloat16* __restrict__ hidden_out, int64_t ldh,
                                                               int D, float eps, int mod_rows, int64_t mod_stride) {
  __shared__ float red[32];
  const int64_t row = blockIdx.x;
  if (mod_rows > 0 && scale != nullptr) {  // per-row-group modulation (causal Wan: one (scale, shift) per latent frame)
    const int64_t g = (row / mod_rows) * mod_stride;
    scale += g;
    shift += g;
  }
  const int nchunks = D >> 3;
  float v[EW_MAX_CHUNKS][8];
  float s = 0.f;
#pragma unroll
  for (int c = 0; c < EW_MAX_CHUNKS; ++c) {
    const int ch = threadIdx.x + c * EW_THREADS;
    if (ch < nchunks) {
      if constexpr (IN_F32) {
        const float4* xp = reinterpret_cast<const float4*>(reinterpret_cast<const float*>(x_) + row * ldx) + 2 * ch;
        float4 a = xp[0], bb = xp[1];
        v[c][0] = a.x; v[c][1] = a.y; v[c][2] = a.z; v[c][3] = a.w;
        v[c][4] = bb.x; v[c][5] = bb.y; v[c][6] = bb.z; v[c][7] = bb.w;
      } else {
        const uint4 u = reinterpret_cast<const uint4*>(reinterpret_cast<const __nv_bfloat16*>(x_) + row * ldx)[ch];
        unpack8(u, v[c]);
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) s += v[c][i];
    }
  }
  const float mean = block_sum(s, red) / float(D);
  float q = 0.f;
#pragma unroll
  for (int c = 0; c < EW_MAX_CHUNKS; ++c) {
    const int ch = threadIdx.x + c * EW_THREADS;
    if (ch < nchunks) {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float d = v[c][i] - mean;
        q += d * d;
      }
    }
  }
  const float var = block_sum(q, red) / float(D);
  const float rstd = rsqrtf(var + eps);
#pragma unroll
  for (int c = 0; c < EW_MAX_CHUNKS; ++c) {
    const int ch = threadIdx.x + c * EW_THREADS;
    if (ch < nchunks) {
      const int col = ch << 3;
      if (hidden_out != nullptr) reinterpret_cast<uint4*>(hidden_out + row * ldh)[ch] = pack8(v[c]);
      float y[8];
      // per-column vectors are read 128 bits at a time (scalar loads made this kernel LSU-issue bound)
      float wv[8], bv[8], sc[8], sh[8];
      if (w != nullptr) {
        const float4 w0 = __ldg(reinterpret_cast<const float4*>(w + col)), w1 = __ldg(reinterpret_cast<const float4*>(w + col + 4));
        const float4 b0 = __ldg(reinterpret_cast<const float4*>(b + col)), b1 = __ldg(reinterpret_cast<const float4*>(b + col + 4));
        wv[0] = w0.x; wv[1] = w0.y; wv[2] = w0.z; wv[3] = w0.w; wv[4] = w1.x; wv[5] = w1.y; wv[6] = w1.z; wv[7] = w1.w;
        bv[0] = b0.x; bv[1] = b0.y; bv[2] = b0.z; bv[3] = b0.w; bv[4] = b1.x; bv[5] = b1.y; bv[6] = b1.z; bv[7] = b1.w;
      }
      if (scale != nullptr) {
        const float4 s0 = __ldg(reinterpret_cast<const float4*>(scale + col)), s1 = __ldg(reinterpret_cast<const float4*>(scale + col + 4));
        const float4 h0 = __ldg(reinterpret_cast<const float4*>(shift + col)), h1 = __ldg(reinterpret_cast<const float4*>(shift + col + 4));
        sc[0] = s0.x; sc[1] = s0.y; sc[2] = s0.z; sc[3] = s0.w; sc[4] = s1.x; sc[5] = s1.y; sc[6] = s1.z; sc[7] = s1.w;
        sh[0] = h0.x; sh[1] = h0.y; sh[2] = h0.z; sh[3] = h0.w; sh[4] = h1.x; sh[5] = h1.y; sh[6] = h1.z; sh[7] = h1.w;
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        float t = (v[c][i] - mean) * rstd;
        if (w != nullptr) t = __fadd_rn(__fmul_rn(t, wv[i]), bv[i]);
        if constexpr (ROUND_LN) t = bf16_round(t);
        if (scale != nullptr) {
          if constexpr (MOD_BF16)  // bf16 tensors all the way: every elementwise op rounds (causal blocks with a bf16 `e`)
            t = bf16_round(__fadd_rn(bf16_round(__fmul_rn(t, bf16_round(__fadd_rn(1.0f, sc[i])))), sh[i]));
          else
            t = __fadd_rn(__fmul_rn(t, __fadd_rn(1.0f, sc[i])), sh[i]);
        }
        y[i] = t;
      }
      reinterpret_cast<uint4*>(out + row * ldo)[ch] = pack8(y);
    }
  }
}

// ------------------------------------------------------------------------------------------
// RMSNorm over the full row (all heads) + weight + optional interleaved-pair RoPE, in place.
//   n = bf16(x * rsqrt(mean(x^2) + eps));  n = bf16(n * w)            (layernorm.py:73-79)
//   rope (cos != NULL), pairs (2i, 2i+1) inside each head:            (rotary_embedding.py:124-135)
//     o[2i]   = bf16(n[2i]   * cos[2i]   + (-n[2i+1]) * sin[2i])
//     o[2i+1] = bf16(n[2i+1] * cos[2i+1] + ( n[2i]  ) * sin[2i+1])
//   cos/sin: fp32 [S_pos, head_dim] (the reference's repeat-interleaved table); rope_row maps a token
//   row to its table row (NULL = identity) so permuted / sharded token orders share one table.
// Up to two tensors (q and k) per launch: blockIdx.y selects.
// ------------------------------------------------------------------------------------------
FVB_DEVICE void load8_f32(const float* p, float (&o)[8]) {
  const float4 a = __ldg(reinterpret_cast<const float4*>(p)), b = __ldg(reinterpret_cast<const float4*>(p) + 1);
  o[0] = a.x; o[1] = a.y; o[2] = a.z; o[3] = a.w; o[4] = b.x; o[5] = b.y; o[6] = b.z; o[7] = b.w;
}

struct RmsRopeArgs {
  __nv_bfloat16* x[2];
  const __nv_bfloat16* w[2];
  int64_t ld[2];
  int w_f32 = 0;  // weights are fp32 [D]: x_norm(bf16) * w stays fp32 through RoPE, ONE rounding at the end (layernorm.py:73-79
                  // with an fp32 parameter: torch promotes the product and everything downstream of it to fp32)
  const int64_t* col_offsets;  // optional: element offset of each 128-column block inside a row (see fvb_linear_bf16_sp)
  // out-of-place scatter (fvb_rmsnorm_rope_scatter): results go to y[t] + row*ldy + out_col_offsets[block] instead of
  // back into x; the offsets may point into peer GPUs' memory. w[t] == NULL copies the row unchanged.
  __nv_bfloat16* y[2] = {nullptr, nullptr};
  int64_t ldy = 0;
  const int64_t* out_col_offsets = nullptr;
};

template <bool ROPE_F64>
__global__ void __launch_bounds__(EW_THREADS) rmsnorm_rope_kernel(RmsRopeArgs a, const void* __restrict__ cos_v,
                                                                  const void* __restrict__ sin_v,
                                                                  const int32_t* __restrict__ rope_row, int D,
                                                                  int head_dim, float eps) {
  const float* cos_t = reinterpret_cast<const float*>(cos_v);
  const float* sin_t = reinterpret_cast<const float*>(sin_v);
  __shared__ float red[32];
  const int which = blockIdx.y;
  const int64_t row = blockIdx.x;
  __nv_bfloat16* xr = a.x[which] + row * a.ld[which];
  const __nv_bfloat16* w = a.w[which];
  const int nchunks = D >> 3;
  float v[EW_MAX_CHUNKS][8];
  float s = 0.f;
#pragma unroll
  for (int c = 0; c < EW_MAX_CHUNKS; ++c) {
    const int ch = threadIdx.x + c * EW_THREADS;
    if (ch < nchunks) {
      const int64_t eoff = a.col_offsets ? __ldg(a.col_offsets + (ch >> 4)) + ((ch & 15) << 3) : int64_t(ch) << 3;
      unpack8(*reinterpret_cast<const uint4*>(xr + eoff), v[c]);
#pragma unroll
      for (int i = 0; i < 8; ++i) s += v[c][i] * v[c][i];
    }
  }
  const float var = block_sum(s, red) / float(D);
  const float rstd = rsqrtf(var + eps);
  const int64_t prow = (rope_row != nullptr) ? int64_t(rope_row[row]) : row;
  // A thread's chunks are EW_THREADS*8 columns apart: when the head size divides that, they all sit at the same offset
  // inside a head and share one 8-entry slice of the table row (the kernel was LSU-bound re-reading it per chunk).
  const bool hoisted = !ROPE_F64 && cos_t != nullptr && (EW_THREADS * 8) % head_dim == 0;
  float cs_h[8], sn_h[8];
  if (hoisted) {
    const int hc = (threadIdx.x << 3) % head_dim;
    const float4* cp = reinterpret_cast<const float4*>(cos_t + prow * head_dim + hc);
    const float4* sp = reinterpret_cast<const float4*>(sin_t + prow * head_dim + hc);
    const float4 c0 = __ldg(cp), c1 = __ldg(cp + 1), s0 = __ldg(sp), s1 = __ldg(sp + 1);
    cs_h[0] = c0.x; cs_h[1] = c0.y; cs_h[2] = c0.z; cs_h[3] = c0.w; cs_h[4] = c1.x; cs_h[5] = c1.y; cs_h[6] = c1.z; cs_h[7] = c1.w;
    sn_h[0] = s0.x; sn_h[1] = s0.y; sn_h[2] = s0.z; sn_h[3] = s0.w; sn_h[4] = s1.x; sn_h[5] = s1.y; sn_h[6] = s1.z; sn_h[7] = s1.w;
  }
#pragma unroll
  for (int c = 0; c < EW_MAX_CHUNKS; ++c) {
    const int ch = threadIdx.x + c * EW_THREADS;
    if (ch < nchunks) {
      const int col = ch << 3;
      float wv[8], n[8], y[8];
      if (a.w_f32) {
        load8_f32(reinterpret_cast<const float*>(w) + col, wv);
#pragma unroll
        for (int i = 0; i < 8; ++i) n[i] = __fmul_rn(bf16_round(__fmul_rn(v[c][i], rstd)), wv[i]);
      } else {
        unpack8(__ldg(reinterpret_cast<const uint4*>(w) + ch), wv);
#pragma unroll
        for (int i = 0; i < 8; ++i) n[i] = bf16_round(__fmul_rn(bf16_round(__fmul_rn(v[c][i], rstd)), wv[i]));
      }
      if constexpr (ROPE_F64) {
        // float64 tables (the causal model hands get_rotary_pos_embed's float64 output to the blocks unconverted,
        // causal_wanvideo.py:589-598): x.float() * cos promotes to float64, the result goes double -> float -> bf16.
        const int hc = col % head_dim;
        const double2* cp = reinterpret_cast<const double2*>(reinterpret_cast<const double*>(cos_v) + prow * head_dim + hc);
        const double2* sp = reinterpret_cast<const double2*>(reinterpret_cast<const double*>(sin_v) + prow * head_dim + hc);
#pragma unroll
        for (int i = 0; i < 8; i += 2) {
          const double2 c = __ldg(cp + (i >> 1)), sn = __ldg(sp + (i >> 1));
          y[i] = __double2float_rn(__dadd_rn(__dmul_rn(double(n[i]), c.x), __dmul_rn(double(-n[i + 1]), sn.x)));
          y[i + 1] = __double2float_rn(__dadd_rn(__dmul_rn(double(n[i + 1]), c.y), __dmul_rn(double(n[i]), sn.y)));
        }
      } else if (cos_t != nullptr) {
        float cs[8], sn[8];
        if (hoisted) {
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            cs[i] = cs_h[i];
            sn[i] = sn_h[i];
          }
        } else {
          const int hc = col % head_dim;  // 8 | head_dim, so a chunk never straddles heads
          const float4* cp = reinterpret_cast<const float4*>(cos_t + prow * head_dim + hc);
          const float4* sp = reinterpret_cast<const float4*>(sin_t + prow * head_dim + hc);
          const float4 c0 = __ldg(cp), c1 = __ldg(cp + 1), s0 = __ldg(sp), s1 = __ldg(sp + 1);
          cs[0] = c0.x; cs[1] = c0.y; cs[2] = c0.z; cs[3] = c0.w; cs[4] = c1.x; cs[5] = c1.y; cs[6] = c1.z; cs[7] = c1.w;
          sn[0] = s0.x; sn[1] = s0.y; sn[2] = s0.z; sn[3] = s0.w; sn[4] = s1.x; sn[5] = s1.y; sn[6] = s1.z; sn[7] = s1.w;
        }
#pragma unroll
        for (int i = 0; i < 8; i += 2) {
          y[i] = __fadd_rn(__fmul_rn(n[i], cs[i]), __fmul_rn(-n[i + 1], sn[i]));
          y[i + 1] = __fadd_rn(__fmul_rn(n[i + 1], cs[i + 1]), __fmul_rn(n[i], sn[i + 1]));
        }
      } else {
#pragma unroll
        for (int i = 0; i < 8; ++i) y[i] = n[i];
      }
      const int64_t eoff = a.col_offsets ? __ldg(a.col_offsets + (ch >> 4)) + ((ch & 15) << 3) : int64_t(ch) << 3;
      *reinterpret_cast<uint4*>(xr + eoff) = pack8(y);
    }
  }
}


// ------------------------------------------------------------------------------------------
// Warp-per-row variants (used for the large activations; the block-per-row kernels above remain the fallback for
// small or oddly laid out inputs). The block-per-row kernels spend ~4000 cycles per row in serial phases (load ->
// two block reductions with four __syncthreads -> write) with 2-4 CTAs per SM, so their time did not depend on the
// bytes moved: 0.56 ms for a bf16 [75600, 5120] LayerNorm (2.7 TB/s) and 0.62 ms for the fp32-input one (5.0 TB/s).
// Here every warp owns whole rows: the row is staged in shared memory by one 1-D bulk copy (cp.async.bulk + mbarrier,
// issued one or more rows ahead by lane 0), the statistics and the output passes re-read it from shared memory, and
// nothing but warp shuffles synchronises. 8 warps x (1-4) staged rows keep ~160 KB per SM in flight.
// ------------------------------------------------------------------------------------------
constexpr int RW_WARPS = 16;
constexpr int RW_MAX_STAGES = 2;
constexpr int RW_SMEM_BUDGET = 192 * 1024;  // row staging
constexpr int RW_SMEM_MAX = 226 * 1024;     // staging + the per-column table of the LayerNorm kernel (static barriers take 256 B more)

FVB_DEVICE float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

template <bool IN_F32>
FVB_DEVICE void load8(const uint8_t* srow, int ch, float* f) {
  if constexpr (IN_F32) {
    const float4* xp = reinterpret_cast<const float4*>(srow) + 2 * ch;
    const float4 a = xp[0], b = xp[1];
    f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w; f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
  } else {
    unpack8(reinterpret_cast<const uint4*>(srow)[ch], f);
  }
}

// eight values as four float pairs: the fp32 pipe's packed instructions (add / mul / fma .f32x2, each lane rounded exactly
// like the scalar instruction) halve the issue slots of the three passes below
template <bool IN_F32>
FVB_DEVICE void load8p(const uint8_t* srow, int ch, float2* f) {
  if constexpr (IN_F32) {
    const float4* xp = reinterpret_cast<const float4*>(srow) + 2 * ch;
    const float4 a = xp[0], b = xp[1];
    f[0] = make_float2(a.x, a.y); f[1] = make_float2(a.z, a.w); f[2] = make_float2(b.x, b.y); f[3] = make_float2(b.z, b.w);
  } else {
    const uint4 u = reinterpret_cast<const uint4*>(srow)[ch];
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) f[i] = make_float2(__uint_as_float(w[i] << 16), __uint_as_float(w[i] & 0xffff0000u));
  }
}
FVB_DEVICE void lds8p(const float* p, float2* f) {
  const float4 a = *reinterpret_cast<const float4*>(p), b = *reinterpret_cast<const float4*>(p + 4);
  f[0] = make_float2(a.x, a.y); f[1] = make_float2(a.z, a.w); f[2] = make_float2(b.x, b.y); f[3] = make_float2(b.z, b.w);
}
FVB_DEVICE void ldg8p(const float* p, float2* f) {
  const float4 a = __ldg(reinterpret_cast<const float4*>(p)), b = __ldg(reinterpret_cast<const float4*>(p + 4));
  f[0] = make_float2(a.x, a.y); f[1] = make_float2(a.z, a.w); f[2] = make_float2(b.x, b.y); f[3] = make_float2(b.z, b.w);
}
FVB_DEVICE float2 bf16_round2(float2 v) {  // one cvt.rn.bf16x2 + two unpacks instead of two cvt + two shifts
  const uint32_t w = pack_bf16x2(v.x, v.y);
  return make_float2(__uint_as_float(w << 16), __uint_as_float(w & 0xffff0000u));
}

// tab_kind: 0 = per-column vectors come from global memory (through L1) for every row; 1 = the affine (w, b) pair, 2 = the
// modulation pair as (1 + scale, shift) sits in a shared-memory table after the row staging area, filled once per CTA. With
// the vectors read through L1, a 10 KB bf16 row dragged 40 KB of fp32 vectors behind it: the kernel ran at 3.1 TB/s, bound
// by the L1 pipe and the issue slots (LDG.128 x 4 + 20 scalar fp32 instructions per 8 elements), not by HBM.
template <bool IN_F32, bool ROUND_LN, bool MOD_BF16>
__global__ void __launch_bounds__(RW_WARPS * 32, 1)
layernorm_warp_kernel(const void* __restrict__ x_, int64_t ldx, const float* __restrict__ w, const float* __restrict__ b,
                      const float* __restrict__ scale0, const float* __restrict__ shift0, __nv_bfloat16* __restrict__ out,
                      int64_t ldo, __nv_bfloat16* __restrict__ hidden_out, int64_t ldh, int D, float eps, int mod_rows,
                      int64_t mod_stride, int M, int stages, int nw, int tab_kind) {
  extern __shared__ __align__(128) uint8_t rw_smem[];
  __shared__ uint64_t bars[RW_WARPS * RW_MAX_STAGES];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t row_bytes = uint32_t(D) * (IN_F32 ? 4u : 2u);
  float* tab = reinterpret_cast<float*>(rw_smem + size_t(nw) * stages * row_bytes);
  if (tab_kind != 0) {
    for (int i = threadIdx.x; i < D; i += blockDim.x) {
      if (tab_kind == 1) {
        tab[i] = w[i];
        tab[D + i] = b[i];
      } else {
        const float m = __fadd_rn(1.0f, scale0[i]);
        tab[i] = MOD_BF16 ? bf16_round(m) : m;
        tab[D + i] = shift0[i];
      }
    }
    __syncthreads();
  }
  if (warp >= nw) return;  // wide rows (fp32, D = 5120: 20 KB): fewer warps own a staging slot; no block-wide barrier follows
  uint8_t* my = rw_smem + size_t(warp) * stages * row_bytes;
  uint64_t* bar = bars + warp * RW_MAX_STAGES;
  const int64_t first = int64_t(blockIdx.x) * nw + warp, stride = int64_t(gridDim.x) * nw;
  auto row_src = [&](int64_t r) { return reinterpret_cast<const uint8_t*>(x_) + r * ldx * int64_t(IN_F32 ? 4 : 2); };
  if (lane == 0) {
    for (int s = 0; s < stages; ++s) mbar_init(&bar[s], 1);
    fence_mbar_init();
    for (int s = 0; s < stages; ++s) {
      const int64_t r = first + s * stride;
      if (r < M) {
        mbar_expect_tx(&bar[s], row_bytes);
        bulk_load_1d(my + s * row_bytes, row_src(r), row_bytes, &bar[s]);
      }
    }
  }
  __syncwarp();
  const int nchunks = D >> 3;
  const float inv_d = 1.0f / float(D);
  int it = 0;
  for (int64_t row = first; row < M; row += stride, ++it) {
    const int stg = it % stages;
    mbar_wait(&bar[stg], (it / stages) & 1);
    const uint8_t* srow = my + stg * row_bytes;
    const float* scale = scale0;
    const float* shift = shift0;
    if (mod_rows > 0 && scale0 != nullptr) {
      const int64_t g = (row / mod_rows) * mod_stride;
      scale += g;
      shift += g;
    }
    float2 s2 = make_float2(0.f, 0.f);
#pragma unroll 4
    for (int ch = lane; ch < nchunks; ch += 32) {
      float2 f[4];
      load8p<IN_F32>(srow, ch, f);
      s2 = add2(s2, add2(add2(f[0], f[1]), add2(f[2], f[3])));
    }
    const float mean = warp_sum(s2.x + s2.y) * inv_d;
    const float2 nmean2 = make_float2(-mean, -mean);
    float2 q2 = make_float2(0.f, 0.f);
#pragma unroll 4
    for (int ch = lane; ch < nchunks; ch += 32) {
      float2 f[4];
      load8p<IN_F32>(srow, ch, f);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float2 d = add2(f[i], nmean2);
        q2 = fma2(d, d, q2);
      }
    }
    const float rstd = rsqrtf(warp_sum(q2.x + q2.y) * inv_d + eps);
    const float2 rstd2 = make_float2(rstd, rstd);
#pragma unroll 4
    for (int ch = lane; ch < nchunks; ch += 32) {
      const int col = ch << 3;
      float2 f[4], m[4], a[4];
      load8p<IN_F32>(srow, ch, f);
      if (hidden_out != nullptr) {
        uint4 hv;
        hv.x = pack_bf16x2(f[0].x, f[0].y); hv.y = pack_bf16x2(f[1].x, f[1].y);
        hv.z = pack_bf16x2(f[2].x, f[2].y); hv.w = pack_bf16x2(f[3].x, f[3].y);
        reinterpret_cast<uint4*>(hidden_out + row * ldh)[ch] = hv;
      }
#pragma unroll
      for (int i = 0; i < 4; ++i) f[i] = mul2(add2(f[i], nmean2), rstd2);  // (x - mean) * rstd
      if (w != nullptr) {
        if (tab_kind == 1) {
          lds8p(tab + col, m);
          lds8p(tab + D + col, a);
        } else {
          ldg8p(w + col, m);
          ldg8p(b + col, a);
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) f[i] = add2(mul2(f[i], m[i]), a[i]);  // fp32 mul, then fp32 add (no fma: torch rounds both)
      }
      if constexpr (ROUND_LN) {
#pragma unroll
        for (int i = 0; i < 4; ++i) f[i] = bf16_round2(f[i]);
      }
      if (scale != nullptr) {
        if (tab_kind == 2) {
          lds8p(tab + col, m);
          lds8p(tab + D + col, a);
        } else {
          ldg8p(scale + col, m);
          ldg8p(shift + col, a);
          const float2 one2 = make_float2(1.0f, 1.0f);
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            m[i] = add2(one2, m[i]);
            if constexpr (MOD_BF16) m[i] = bf16_round2(m[i]);
          }
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          if constexpr (MOD_BF16) f[i] = bf16_round2(add2(bf16_round2(mul2(f[i], m[i])), a[i]));
          else f[i] = add2(mul2(f[i], m[i]), a[i]);
        }
      }
      uint4 ov;
      ov.x = pack_bf16x2(f[0].x, f[0].y); ov.y = pack_bf16x2(f[1].x, f[1].y);
      ov.z = pack_bf16x2(f[2].x, f[2].y); ov.w = pack_bf16x2(f[3].x, f[3].y);
      reinterpret_cast<uint4*>(out + row * ldo)[ch] = ov;
    }
    __syncwarp();  // every lane is done with the staged row: refill the stage
    if (lane == 0) {
      const int64_t nr = row + int64_t(stages) * stride;
      if (nr < M) {
        mbar_expect_tx(&bar[stg], row_bytes);
        bulk_load_1d(my + stg * row_bytes, row_src(nr), row_bytes, &bar[stg]);
      }
    }
  }
}

template <bool ROPE_F64>
__global__ void __launch_bounds__(RW_WARPS * 32, 1)
rmsnorm_rope_warp_kernel(RmsRopeArgs a, const void* __restrict__ cos_v, const void* __restrict__ sin_v,
                         const int32_t* __restrict__ rope_row, int D, int head_dim, float eps, int M, int stages, int w_tab) {
  extern __shared__ __align__(128) uint8_t rw_smem[];
  __shared__ uint64_t bars[RW_WARPS * RW_MAX_STAGES];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int which = blockIdx.y;
  __nv_bfloat16* const xbase = which ? a.x[1] : a.x[0];
  const int64_t xld = which ? a.ld[1] : a.ld[0];
  const __nv_bfloat16* w = which ? a.w[1] : a.w[0];
  const uint32_t row_bytes = uint32_t(D) * 2u;
  // w_tab: the norm weight as fp32 in shared memory after the staging area (filled once per CTA) instead of a 10-20 KB
  // trip through L1 behind every 10 KB row
  float* wtab = reinterpret_cast<float*>(rw_smem + size_t(RW_WARPS) * stages * row_bytes);
  if (w_tab != 0 && w != nullptr) {
    for (int i = threadIdx.x; i < D; i += blockDim.x)
      wtab[i] = a.w_f32 ? reinterpret_cast<const float*>(w)[i] : __bfloat162float(w[i]);
    __syncthreads();
  }
  uint8_t* my = rw_smem + size_t(warp) * stages * row_bytes;
  uint64_t* bar = bars + warp * RW_MAX_STAGES;
  const int64_t first = int64_t(blockIdx.x) * RW_WARPS + warp, stride = int64_t(gridDim.x) * RW_WARPS;
  // Stage one row. Contiguous rows: one bulk copy. Head-scattered rows (the sequence-parallel send buffer, see
  // fvb_linear_bf16_sp): one 256-byte bulk copy per head, issued by the lanes in parallel onto the same barrier.
  auto stage_row = [&](int s, int64_t r) {
    if (a.col_offsets == nullptr) {
      if (lane == 0) {
        mbar_expect_tx(&bar[s], row_bytes);
        bulk_load_1d(my + s * row_bytes, xbase + r * xld, row_bytes, &bar[s]);
      }
    } else {
      if (lane == 0) mbar_expect_tx(&bar[s], row_bytes);
      __syncwarp();
      for (int j = lane; j < (D >> 7); j += 32)
        bulk_load_1d(my + s * row_bytes + j * 256, xbase + r * xld + __ldg(a.col_offsets + j), 256, &bar[s]);
    }
  };
  if (lane == 0) {
    for (int s = 0; s < stages; ++s) mbar_init(&bar[s], 1);
    fence_mbar_init();
  }
  __syncwarp();
  for (int s = 0; s < stages; ++s) {
    const int64_t r = first + s * stride;
    if (r < M) stage_row(s, r);
  }
  __syncwarp();
  const int nchunks = D >> 3;
  const float inv_d = 1.0f / float(D);
  int it = 0;
  for (int64_t row = first; row < M; row += stride, ++it) {
    const int stg = it % stages;
    mbar_wait(&bar[stg], (it / stages) & 1);
    const uint8_t* srow = my + stg * row_bytes;
    __nv_bfloat16* const ybase = which ? a.y[1] : a.y[0];
    __nv_bfloat16* xr = ybase ? ybase + row * a.ldy : xbase + row * xld;
    const int64_t* out_off = ybase ? a.out_col_offsets : a.col_offsets;
    if (w == nullptr && cos_v == nullptr) {  // copy mode (v / gate rows of the sequence-parallel push): no statistics, no weight, no RoPE
#pragma unroll 4
      for (int ch = lane; ch < nchunks; ch += 32) {
        const int64_t eoff = out_off ? __ldg(out_off + (ch >> 4)) + ((ch & 15) << 3) : int64_t(ch) << 3;
        *reinterpret_cast<uint4*>(xr + eoff) = reinterpret_cast<const uint4*>(srow)[ch];
      }
      __syncwarp();
      const int64_t nr = row + int64_t(stages) * stride;
      if (nr < M) stage_row(stg, nr);
      continue;
    }
    // w == NULL with tables: RoPE only -- the row is already normalised (un-roped keys of the "relativistic" KV-cache
    // policy, causal_wanvideo.py:140, 174-181, are roped again from position 0 on every call)
    const bool has_w = w != nullptr;
    float rstd = 1.0f;
    if (has_w) {
      float2 s2 = make_float2(0.f, 0.f);
#pragma unroll 4
      for (int ch = lane; ch < nchunks; ch += 32) {
        float2 f[4];
        load8p<false>(srow, ch, f);
#pragma unroll
        for (int i = 0; i < 4; ++i) s2 = fma2(f[i], f[i], s2);
      }
      rstd = rsqrtf(warp_sum(s2.x + s2.y) * inv_d + eps);
    }
    const float2 rstd2 = make_float2(rstd, rstd);
    const int64_t prow = (rope_row != nullptr) ? int64_t(rope_row[row]) : row;
    // fp32 tables, head_dim | 256: every chunk of a lane (columns 8 lane + 256 j) sits at the same offset inside its head, so
    // the lane's eight cos / sin values are loaded once per row, not once per chunk (40 KB through L1 per 10 KB row before)
    const bool rope32 = !ROPE_F64 && cos_v != nullptr;
    const bool cs_row = rope32 && (256 % head_dim) == 0;
    float2 cs[4], sn[4];
    if (cs_row) {
      const int hc = (lane << 3) % head_dim;
      ldg8p(reinterpret_cast<const float*>(cos_v) + prow * head_dim + hc, cs);
      ldg8p(reinterpret_cast<const float*>(sin_v) + prow * head_dim + hc, sn);
    }
#pragma unroll 4
    for (int ch = lane; ch < nchunks; ch += 32) {
      const int col = ch << 3;
      float2 n[4];
      load8p<false>(srow, ch, n);
      if (has_w) {
        float2 wv[4];
        if (w_tab != 0) lds8p(wtab + col, wv);
        else if (a.w_f32) ldg8p(reinterpret_cast<const float*>(w) + col, wv);
        else {
          float t[8];
          unpack8(__ldg(reinterpret_cast<const uint4*>(w) + ch), t);
#pragma unroll
          for (int i = 0; i < 4; ++i) wv[i] = make_float2(t[2 * i], t[2 * i + 1]);
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          n[i] = mul2(bf16_round2(mul2(n[i], rstd2)), wv[i]);
          if (!a.w_f32) n[i] = bf16_round2(n[i]);  // bf16 weights: the product is a bf16 tensor; fp32 weights: rounded once, at the store
        }
      }
      float2 y[4];
      if constexpr (ROPE_F64) {
        const int hc = col % head_dim;
        const double2* cp = reinterpret_cast<const double2*>(reinterpret_cast<const double*>(cos_v) + prow * head_dim + hc);
        const double2* sp = reinterpret_cast<const double2*>(reinterpret_cast<const double*>(sin_v) + prow * head_dim + hc);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const double2 c = __ldg(cp + i), sv = __ldg(sp + i);
          y[i].x = __double2float_rn(__dadd_rn(__dmul_rn(double(n[i].x), c.x), __dmul_rn(double(-n[i].y), sv.x)));
          y[i].y = __double2float_rn(__dadd_rn(__dmul_rn(double(n[i].y), c.y), __dmul_rn(double(n[i].x), sv.y)));
        }
      } else if (rope32) {
        if (!cs_row) {
          const int hc = col % head_dim;  // 8 | head_dim, so a chunk never straddles heads
          ldg8p(reinterpret_cast<const float*>(cos_v) + prow * head_dim + hc, cs);
          ldg8p(reinterpret_cast<const float*>(sin_v) + prow * head_dim + hc, sn);
        }
#pragma unroll
        for (int i = 0; i < 4; ++i)  // (n0 c0 + (-n1) s0, n1 c1 + n0 s1): both products rounded, then the sum
          y[i] = add2(mul2(n[i], cs[i]), mul2(make_float2(-n[i].y, n[i].x), sn[i]));
      } else {
#pragma unroll
        for (int i = 0; i < 4; ++i) y[i] = n[i];
      }
      const int64_t eoff = out_off ? __ldg(out_off + (ch >> 4)) + ((ch & 15) << 3) : int64_t(ch) << 3;
      uint4 ov;
      ov.x = pack_bf16x2(y[0].x, y[0].y); ov.y = pack_bf16x2(y[1].x, y[1].y);
      ov.z = pack_bf16x2(y[2].x, y[2].y); ov.w = pack_bf16x2(y[3].x, y[3].y);
      *reinterpret_cast<uint4*>(xr + eoff) = ov;
    }
    __syncwarp();
    {
      const int64_t nr = row + int64_t(stages) * stride;
      if (nr < M) stage_row(stg, nr);
    }
  }
}

static int rw_stages(int row_bytes) {
  return std::max(1, std::min(RW_MAX_STAGES, RW_SMEM_BUDGET / (RW_WARPS * row_bytes)));
}

// ------------------------------------------------------------------------------------------
// RMSNorm backward (fvb_rmsnorm_bwd; arithmetic in include/fvb200.h). Block per row, rows blockIdx.x + k * gridDim.x, the
// row in registers between the statistics pass and the write. Each thread keeps the fp32 dw partial of its own columns
// across its CTA's rows; the partials are summed over CTAs in CTA order by rmsnorm_bwd_dw_kernel (no atomics).
// ------------------------------------------------------------------------------------------
constexpr int RB_CTAS = 528;  // fixed (not per device), so dw's summation order is the same on every GPU

FVB_DEVICE float2 block_sum2(float2 v, float2* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    v.x += __shfl_xor_sync(0xffffffffu, v.x, o);
    v.y += __shfl_xor_sync(0xffffffffu, v.y, o);
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();  // protect `red` from the previous use
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float2 t = (lane < EW_THREADS / 32) ? red[lane] : make_float2(0.f, 0.f);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    t.x += __shfl_xor_sync(0xffffffffu, t.x, o);
    t.y += __shfl_xor_sync(0xffffffffu, t.y, o);
  }
  return t;
}

// ROPE (fvb_rmsnorm_rope_bwd): dy is the gradient of the rotated output; each row is first un-rotated with the forward's
// table row, dn = bf16(R^T dy) per interleaved pair, and dn takes dy's place below.
template <bool ROPE>
FVB_DEVICE void rmsnorm_bwd_body(const __nv_bfloat16* __restrict__ x, int64_t ldx,
                                                 const __nv_bfloat16* __restrict__ w,
                                                 const __nv_bfloat16* __restrict__ dy, int64_t lddy,
                                                 __nv_bfloat16* __restrict__ dx, int64_t lddx,
                                                 float* __restrict__ dw_part, int M, int D, float eps,
                                                 const float* __restrict__ cos_t, const float* __restrict__ sin_t,
                                                 const int32_t* __restrict__ rope_row, int head_dim) {
  __shared__ float2 red[32];
  const int nchunks = D >> 3;
  float acc[EW_MAX_CHUNKS][8];
#pragma unroll
  for (int c = 0; c < EW_MAX_CHUNKS; ++c)
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[c][i] = 0.f;
  for (int64_t row = blockIdx.x; row < M; row += gridDim.x) {
    float xv[EW_MAX_CHUNKS][8], dv[EW_MAX_CHUNKS][8];
    float2 s = make_float2(0.f, 0.f);  // (sum x^2, sum g x)
#pragma unroll
    for (int c = 0; c < EW_MAX_CHUNKS; ++c) {
      const int ch = threadIdx.x + c * EW_THREADS;
      if (ch < nchunks) {
        unpack8(*reinterpret_cast<const uint4*>(x + row * ldx + (ch << 3)), xv[c]);
        unpack8(*reinterpret_cast<const uint4*>(dy + row * lddy + (ch << 3)), dv[c]);
        if constexpr (ROPE) {
          // forward: o[2i] = n[2i] c[2i] - n[2i+1] s[2i], o[2i+1] = n[2i+1] c[2i+1] + n[2i] s[2i+1]
          const int64_t prow = rope_row != nullptr ? int64_t(rope_row[row]) : row;
          float cs[8], sn[8];
          load8_f32(cos_t + prow * head_dim + (ch << 3) % head_dim, cs);
          load8_f32(sin_t + prow * head_dim + (ch << 3) % head_dim, sn);
#pragma unroll
          for (int i = 0; i < 8; i += 2) {
            const float g0 = dv[c][i], g1 = dv[c][i + 1];
            dv[c][i] = bf16_round(__fadd_rn(__fmul_rn(g0, cs[i]), __fmul_rn(g1, sn[i + 1])));
            dv[c][i + 1] = bf16_round(__fsub_rn(__fmul_rn(g1, cs[i + 1]), __fmul_rn(g0, sn[i])));
          }
        }
        float wv[8];
        if (w != nullptr) unpack8(__ldg(reinterpret_cast<const uint4*>(w) + ch), wv);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float g = w != nullptr ? bf16_round(__fmul_rn(dv[c][i], wv[i])) : dv[c][i];
          s.x = __fmaf_rn(xv[c][i], xv[c][i], s.x);
          s.y = __fmaf_rn(g, xv[c][i], s.y);
        }
      }
    }
    s = block_sum2(s, red);
    const float r = rsqrtf(__fdiv_rn(s.x, float(D)) + eps);
    const float k = __fdiv_rn(__fmul_rn(r, s.y), float(D));  // sum_c (g x^) / D
#pragma unroll
    for (int c = 0; c < EW_MAX_CHUNKS; ++c) {
      const int ch = threadIdx.x + c * EW_THREADS;
      if (ch < nchunks) {
        float wv[8], o[8];
        if (w != nullptr) unpack8(__ldg(reinterpret_cast<const uint4*>(w) + ch), wv);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float g = w != nullptr ? bf16_round(__fmul_rn(dv[c][i], wv[i])) : dv[c][i];
          const float xh = __fmul_rn(xv[c][i], r);
          o[i] = __fmul_rn(r, __fsub_rn(g, __fmul_rn(xh, k)));
          acc[c][i] = __fmaf_rn(dv[c][i], bf16_round(xh), acc[c][i]);
        }
        *reinterpret_cast<uint4*>(dx + row * lddx + (ch << 3)) = pack8(o);
      }
    }
  }
  if (dw_part == nullptr) return;
#pragma unroll
  for (int c = 0; c < EW_MAX_CHUNKS; ++c) {
    const int ch = threadIdx.x + c * EW_THREADS;
    if (ch < nchunks) {
      float4* dst = reinterpret_cast<float4*>(dw_part + int64_t(blockIdx.x) * D + (ch << 3));
      dst[0] = make_float4(acc[c][0], acc[c][1], acc[c][2], acc[c][3]);
      dst[1] = make_float4(acc[c][4], acc[c][5], acc[c][6], acc[c][7]);
    }
  }
}

__global__ void __launch_bounds__(EW_THREADS) rmsnorm_bwd_kernel(const __nv_bfloat16* __restrict__ x, int64_t ldx,
                                                                 const __nv_bfloat16* __restrict__ w,
                                                                 const __nv_bfloat16* __restrict__ dy, int64_t lddy,
                                                                 __nv_bfloat16* __restrict__ dx, int64_t lddx,
                                                                 float* __restrict__ dw_part, int M, int D, float eps) {
  rmsnorm_bwd_body<false>(x, ldx, w, dy, lddy, dx, lddx, dw_part, M, D, eps, nullptr, nullptr, nullptr, 0);
}

// Up to two tensors (q and k) per launch, blockIdx.y selects; tensor t's dw partials go to dw_part + t * gridDim.x * D.
struct RmsRopeBwdArgs {
  const __nv_bfloat16* x[2];
  const __nv_bfloat16* w[2];
  const __nv_bfloat16* dy[2];
  __nv_bfloat16* dx[2];
  int64_t ldx[2], lddy[2], lddx[2];
};

__global__ void __launch_bounds__(EW_THREADS) rmsnorm_rope_bwd_kernel(RmsRopeBwdArgs a, float* __restrict__ dw_part,
                                                                      const float* __restrict__ cos_t,
                                                                      const float* __restrict__ sin_t,
                                                                      const int32_t* __restrict__ rope_row, int M, int D,
                                                                      int head_dim, float eps) {
  // fields selected with ternaries, not indexed by blockIdx.y: a dynamic index would copy the arrays to local memory
  const bool t = blockIdx.y != 0;
  rmsnorm_bwd_body<true>(t ? a.x[1] : a.x[0], t ? a.ldx[1] : a.ldx[0], t ? a.w[1] : a.w[0], t ? a.dy[1] : a.dy[0],
                         t ? a.lddy[1] : a.lddy[0], t ? a.dx[1] : a.dx[0], t ? a.lddx[1] : a.lddx[0],
                         dw_part != nullptr ? dw_part + int64_t(blockIdx.y) * gridDim.x * D : nullptr, M, D, eps, cos_t,
                         sin_t, rope_row, head_dim);
}

__global__ void __launch_bounds__(256) rmsnorm_bwd_dw_kernel(const float* __restrict__ dw_part, int nparts, int D,
                                                              __nv_bfloat16* __restrict__ dw) {
  const int col = blockIdx.x * 256 + threadIdx.x;
  if (col >= D) return;
  float s = 0.f;
  for (int i = 0; i < nparts; ++i) s = __fadd_rn(s, __ldg(dw_part + int64_t(i) * D + col));
  dw[col] = __float2bfloat16_rn(s);
}

// ------------------------------------------------------------------------------------------
// Bias gradient of the bf16 linear (fvb_bias_grad_bf16): db[n] = bf16(sum_m dy[m, n]). blockIdx.y picks 1024 columns
// (8 per thread), blockIdx.x one of BG_PARTS fixed row sets (rows part, part + BG_PARTS, ...), summed in row order into
// fp32 partials; rmsnorm_bwd_dw_kernel then adds the partials in part order and rounds once. No atomics: the summation
// order depends on M and N only.
// ------------------------------------------------------------------------------------------
constexpr int BG_PARTS = 256;  // fixed (not per device), so db's summation order is the same on every GPU
constexpr int BG_THREADS = 128;
constexpr int BG_UNROLL = 8;  // row loads in flight per thread

__global__ void __launch_bounds__(BG_THREADS) bias_grad_kernel(const __nv_bfloat16* __restrict__ dy, int64_t lddy,
                                                               float* __restrict__ part, int M, int N, int nparts) {
  const int col = (blockIdx.y * BG_THREADS + threadIdx.x) * 8;
  if (col >= N) return;
  float acc[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i] = 0.f;
  const int64_t step = int64_t(nparts) * lddy;
  const __nv_bfloat16* p = dy + int64_t(blockIdx.x) * lddy + col;
  int row = blockIdx.x;
  for (; row + (BG_UNROLL - 1) * nparts < M; row += BG_UNROLL * nparts) {
    uint4 v[BG_UNROLL];
#pragma unroll
    for (int u = 0; u < BG_UNROLL; ++u) v[u] = __ldg(reinterpret_cast<const uint4*>(p + u * step));
    p += BG_UNROLL * step;
#pragma unroll
    for (int u = 0; u < BG_UNROLL; ++u) {
      float f[8];
      unpack8(v[u], f);
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] = __fadd_rn(acc[i], f[i]);
    }
  }
  for (; row < M; row += nparts, p += step) {
    float f[8];
    unpack8(__ldg(reinterpret_cast<const uint4*>(p)), f);
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = __fadd_rn(acc[i], f[i]);
  }
  float4* dst = reinterpret_cast<float4*>(part + int64_t(blockIdx.x) * N + col);
  dst[0] = make_float4(acc[0], acc[1], acc[2], acc[3]);
  dst[1] = make_float4(acc[4], acc[5], acc[6], acc[7]);
}

// fp32 column sums of per-part partials, added in part order (the fp32 twin of rmsnorm_bwd_dw_kernel)
__global__ void __launch_bounds__(256) colsum_f32_kernel(const float* __restrict__ part, int nparts, int N, float* __restrict__ out) {
  const int col = blockIdx.x * 256 + threadIdx.x;
  if (col >= N) return;
  float s = 0.f;
  for (int i = 0; i < nparts; ++i) s = __fadd_rn(s, __ldg(part + int64_t(i) * N + col));
  out[col] = s;
}

// ------------------------------------------------------------------------------------------
// Gated-residual backward (fvb_resid_gate_bwd; arithmetic in include/fvb200.h). The layout of bias_grad_kernel: blockIdx.y
// picks 1024 columns (8 per thread), blockIdx.x one of BG_PARTS fixed row sets; the fp32 partials of sum dout * y (d_gate)
// and of sum dy (bias grad) go to part[0][part][N] and part[1][part][N].
// ------------------------------------------------------------------------------------------
template <bool DOUT_F32>
__global__ void __launch_bounds__(BG_THREADS) resid_gate_bwd_kernel(const void* __restrict__ dout_, int64_t lddout,
                                                                    const __nv_bfloat16* __restrict__ y, int64_t ldy,
                                                                    const float* __restrict__ gate,
                                                                    __nv_bfloat16* __restrict__ dy, int64_t lddy,
                                                                    float* __restrict__ part, int M, int N, int nparts) {
  const int col = (blockIdx.y * BG_THREADS + threadIdx.x) * 8;
  if (col >= N) return;
  float g[8], ag[8], ab[8];
  load8_f32(gate + col, g);
#pragma unroll
  for (int i = 0; i < 8; ++i) ag[i] = ab[i] = 0.f;
  for (int64_t row = blockIdx.x; row < M; row += nparts) {
    float d[8], yv[8], o[8];
    if constexpr (DOUT_F32) {
      const float4* p = reinterpret_cast<const float4*>(reinterpret_cast<const float*>(dout_) + row * lddout + col);
      const float4 a = p[0], b = p[1];
      d[0] = a.x; d[1] = a.y; d[2] = a.z; d[3] = a.w; d[4] = b.x; d[5] = b.y; d[6] = b.z; d[7] = b.w;
    } else {
      unpack8(*reinterpret_cast<const uint4*>(reinterpret_cast<const __nv_bfloat16*>(dout_) + row * lddout + col), d);
    }
    unpack8(*reinterpret_cast<const uint4*>(y + row * ldy + col), yv);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      o[i] = bf16_round(__fmul_rn(d[i], g[i]));
      ag[i] = __fmaf_rn(d[i], yv[i], ag[i]);
      ab[i] = __fadd_rn(ab[i], o[i]);
    }
    *reinterpret_cast<uint4*>(dy + row * lddy + col) = pack8(o);
  }
  float4* dg = reinterpret_cast<float4*>(part + int64_t(blockIdx.x) * N + col);
  float4* db = reinterpret_cast<float4*>(part + (int64_t(nparts) + blockIdx.x) * N + col);
  dg[0] = make_float4(ag[0], ag[1], ag[2], ag[3]);
  dg[1] = make_float4(ag[4], ag[5], ag[6], ag[7]);
  db[0] = make_float4(ab[0], ab[1], ab[2], ab[3]);
  db[1] = make_float4(ab[4], ab[5], ab[6], ab[7]);
}

// ------------------------------------------------------------------------------------------
// LayerNorm + modulation backward (fvb_layernorm_modulate_bwd; arithmetic in include/fvb200.h). The structure of
// rmsnorm_bwd_kernel: block per row over fixed row sets, the row in registers, mean / variance recomputed from x as the
// forward does; each thread keeps the fp32 partials sum dn * t and sum dn of its own columns, written to
// part[0][cta][D] and part[1][cta][D] and added in CTA order by colsum_f32_kernel.
// ------------------------------------------------------------------------------------------
template <bool IN_F32, bool GIN_F32>
__global__ void __launch_bounds__(EW_THREADS) layernorm_modulate_bwd_kernel(
    const void* __restrict__ x_, int64_t ldx, const __nv_bfloat16* __restrict__ dn, int64_t lddn,
    const float* __restrict__ gain, int gain_is_scale, int round_ln, const void* __restrict__ gin_, int64_t ldgin,
    void* __restrict__ dx_, int64_t lddx, float* __restrict__ part, int M, int D, float eps) {
  __shared__ float red[32];
  __shared__ float2 red2[32];
  const int nchunks = D >> 3;
  float as[EW_MAX_CHUNKS][8], ah[EW_MAX_CHUNKS][8];
#pragma unroll
  for (int c = 0; c < EW_MAX_CHUNKS; ++c)
#pragma unroll
    for (int i = 0; i < 8; ++i) as[c][i] = ah[c][i] = 0.f;
  for (int64_t row = blockIdx.x; row < M; row += gridDim.x) {
    float xv[EW_MAX_CHUNKS][8], dv[EW_MAX_CHUNKS][8];
    float s = 0.f;
#pragma unroll
    for (int c = 0; c < EW_MAX_CHUNKS; ++c) {
      const int ch = threadIdx.x + c * EW_THREADS;
      if (ch < nchunks) {
        if constexpr (IN_F32) {
          load8_f32(reinterpret_cast<const float*>(x_) + row * ldx + (ch << 3), xv[c]);
        } else {
          unpack8(*reinterpret_cast<const uint4*>(reinterpret_cast<const __nv_bfloat16*>(x_) + row * ldx + (ch << 3)), xv[c]);
        }
        unpack8(*reinterpret_cast<const uint4*>(dn + row * lddn + (ch << 3)), dv[c]);
#pragma unroll
        for (int i = 0; i < 8; ++i) s += xv[c][i];
      }
    }
    const float mean = block_sum(s, red) / float(D);
    float q = 0.f;
#pragma unroll
    for (int c = 0; c < EW_MAX_CHUNKS; ++c) {
      const int ch = threadIdx.x + c * EW_THREADS;
      if (ch < nchunks)
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float d = xv[c][i] - mean;
          q += d * d;
        }
    }
    const float rstd = rsqrtf(block_sum(q, red) / float(D) + eps);
    float2 st = make_float2(0.f, 0.f);  // (sum dt, sum dt * xhat)
#pragma unroll
    for (int c = 0; c < EW_MAX_CHUNKS; ++c) {
      const int ch = threadIdx.x + c * EW_THREADS;
      if (ch < nchunks) {
        float gv[8];
        load8_f32(gain + (ch << 3), gv);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float xh = (xv[c][i] - mean) * rstd;  // the forward's t
          xv[c][i] = xh;
          const float dt = __fmul_rn(dv[c][i], gain_is_scale ? __fadd_rn(1.0f, gv[i]) : gv[i]);
          st.x += dt;
          st.y = __fmaf_rn(dt, xh, st.y);
          as[c][i] = __fmaf_rn(dv[c][i], round_ln ? bf16_round(xh) : xh, as[c][i]);
          ah[c][i] = __fadd_rn(ah[c][i], dv[c][i]);
        }
      }
    }
    st = block_sum2(st, red2);
    const float mdt = __fdiv_rn(st.x, float(D)), mdx = __fdiv_rn(st.y, float(D));
#pragma unroll
    for (int c = 0; c < EW_MAX_CHUNKS; ++c) {
      const int ch = threadIdx.x + c * EW_THREADS;
      if (ch < nchunks) {
        float gv[8], o[8], gi[8];
        load8_f32(gain + (ch << 3), gv);
        if (gin_ != nullptr) {
          if constexpr (GIN_F32)
            load8_f32(reinterpret_cast<const float*>(gin_) + row * ldgin + (ch << 3), gi);
          else
            unpack8(*reinterpret_cast<const uint4*>(reinterpret_cast<const __nv_bfloat16*>(gin_) + row * ldgin + (ch << 3)), gi);
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float dt = __fmul_rn(dv[c][i], gain_is_scale ? __fadd_rn(1.0f, gv[i]) : gv[i]);
          o[i] = __fmul_rn(rstd, __fsub_rn(__fsub_rn(dt, mdt), __fmul_rn(xv[c][i], mdx)));
          if (gin_ != nullptr) o[i] = __fadd_rn(o[i], gi[i]);
        }
        if constexpr (IN_F32) {
          float4* dst = reinterpret_cast<float4*>(reinterpret_cast<float*>(dx_) + row * lddx + (ch << 3));
          dst[0] = make_float4(o[0], o[1], o[2], o[3]);
          dst[1] = make_float4(o[4], o[5], o[6], o[7]);
        } else {
          *reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(dx_) + row * lddx + (ch << 3)) = pack8(o);
        }
      }
    }
  }
#pragma unroll
  for (int c = 0; c < EW_MAX_CHUNKS; ++c) {
    const int ch = threadIdx.x + c * EW_THREADS;
    if (ch < nchunks) {
      float4* ds = reinterpret_cast<float4*>(part + int64_t(blockIdx.x) * D + (ch << 3));
      float4* dh = reinterpret_cast<float4*>(part + (int64_t(gridDim.x) + blockIdx.x) * D + (ch << 3));
      ds[0] = make_float4(as[c][0], as[c][1], as[c][2], as[c][3]);
      ds[1] = make_float4(as[c][4], as[c][5], as[c][6], as[c][7]);
      dh[0] = make_float4(ah[c][0], ah[c][1], ah[c][2], ah[c][3]);
      dh[1] = make_float4(ah[c][4], ah[c][5], ah[c][6], ah[c][7]);
    }
  }
}

// ------------------------------------------------------------------------------------------
// Per-row-group (per latent frame) backward of the bf16 modulation flow (fvb_layernorm_modulate_grouped_bwd,
// fvb_resid_gate_grouped_bwd; arithmetic in include/fvb200.h). Group g = rows [g R, min((g + 1) R, M)); `parts` CTAs per
// group, CTA (g, p) = blockIdx.x = g * parts + p takes the group's rows p, p + parts, ... in row order, and writes its
// fp32 column partials to part[blockIdx.x]. grouped_colsum_kernel adds a group's partials in p order: no atomics, the
// summation order depends on (M, R, D) only.
// ------------------------------------------------------------------------------------------
static inline int grouped_parts(int M, int R, int budget) {
  const int G = (M + R - 1) / R;
  const int p = budget / G;
  return p < 1 ? 1 : (p > R ? R : p);
}

template <bool GIN_F32>
__global__ void __launch_bounds__(EW_THREADS) layernorm_modulate_grouped_bwd_kernel(
    const __nv_bfloat16* __restrict__ x, int64_t ldx, const __nv_bfloat16* __restrict__ dn, int64_t lddn,
    const float* __restrict__ scale, int mod_rows, int64_t mod_stride, const void* __restrict__ gin_, int64_t ldgin,
    __nv_bfloat16* __restrict__ dx, int64_t lddx, float* __restrict__ part, int M, int D, float eps, int parts) {
  __shared__ float red[32];
  __shared__ float2 red2[32];
  const int g = blockIdx.x / parts, p = blockIdx.x - g * parts;
  const int64_t r1 = min(int64_t(g + 1) * mod_rows, int64_t(M));
  scale += int64_t(g) * mod_stride;
  const int nchunks = D >> 3;
  float as[EW_MAX_CHUNKS][8], ah[EW_MAX_CHUNKS][8];
#pragma unroll
  for (int c = 0; c < EW_MAX_CHUNKS; ++c)
#pragma unroll
    for (int i = 0; i < 8; ++i) as[c][i] = ah[c][i] = 0.f;
  for (int64_t row = int64_t(g) * mod_rows + p; row < r1; row += parts) {
    float xv[EW_MAX_CHUNKS][8], dv[EW_MAX_CHUNKS][8];
    float s = 0.f;
#pragma unroll
    for (int c = 0; c < EW_MAX_CHUNKS; ++c) {
      const int ch = threadIdx.x + c * EW_THREADS;
      if (ch < nchunks) {
        unpack8(*reinterpret_cast<const uint4*>(x + row * ldx + (ch << 3)), xv[c]);
        unpack8(*reinterpret_cast<const uint4*>(dn + row * lddn + (ch << 3)), dv[c]);
#pragma unroll
        for (int i = 0; i < 8; ++i) s += xv[c][i];
      }
    }
    const float mean = block_sum(s, red) / float(D);
    float q = 0.f;
#pragma unroll
    for (int c = 0; c < EW_MAX_CHUNKS; ++c) {
      const int ch = threadIdx.x + c * EW_THREADS;
      if (ch < nchunks)
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float d = xv[c][i] - mean;
          q += d * d;
        }
    }
    const float rstd = rsqrtf(block_sum(q, red) / float(D) + eps);
    float2 st = make_float2(0.f, 0.f);  // (sum dt, sum dt * xhat)
#pragma unroll
    for (int c = 0; c < EW_MAX_CHUNKS; ++c) {
      const int ch = threadIdx.x + c * EW_THREADS;
      if (ch < nchunks) {
        float sc[8];
        load8_f32(scale + (ch << 3), sc);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float xh = (xv[c][i] - mean) * rstd;  // the forward's LN output before its bf16 rounding
          xv[c][i] = xh;
          // dv becomes dt = bf16(dn * bf16(1 + scale)) once dn has gone into the group sums
          as[c][i] = __fmaf_rn(dv[c][i], bf16_round(xh), as[c][i]);
          ah[c][i] = __fadd_rn(ah[c][i], dv[c][i]);
          dv[c][i] = bf16_round(__fmul_rn(dv[c][i], bf16_round(__fadd_rn(1.0f, sc[i]))));
          st.x += dv[c][i];
          st.y = __fmaf_rn(dv[c][i], xh, st.y);
        }
      }
    }
    st = block_sum2(st, red2);
    const float mdt = __fdiv_rn(st.x, float(D)), mdx = __fdiv_rn(st.y, float(D));
#pragma unroll
    for (int c = 0; c < EW_MAX_CHUNKS; ++c) {
      const int ch = threadIdx.x + c * EW_THREADS;
      if (ch < nchunks) {
        float o[8], gi[8];
        if (gin_ != nullptr) {
          if constexpr (GIN_F32)
            load8_f32(reinterpret_cast<const float*>(gin_) + row * ldgin + (ch << 3), gi);
          else
            unpack8(*reinterpret_cast<const uint4*>(reinterpret_cast<const __nv_bfloat16*>(gin_) + row * ldgin + (ch << 3)), gi);
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          o[i] = __fmul_rn(rstd, __fsub_rn(__fsub_rn(dv[c][i], mdt), __fmul_rn(xv[c][i], mdx)));
          if (gin_ != nullptr) o[i] = __fadd_rn(o[i], gi[i]);
        }
        *reinterpret_cast<uint4*>(dx + row * lddx + (ch << 3)) = pack8(o);
      }
    }
  }
  const int64_t nblk = gridDim.x;
#pragma unroll
  for (int c = 0; c < EW_MAX_CHUNKS; ++c) {
    const int ch = threadIdx.x + c * EW_THREADS;
    if (ch < nchunks) {
      float4* ds = reinterpret_cast<float4*>(part + int64_t(blockIdx.x) * D + (ch << 3));
      float4* dh = reinterpret_cast<float4*>(part + (nblk + blockIdx.x) * D + (ch << 3));
      ds[0] = make_float4(as[c][0], as[c][1], as[c][2], as[c][3]);
      ds[1] = make_float4(as[c][4], as[c][5], as[c][6], as[c][7]);
      dh[0] = make_float4(ah[c][0], ah[c][1], ah[c][2], ah[c][3]);
      dh[1] = make_float4(ah[c][4], ah[c][5], ah[c][6], ah[c][7]);
    }
  }
}

// The layout of resid_gate_bwd_kernel (blockIdx.y picks 1024 columns, 8 per thread) with blockIdx.x = g * parts + p as above.
__global__ void __launch_bounds__(BG_THREADS) resid_gate_grouped_bwd_kernel(
    const __nv_bfloat16* __restrict__ dout, int64_t lddout, const __nv_bfloat16* __restrict__ y, int64_t ldy,
    const float* __restrict__ gate, int gate_rows, int64_t gate_stride, __nv_bfloat16* __restrict__ dy, int64_t lddy,
    float* __restrict__ part, int M, int N, int parts) {
  const int col = (blockIdx.y * BG_THREADS + threadIdx.x) * 8;
  if (col >= N) return;
  const int g = blockIdx.x / parts, p = blockIdx.x - g * parts;
  const int64_t r1 = min(int64_t(g + 1) * gate_rows, int64_t(M));
  float gv[8], ag[8], ab[8];
  load8_f32(gate + int64_t(g) * gate_stride + col, gv);
#pragma unroll
  for (int i = 0; i < 8; ++i) ag[i] = ab[i] = 0.f;
  for (int64_t row = int64_t(g) * gate_rows + p; row < r1; row += parts) {
    float d[8], yv[8], o[8];
    unpack8(*reinterpret_cast<const uint4*>(dout + row * lddout + col), d);
    unpack8(*reinterpret_cast<const uint4*>(y + row * ldy + col), yv);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      o[i] = bf16_round(__fmul_rn(d[i], gv[i]));
      ag[i] = __fmaf_rn(d[i], yv[i], ag[i]);
      ab[i] = __fadd_rn(ab[i], o[i]);
    }
    *reinterpret_cast<uint4*>(dy + row * lddy + col) = pack8(o);
  }
  float4* dg = reinterpret_cast<float4*>(part + int64_t(blockIdx.x) * N + col);
  float4* db = reinterpret_cast<float4*>(part + (int64_t(gridDim.x) + blockIdx.x) * N + col);
  dg[0] = make_float4(ag[0], ag[1], ag[2], ag[3]);
  dg[1] = make_float4(ag[4], ag[5], ag[6], ag[7]);
  db[0] = make_float4(ab[0], ab[1], ab[2], ab[3]);
  db[1] = make_float4(ab[4], ab[5], ab[6], ab[7]);
}

// out[g * ldo + col] = sum over p (in order) of part[(g * parts + p) * N + col]; blockIdx.y = g
__global__ void __launch_bounds__(256) grouped_colsum_kernel(const float* __restrict__ part, int parts, int N,
                                                             float* __restrict__ out, int64_t ldo) {
  const int col = blockIdx.x * 256 + threadIdx.x;
  if (col >= N) return;
  const float* src = part + int64_t(blockIdx.y) * parts * N + col;
  float s = 0.f;
  for (int i = 0; i < parts; ++i) s = __fadd_rn(s, __ldg(src + int64_t(i) * N));
  out[int64_t(blockIdx.y) * ldo + col] = s;
}

}  // namespace fvb

using namespace fvb;

// Every pointer a row kernel reads or writes with 128-bit vectors (uint4 bf16 rows, float4 fp32 rows, per-column vectors, cos /
// sin tables and workspace partials, double2 float64 tables) must be 16-byte aligned; NULL passes.
static inline bool al16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

extern "C" int fvb_layernorm_modulate(const void* x, int x_is_f32, int64_t ldx, const float* w, const float* b,
                                      const float* scale, const float* shift, int mod_rows, int64_t mod_stride,
                                      int round_ln, void* out, int64_t ldo, void* hidden_out, int64_t ldh, int M, int D,
                                      float eps, void* stream) {
  FVB_CHECK_ARG(x && out, "null pointer");
  FVB_CHECK_ARG(M > 0 && D > 0 && D % 8 == 0 && D <= EW_THREADS * EW_MAX_CHUNKS * 8, "D must be a multiple of 8, <= 8192");
  FVB_CHECK_ARG(ldx % 8 == 0 && ldo % 8 == 0 && (hidden_out == nullptr || ldh % 8 == 0), "strides must be multiples of 8");
  FVB_CHECK_ARG((w == nullptr) == (b == nullptr), "affine weight and bias must come together");
  FVB_CHECK_ARG((scale == nullptr) == (shift == nullptr), "scale and shift must come together");
  FVB_CHECK_ARG(mod_rows >= 0 && (mod_rows == 0 || mod_stride % 4 == 0), "bad modulation grouping (stride must be a multiple of 4)");
  FVB_CHECK_ARG(al16(x) && al16(out) && al16(hidden_out) && al16(w) && al16(b) && al16(scale) && al16(shift),
                "x, out, hidden_out, w, b, scale and shift must be 16-byte aligned");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  auto* o = reinterpret_cast<__nv_bfloat16*>(out);
  auto* h = reinterpret_cast<__nv_bfloat16*>(hidden_out);
  if (round_ln & 2) FVB_CHECK_ARG(!x_is_f32 && (round_ln & 1), "bf16 modulation arithmetic implies a bf16 input and a bf16 LayerNorm output");
  const int row_bytes = D * (x_is_f32 ? 4 : 2);
  // warp-per-row kernel: 16 warps when 16 rows fit the staging budget, else as many as fit (>= 8: fp32 rows of D = 5120 are
  // 20 KB -> 9 warps x 1 stage; the block-per-row fallback ran those at 2.1 TB/s)
  const int nw = std::min(RW_WARPS, RW_SMEM_BUDGET / row_bytes);
  const bool use_warp = M >= 256 && nw >= 8;
  if (use_warp) {
    const int stages = std::max(1, std::min(RW_MAX_STAGES, RW_SMEM_BUDGET / (nw * row_bytes)));
    size_t smem = size_t(nw) * stages * row_bytes;
    // per-column vectors in shared memory: the modulation pair when one (scale, shift) serves every row, else the affine pair
    int tab_kind = 0;
    if (smem + size_t(D) * 8 <= RW_SMEM_MAX) {
      if (scale != nullptr && (mod_rows == 0 || mod_rows >= M)) tab_kind = 2;
      else if (w != nullptr) tab_kind = 1;
    }
    if (tab_kind != 0) smem += size_t(D) * 8;
    const int grid = std::min((M + nw - 1) / nw, sm_count());
    auto launch = [&](auto kern) -> int {
      FVB_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, RW_SMEM_MAX));
      kern<<<grid, RW_WARPS * 32, smem, st>>>(x, ldx, w, b, scale, shift, o, ldo, h, ldh, D, eps, mod_rows, mod_stride, M, stages, nw,
                                              tab_kind);
      return FVB_OK;
    };
    int rc;
    if (round_ln & 2) rc = launch(layernorm_warp_kernel<false, true, true>);
    else if (x_is_f32) rc = round_ln ? launch(layernorm_warp_kernel<true, true, false>) : launch(layernorm_warp_kernel<true, false, false>);
    else rc = round_ln ? launch(layernorm_warp_kernel<false, true, false>) : launch(layernorm_warp_kernel<false, false, false>);
    if (rc) return rc;
  } else if (round_ln & 2) {
    layernorm_kernel<false, true, true><<<M, EW_THREADS, 0, st>>>(x, ldx, w, b, scale, shift, o, ldo, h, ldh, D, eps, mod_rows, mod_stride);
  } else if (x_is_f32) {
    if (round_ln) layernorm_kernel<true, true><<<M, EW_THREADS, 0, st>>>(x, ldx, w, b, scale, shift, o, ldo, h, ldh, D, eps, mod_rows, mod_stride);
    else layernorm_kernel<true, false><<<M, EW_THREADS, 0, st>>>(x, ldx, w, b, scale, shift, o, ldo, h, ldh, D, eps, mod_rows, mod_stride);
  } else {
    if (round_ln) layernorm_kernel<false, true><<<M, EW_THREADS, 0, st>>>(x, ldx, w, b, scale, shift, o, ldo, h, ldh, D, eps, mod_rows, mod_stride);
    else layernorm_kernel<false, false><<<M, EW_THREADS, 0, st>>>(x, ldx, w, b, scale, shift, o, ldo, h, ldh, D, eps, mod_rows, mod_stride);
  }
  FVB_CHECK_CUDA(cudaGetLastError());
  return FVB_OK;
}

extern "C" int fvb_rmsnorm_rope_scatter(const void* x0, const void* w0, int64_t ld0, const void* x1, const void* w1, int64_t ld1,
                                        void* y0, void* y1, int64_t ldy, const int64_t* out_col_offsets, const void* cos_t,
                                        const void* sin_t, int rope_f64, const int32_t* rope_row, int M, int D, int head_dim,
                                        float eps, void* stream) {
  FVB_CHECK_ARG(x0 && y0 && out_col_offsets, "null pointer");
  FVB_CHECK_ARG((x1 == nullptr) == (y1 == nullptr), "x1 and y1 must come together");
  FVB_CHECK_ARG(M > 0 && D > 0 && D % 128 == 0 && RW_WARPS * D * 2 <= RW_SMEM_BUDGET, "D must be a multiple of 128, <= 6144");
  FVB_CHECK_ARG(head_dim % 8 == 0 && D % head_dim == 0, "head_dim must divide D and be a multiple of 8");
  FVB_CHECK_ARG(ld0 % 8 == 0 && (x1 == nullptr || ld1 % 8 == 0) && ldy % 8 == 0, "strides must be multiples of 8");
  FVB_CHECK_ARG(al16(x0) && al16(x1) && al16(y0) && al16(y1) && al16(w0) && al16(w1) && al16(cos_t) && al16(sin_t),
                "x0, x1, y0, y1, w0, w1, cos and sin must be 16-byte aligned");
  FVB_CHECK_ARG((cos_t == nullptr) == (sin_t == nullptr), "cos and sin must come together");
  const int w_f32 = (rope_f64 >> 1) & 1;  // flags: bit 0 = float64 tables, bit 1 = fp32 weights
  rope_f64 &= 1;
  FVB_CHECK_ARG(!rope_f64 || cos_t != nullptr, "float64 RoPE needs tables");
  RmsRopeArgs a;
  a.w_f32 = w_f32;
  a.x[0] = reinterpret_cast<__nv_bfloat16*>(const_cast<void*>(x0));
  a.w[0] = reinterpret_cast<const __nv_bfloat16*>(w0);
  a.ld[0] = ld0;
  a.x[1] = reinterpret_cast<__nv_bfloat16*>(const_cast<void*>(x1));
  a.w[1] = reinterpret_cast<const __nv_bfloat16*>(w1);
  a.ld[1] = ld1;
  a.col_offsets = nullptr;
  a.y[0] = reinterpret_cast<__nv_bfloat16*>(y0);
  a.y[1] = reinterpret_cast<__nv_bfloat16*>(y1);
  a.ldy = ldy;
  a.out_col_offsets = out_col_offsets;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int row_bytes = D * 2;
  const int stages = rw_stages(row_bytes);
  size_t smem = size_t(RW_WARPS) * stages * row_bytes;
  const int w_tab = (smem + size_t(D) * 4 <= RW_SMEM_MAX) ? 1 : 0;  // fp32 norm weight in shared memory
  if (w_tab) smem += size_t(D) * 4;
  dim3 grid(std::min((M + RW_WARPS - 1) / RW_WARPS, sm_count()), x1 ? 2 : 1);
  auto launch = [&](auto kern) -> int {
    FVB_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, RW_SMEM_MAX));
    kern<<<grid, RW_WARPS * 32, smem, st>>>(a, cos_t, sin_t, rope_row, D, head_dim, eps, M, stages, w_tab);
    return FVB_OK;
  };
  const int rc = rope_f64 ? launch(rmsnorm_rope_warp_kernel<true>) : launch(rmsnorm_rope_warp_kernel<false>);
  if (rc) return rc;
  FVB_CHECK_CUDA(cudaGetLastError());
  return FVB_OK;
}

extern "C" int fvb_rmsnorm_rope(void* x0, const void* w0, int64_t ld0, void* x1, const void* w1, int64_t ld1,
                                const void* cos_t, const void* sin_t, int rope_f64, const int32_t* rope_row,
                                const int64_t* col_offsets, int M, int D, int head_dim, float eps, void* stream) {
  FVB_CHECK_ARG(x0 && w0, "null pointer");
  FVB_CHECK_ARG(M > 0 && D > 0 && D % 8 == 0 && D <= EW_THREADS * EW_MAX_CHUNKS * 8, "D must be a multiple of 8, <= 8192");
  FVB_CHECK_ARG(head_dim % 8 == 0 && D % head_dim == 0, "head_dim must divide D and be a multiple of 8");
  FVB_CHECK_ARG(ld0 % 8 == 0 && (x1 == nullptr || ld1 % 8 == 0), "strides must be multiples of 8");
  FVB_CHECK_ARG(al16(x0) && al16(x1) && al16(w0) && al16(w1) && al16(cos_t) && al16(sin_t),
                "x0, x1, w0, w1, cos and sin must be 16-byte aligned");
  FVB_CHECK_ARG((cos_t == nullptr) == (sin_t == nullptr), "cos and sin must come together");
  const int w_f32 = (rope_f64 >> 1) & 1;  // flags: bit 0 = float64 tables, bit 1 = fp32 weights
  rope_f64 &= 1;
  FVB_CHECK_ARG(!rope_f64 || cos_t != nullptr, "float64 RoPE needs tables");
  RmsRopeArgs a;
  a.w_f32 = w_f32;
  a.x[0] = reinterpret_cast<__nv_bfloat16*>(x0);
  a.w[0] = reinterpret_cast<const __nv_bfloat16*>(w0);
  a.ld[0] = ld0;
  a.x[1] = reinterpret_cast<__nv_bfloat16*>(x1);
  a.w[1] = reinterpret_cast<const __nv_bfloat16*>(w1);
  a.ld[1] = ld1;
  a.col_offsets = col_offsets;
  FVB_CHECK_ARG(col_offsets == nullptr || D % 128 == 0, "column-block offsets need D % 128 == 0");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int row_bytes = D * 2;
  const bool use_warp = M >= 256 && RW_WARPS * row_bytes <= RW_SMEM_BUDGET;
  if (use_warp) {
    const int stages = rw_stages(row_bytes);
    size_t smem = size_t(RW_WARPS) * stages * row_bytes;
    const int w_tab = (smem + size_t(D) * 4 <= RW_SMEM_MAX) ? 1 : 0;  // fp32 norm weight in shared memory
    if (w_tab) smem += size_t(D) * 4;
    dim3 grid(std::min((M + RW_WARPS - 1) / RW_WARPS, sm_count()), x1 ? 2 : 1);
    auto launch = [&](auto kern) -> int {
      FVB_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, RW_SMEM_MAX));
      kern<<<grid, RW_WARPS * 32, smem, st>>>(a, cos_t, sin_t, rope_row, D, head_dim, eps, M, stages, w_tab);
      return FVB_OK;
    };
    const int rc = rope_f64 ? launch(rmsnorm_rope_warp_kernel<true>) : launch(rmsnorm_rope_warp_kernel<false>);
    if (rc) return rc;
  } else {
    dim3 grid(M, x1 ? 2 : 1);
    if (rope_f64) rmsnorm_rope_kernel<true><<<grid, EW_THREADS, 0, st>>>(a, cos_t, sin_t, rope_row, D, head_dim, eps);
    else rmsnorm_rope_kernel<false><<<grid, EW_THREADS, 0, st>>>(a, cos_t, sin_t, rope_row, D, head_dim, eps);
  }
  FVB_CHECK_CUDA(cudaGetLastError());
  return FVB_OK;
}

extern "C" int64_t fvb_rmsnorm_bwd_workspace_bytes(int M, int D) {
  return int64_t(std::max(1, std::min(M, RB_CTAS))) * std::max(D, 0) * 4;
}

extern "C" int fvb_rmsnorm_bwd(const void* x, int64_t ldx, const void* w, const void* dy, int64_t lddy, void* dx, int64_t lddx,
                               void* dw, float* workspace, int64_t workspace_bytes, int M, int D, float eps, void* stream) {
  FVB_CHECK_ARG(x && dy && dx, "null pointer");
  FVB_CHECK_ARG(M > 0 && D > 0 && D % 8 == 0 && D <= EW_THREADS * EW_MAX_CHUNKS * 8, "D must be a multiple of 8, <= 8192");
  FVB_CHECK_ARG(ldx % 8 == 0 && lddy % 8 == 0 && lddx % 8 == 0, "strides must be multiples of 8");
  FVB_CHECK_ARG(dw == nullptr || w != nullptr, "dw needs the weight");
  FVB_CHECK_ARG(al16(x) && al16(w) && al16(dy) && al16(dx) && al16(workspace), "x, w, dy, dx and workspace must be 16-byte aligned");
  const int ctas = std::min(M, RB_CTAS);
  if (dw != nullptr)
    FVB_CHECK_ARG(workspace != nullptr && workspace_bytes >= fvb_rmsnorm_bwd_workspace_bytes(M, D), "workspace too small");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  rmsnorm_bwd_kernel<<<ctas, EW_THREADS, 0, st>>>(
      reinterpret_cast<const __nv_bfloat16*>(x), ldx, reinterpret_cast<const __nv_bfloat16*>(w),
      reinterpret_cast<const __nv_bfloat16*>(dy), lddy, reinterpret_cast<__nv_bfloat16*>(dx), lddx,
      dw != nullptr ? workspace : nullptr, M, D, eps);
  FVB_CHECK_CUDA(cudaGetLastError());
  if (dw != nullptr) {
    rmsnorm_bwd_dw_kernel<<<(D + 255) / 256, 256, 0, st>>>(workspace, ctas, D, reinterpret_cast<__nv_bfloat16*>(dw));
    FVB_CHECK_CUDA(cudaGetLastError());
  }
  return FVB_OK;
}

extern "C" int64_t fvb_bias_grad_bf16_workspace_bytes(int M, int N) {
  return int64_t(std::max(1, std::min(M, BG_PARTS))) * std::max(N, 0) * 4;
}

extern "C" int fvb_bias_grad_bf16(const void* dy, int64_t lddy, void* db, float* workspace, int64_t workspace_bytes, int M, int N,
                                  void* stream) {
  FVB_CHECK_ARG(dy && db && workspace, "null pointer");
  FVB_CHECK_ARG(M > 0 && N > 0 && N % 8 == 0, "N must be a positive multiple of 8");
  FVB_CHECK_ARG(lddy % 8 == 0, "lddy must be a multiple of 8");
  FVB_CHECK_ARG(al16(dy) && al16(workspace), "dy and workspace must be 16-byte aligned");
  FVB_CHECK_ARG(workspace_bytes >= fvb_bias_grad_bf16_workspace_bytes(M, N), "workspace too small");
  const int parts = std::min(M, BG_PARTS);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  bias_grad_kernel<<<dim3(parts, (N / 8 + BG_THREADS - 1) / BG_THREADS), BG_THREADS, 0, st>>>(
      reinterpret_cast<const __nv_bfloat16*>(dy), lddy, workspace, M, N, parts);
  FVB_CHECK_CUDA(cudaGetLastError());
  rmsnorm_bwd_dw_kernel<<<(N + 255) / 256, 256, 0, st>>>(workspace, parts, N, reinterpret_cast<__nv_bfloat16*>(db));
  FVB_CHECK_CUDA(cudaGetLastError());
  return FVB_OK;
}

extern "C" int64_t fvb_rmsnorm_rope_bwd_workspace_bytes(int M, int D) { return 2 * fvb_rmsnorm_bwd_workspace_bytes(M, D); }

extern "C" int fvb_rmsnorm_rope_bwd(const void* x0, int64_t ldx0, const void* w0, const void* dy0, int64_t lddy0, void* dx0,
                                    int64_t lddx0, void* dw0, const void* x1, int64_t ldx1, const void* w1, const void* dy1,
                                    int64_t lddy1, void* dx1, int64_t lddx1, void* dw1, const float* cos_t, const float* sin_t,
                                    const int32_t* rope_row, float* workspace, int64_t workspace_bytes, int M, int D,
                                    int head_dim, float eps, void* stream) {
  FVB_CHECK_ARG(x0 && w0 && dy0 && dx0 && cos_t && sin_t, "null pointer");
  FVB_CHECK_ARG(x1 == nullptr || (w1 && dy1 && dx1), "x1 needs w1, dy1 and dx1");
  FVB_CHECK_ARG(M > 0 && D > 0 && D % 8 == 0 && D <= EW_THREADS * EW_MAX_CHUNKS * 8, "D must be a multiple of 8, <= 8192");
  FVB_CHECK_ARG(head_dim % 8 == 0 && D % head_dim == 0, "head_dim must divide D and be a multiple of 8");
  FVB_CHECK_ARG(ldx0 % 8 == 0 && lddy0 % 8 == 0 && lddx0 % 8 == 0, "strides must be multiples of 8");
  FVB_CHECK_ARG(x1 == nullptr || (ldx1 % 8 == 0 && lddy1 % 8 == 0 && lddx1 % 8 == 0), "strides must be multiples of 8");
  FVB_CHECK_ARG(x1 == nullptr || (dw0 != nullptr) == (dw1 != nullptr), "dw0 and dw1 come together");
  FVB_CHECK_ARG(al16(x0) && al16(w0) && al16(dy0) && al16(dx0) && al16(x1) && al16(w1) && al16(dy1) && al16(dx1) && al16(cos_t) &&
                    al16(sin_t) && al16(workspace),
                "x, w, dy, dx, cos, sin and workspace must be 16-byte aligned");
  const int ctas = std::min(M, RB_CTAS);
  const bool want_dw = dw0 != nullptr;
  if (want_dw)
    FVB_CHECK_ARG(workspace != nullptr && workspace_bytes >= fvb_rmsnorm_rope_bwd_workspace_bytes(M, D), "workspace too small");
  RmsRopeBwdArgs a;
  a.x[0] = reinterpret_cast<const __nv_bfloat16*>(x0);
  a.w[0] = reinterpret_cast<const __nv_bfloat16*>(w0);
  a.dy[0] = reinterpret_cast<const __nv_bfloat16*>(dy0);
  a.dx[0] = reinterpret_cast<__nv_bfloat16*>(dx0);
  a.ldx[0] = ldx0;
  a.lddy[0] = lddy0;
  a.lddx[0] = lddx0;
  a.x[1] = reinterpret_cast<const __nv_bfloat16*>(x1);
  a.w[1] = reinterpret_cast<const __nv_bfloat16*>(w1);
  a.dy[1] = reinterpret_cast<const __nv_bfloat16*>(dy1);
  a.dx[1] = reinterpret_cast<__nv_bfloat16*>(dx1);
  a.ldx[1] = ldx1;
  a.lddy[1] = lddy1;
  a.lddx[1] = lddx1;
  const int nt = x1 != nullptr ? 2 : 1;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  rmsnorm_rope_bwd_kernel<<<dim3(ctas, nt), EW_THREADS, 0, st>>>(a, want_dw ? workspace : nullptr, cos_t, sin_t, rope_row, M, D,
                                                                 head_dim, eps);
  FVB_CHECK_CUDA(cudaGetLastError());
  if (want_dw) {
    void* dws[2] = {dw0, dw1};
    for (int t = 0; t < nt; ++t) {
      rmsnorm_bwd_dw_kernel<<<(D + 255) / 256, 256, 0, st>>>(workspace + int64_t(t) * ctas * D, ctas, D,
                                                             reinterpret_cast<__nv_bfloat16*>(dws[t]));
      FVB_CHECK_CUDA(cudaGetLastError());
    }
  }
  return FVB_OK;
}

extern "C" int64_t fvb_resid_gate_bwd_workspace_bytes(int M, int N) { return 2 * fvb_bias_grad_bf16_workspace_bytes(M, N); }

extern "C" int fvb_resid_gate_bwd(const void* dout, int dout_is_f32, int64_t lddout, const void* y, int64_t ldy, const float* gate,
                                  void* dy, int64_t lddy, float* d_gate, void* db, float* workspace, int64_t workspace_bytes,
                                  int M, int N, void* stream) {
  FVB_CHECK_ARG(dout && y && gate && dy && d_gate && workspace, "null pointer");
  FVB_CHECK_ARG(M > 0 && N > 0 && N % 8 == 0, "N must be a positive multiple of 8");
  FVB_CHECK_ARG(lddout % (dout_is_f32 ? 4 : 8) == 0 && ldy % 8 == 0 && lddy % 8 == 0, "strides must keep rows 16-byte aligned");
  FVB_CHECK_ARG(al16(dout) && al16(y) && al16(gate) && al16(dy) && al16(workspace),
                "dout, y, gate, dy and workspace must be 16-byte aligned");
  FVB_CHECK_ARG(workspace_bytes >= fvb_resid_gate_bwd_workspace_bytes(M, N), "workspace too small");
  const int parts = std::min(M, BG_PARTS);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const dim3 grid(parts, (N / 8 + BG_THREADS - 1) / BG_THREADS);
  auto* yb = reinterpret_cast<const __nv_bfloat16*>(y);
  auto* dyb = reinterpret_cast<__nv_bfloat16*>(dy);
  if (dout_is_f32)
    resid_gate_bwd_kernel<true><<<grid, BG_THREADS, 0, st>>>(dout, lddout, yb, ldy, gate, dyb, lddy, workspace, M, N, parts);
  else
    resid_gate_bwd_kernel<false><<<grid, BG_THREADS, 0, st>>>(dout, lddout, yb, ldy, gate, dyb, lddy, workspace, M, N, parts);
  FVB_CHECK_CUDA(cudaGetLastError());
  colsum_f32_kernel<<<(N + 255) / 256, 256, 0, st>>>(workspace, parts, N, d_gate);
  FVB_CHECK_CUDA(cudaGetLastError());
  if (db != nullptr) {
    rmsnorm_bwd_dw_kernel<<<(N + 255) / 256, 256, 0, st>>>(workspace + int64_t(parts) * N, parts, N, reinterpret_cast<__nv_bfloat16*>(db));
    FVB_CHECK_CUDA(cudaGetLastError());
  }
  return FVB_OK;
}

extern "C" int64_t fvb_layernorm_modulate_bwd_workspace_bytes(int M, int D) { return 2 * fvb_rmsnorm_bwd_workspace_bytes(M, D); }

extern "C" int fvb_layernorm_modulate_bwd(const void* x, int x_is_f32, int64_t ldx, const void* dn, int64_t lddn, const float* gain,
                                          int gain_is_scale, int round_ln, const void* gin, int gin_is_f32, int64_t ldgin, void* dx,
                                          int64_t lddx, float* d_gain, float* d_offset, float* workspace, int64_t workspace_bytes,
                                          int M, int D, float eps, void* stream) {
  FVB_CHECK_ARG(x && dn && gain && dx && d_gain && d_offset && workspace, "null pointer");
  FVB_CHECK_ARG(M > 0 && D > 0 && D % 8 == 0 && D <= EW_THREADS * EW_MAX_CHUNKS * 8, "D must be a multiple of 8, <= 8192");
  FVB_CHECK_ARG(ldx % 8 == 0 && lddn % 8 == 0 && lddx % 8 == 0 && (gin == nullptr || ldgin % 8 == 0), "strides must be multiples of 8");
  FVB_CHECK_ARG(al16(x) && al16(dn) && al16(gain) && al16(gin) && al16(dx) && al16(workspace),
                "x, dn, gain, gin, dx and workspace must be 16-byte aligned");
  FVB_CHECK_ARG(workspace_bytes >= fvb_layernorm_modulate_bwd_workspace_bytes(M, D), "workspace too small");
  FVB_CHECK_ARG(gain_is_scale || !round_ln, "round_ln belongs to the modulation form (the affine forward rounds after w, b)");
  const int ctas = std::min(M, RB_CTAS);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  auto* dnb = reinterpret_cast<const __nv_bfloat16*>(dn);
  auto launch = [&](auto kern) {
    kern<<<ctas, EW_THREADS, 0, st>>>(x, ldx, dnb, lddn, gain, gain_is_scale, round_ln, gin, ldgin, dx, lddx, workspace, M, D, eps);
  };
  if (x_is_f32) gin_is_f32 ? launch(layernorm_modulate_bwd_kernel<true, true>) : launch(layernorm_modulate_bwd_kernel<true, false>);
  else gin_is_f32 ? launch(layernorm_modulate_bwd_kernel<false, true>) : launch(layernorm_modulate_bwd_kernel<false, false>);
  FVB_CHECK_CUDA(cudaGetLastError());
  colsum_f32_kernel<<<(D + 255) / 256, 256, 0, st>>>(workspace, ctas, D, d_gain);
  FVB_CHECK_CUDA(cudaGetLastError());
  colsum_f32_kernel<<<(D + 255) / 256, 256, 0, st>>>(workspace + int64_t(ctas) * D, ctas, D, d_offset);
  FVB_CHECK_CUDA(cudaGetLastError());
  return FVB_OK;
}

extern "C" int64_t fvb_layernorm_modulate_grouped_bwd_workspace_bytes(int M, int mod_rows, int D) {
  if (M <= 0 || mod_rows <= 0 || D <= 0) return 0;
  const int64_t G = (M + mod_rows - 1) / mod_rows;
  return 2 * G * grouped_parts(M, mod_rows, RB_CTAS) * int64_t(D) * int64_t(sizeof(float));
}

extern "C" int fvb_layernorm_modulate_grouped_bwd(const void* x, int64_t ldx, const void* dn, int64_t lddn, const float* scale,
                                                  int mod_rows, int64_t mod_stride, const void* gin, int gin_is_f32,
                                                  int64_t ldgin, void* dx, int64_t lddx, float* d_scale, float* d_shift,
                                                  int64_t ld_dmod, float* workspace, int64_t workspace_bytes, int M, int D,
                                                  float eps, void* stream) {
  FVB_CHECK_ARG(x && dn && scale && dx && d_scale && d_shift && workspace, "null pointer");
  FVB_CHECK_ARG(M > 0 && D > 0 && D % 8 == 0 && D <= EW_THREADS * EW_MAX_CHUNKS * 8, "D must be a multiple of 8, <= 8192");
  FVB_CHECK_ARG(mod_rows > 0 && mod_stride % 4 == 0 && mod_stride >= D, "bad modulation grouping (rows > 0, stride >= D and a multiple of 4)");
  FVB_CHECK_ARG(ldx % 8 == 0 && lddn % 8 == 0 && lddx % 8 == 0 && (gin == nullptr || ldgin % 8 == 0), "strides must be multiples of 8");
  FVB_CHECK_ARG(ld_dmod >= D, "ld_dmod must be >= D");
  FVB_CHECK_ARG(al16(x) && al16(dn) && al16(scale) && al16(gin) && al16(dx) && al16(workspace),
                "x, dn, scale, gin, dx and workspace must be 16-byte aligned");
  FVB_CHECK_ARG(workspace_bytes >= fvb_layernorm_modulate_grouped_bwd_workspace_bytes(M, mod_rows, D), "workspace too small");
  const int G = (M + mod_rows - 1) / mod_rows;
  const int parts = grouped_parts(M, mod_rows, RB_CTAS);
  const int ctas = G * parts;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  auto* xb = reinterpret_cast<const __nv_bfloat16*>(x);
  auto* dnb = reinterpret_cast<const __nv_bfloat16*>(dn);
  auto* dxb = reinterpret_cast<__nv_bfloat16*>(dx);
  if (gin_is_f32)
    layernorm_modulate_grouped_bwd_kernel<true><<<ctas, EW_THREADS, 0, st>>>(xb, ldx, dnb, lddn, scale, mod_rows, mod_stride, gin,
                                                                             ldgin, dxb, lddx, workspace, M, D, eps, parts);
  else
    layernorm_modulate_grouped_bwd_kernel<false><<<ctas, EW_THREADS, 0, st>>>(xb, ldx, dnb, lddn, scale, mod_rows, mod_stride, gin,
                                                                              ldgin, dxb, lddx, workspace, M, D, eps, parts);
  FVB_CHECK_CUDA(cudaGetLastError());
  const dim3 cgrid((D + 255) / 256, G);
  grouped_colsum_kernel<<<cgrid, 256, 0, st>>>(workspace, parts, D, d_scale, ld_dmod);
  FVB_CHECK_CUDA(cudaGetLastError());
  grouped_colsum_kernel<<<cgrid, 256, 0, st>>>(workspace + int64_t(ctas) * D, parts, D, d_shift, ld_dmod);
  FVB_CHECK_CUDA(cudaGetLastError());
  return FVB_OK;
}

extern "C" int64_t fvb_resid_gate_grouped_bwd_workspace_bytes(int M, int gate_rows, int N) {
  if (M <= 0 || gate_rows <= 0 || N <= 0) return 0;
  const int64_t G = (M + gate_rows - 1) / gate_rows;
  return 2 * G * grouped_parts(M, gate_rows, BG_PARTS) * int64_t(N) * int64_t(sizeof(float));
}

extern "C" int fvb_resid_gate_grouped_bwd(const void* dout, int64_t lddout, const void* y, int64_t ldy, const float* gate,
                                          int gate_rows, int64_t gate_stride, void* dy, int64_t lddy, float* d_gate,
                                          int64_t ld_dgate, void* db, float* workspace, int64_t workspace_bytes, int M, int N,
                                          void* stream) {
  FVB_CHECK_ARG(dout && y && gate && dy && d_gate && workspace, "null pointer");
  FVB_CHECK_ARG(M > 0 && N > 0 && N % 8 == 0, "N must be a positive multiple of 8");
  FVB_CHECK_ARG(gate_rows > 0 && gate_stride % 4 == 0 && gate_stride >= N, "bad gate grouping (rows > 0, stride >= N and a multiple of 4)");
  FVB_CHECK_ARG(lddout % 8 == 0 && ldy % 8 == 0 && lddy % 8 == 0, "strides must keep rows 16-byte aligned");
  FVB_CHECK_ARG(ld_dgate >= N, "ld_dgate must be >= N");
  FVB_CHECK_ARG(al16(dout) && al16(y) && al16(gate) && al16(dy) && al16(workspace),
                "dout, y, gate, dy and workspace must be 16-byte aligned");
  FVB_CHECK_ARG(workspace_bytes >= fvb_resid_gate_grouped_bwd_workspace_bytes(M, gate_rows, N), "workspace too small");
  const int G = (M + gate_rows - 1) / gate_rows;
  const int parts = grouped_parts(M, gate_rows, BG_PARTS);
  const int ctas = G * parts;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  resid_gate_grouped_bwd_kernel<<<dim3(ctas, (N / 8 + BG_THREADS - 1) / BG_THREADS), BG_THREADS, 0, st>>>(
      reinterpret_cast<const __nv_bfloat16*>(dout), lddout, reinterpret_cast<const __nv_bfloat16*>(y), ldy, gate, gate_rows,
      gate_stride, reinterpret_cast<__nv_bfloat16*>(dy), lddy, workspace, M, N, parts);
  FVB_CHECK_CUDA(cudaGetLastError());
  grouped_colsum_kernel<<<dim3((N + 255) / 256, G), 256, 0, st>>>(workspace, parts, N, d_gate, ld_dgate);
  FVB_CHECK_CUDA(cudaGetLastError());
  if (db != nullptr) {  // every group's partials, in (g, p) order
    rmsnorm_bwd_dw_kernel<<<(N + 255) / 256, 256, 0, st>>>(workspace + int64_t(ctas) * N, ctas, N, reinterpret_cast<__nv_bfloat16*>(db));
    FVB_CHECK_CUDA(cudaGetLastError());
  }
  return FVB_OK;
}
