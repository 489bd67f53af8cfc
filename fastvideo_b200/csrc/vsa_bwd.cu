// vsa_bwd.cu -- the bandwidth-bound pieces of Video Sparse Attention's backward, padded layout (64-row tiles, the first
// variable_block_sizes[i] rows of tile i valid). With the forward
//   q_c = block_mean(q), k_c, v_c likewise; attn = softmax(q_c k_c^T / sqrt(d)); out_c = attn v_c
//   out = out_c (broadcast over its tile) * gate + out_s
// and dO given, these kernels produce (the matmuls between them run on fvb_gemm_batched_bf16, the sparse branch on
// fvb_attention_blocklist_bwd). Pad rows are not tokens: every gradient treats dO there as zero.
//   fvb_vsa_combine_bwd    d_gate = dO * out_c,  d_out_c = sum over a tile's valid rows of dO * gate (fixed order, fp32)
//   fvb_softmax_rows_bwd   d_scores = attn * (d_attn - rowsum(d_attn * attn)) * scale, optionally with d_scores^T and attn^T
//   fvb_block_mean_bwd     dx = dx_s + d_x_c / len on the valid rows, 0 on the pad rows
// The *_compact variants (template flag COMPACT) take the compact layout instead: tile i is rows [off[i], off[i + 1]) of a
// tile-major sequence without pad rows, so every row is a token and a tile's rows are never another tile's.
#include "fvb_host.cuh"
#include "fvb_ptx.cuh"

namespace fvb {

struct BwdStrides3 {
  int64_t v[3];
};

constexpr int VSA_TILE = 64;

// One CTA (256 threads) per (tile, h, b). Thread t owns channels 8 (t & 15) .. +7 of rows t >> 4, +16, +32, +48; the 16 row
// groups' partial sums are added in row-group order through shared memory, so the result does not depend on scheduling.
// block_len is block_off [nblk + 1] when COMPACT; rows of the tile past its length are then neither read nor written.
template <bool COMPACT>
__global__ void __launch_bounds__(256) vsa_combine_bwd_kernel(const __nv_bfloat16* __restrict__ dO, BwdStrides3 ds,
                                                              const __nv_bfloat16* __restrict__ gate, BwdStrides3 gs,
                                                              const __nv_bfloat16* __restrict__ out_c,
                                                              const int32_t* __restrict__ block_len,
                                                              __nv_bfloat16* __restrict__ d_gate, BwdStrides3 dgs,
                                                              __nv_bfloat16* __restrict__ d_out_c,
                                                              __nv_bfloat16* __restrict__ d_out_c_t, int64_t ldt, int nblk,
                                                              int H) {
  __shared__ float red[16][128];
  const int blk = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int c8 = threadIdx.x & 15, rg = threadIdx.x >> 4;
  const int len = COMPACT ? block_len[blk + 1] - block_len[blk] : block_len[blk];
  const int row0 = COMPACT ? block_len[blk] : 0;
  const int64_t bh = int64_t(b) * H + h;
  float oc[8];
  {
    const uint4 u = *reinterpret_cast<const uint4*>(out_c + (bh * nblk + blk) * 128 + c8 * 8);
    const __nv_bfloat162* c2 = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 f = __bfloat1622float2(c2[i]);
      oc[2 * i] = f.x;
      oc[2 * i + 1] = f.y;
    }
  }
  float acc[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i] = 0.f;
#pragma unroll
  for (int j = 0; j < VSA_TILE / 16; ++j) {
    const int r = rg + 16 * j;
    if (COMPACT && r >= len) continue;
    const int64_t tok = COMPACT ? int64_t(row0) + r : int64_t(blk) * VSA_TILE + r;
    const uint4 ud = *reinterpret_cast<const uint4*>(dO + b * ds.v[0] + tok * ds.v[1] + h * ds.v[2] + c8 * 8);
    const __nv_bfloat162* d2 = reinterpret_cast<const __nv_bfloat162*>(&ud);
    float dv[8];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 f = __bfloat1622float2(d2[i]);
      dv[2 * i] = f.x;
      dv[2 * i + 1] = f.y;
    }
    if (gate != nullptr) {
      const uint4 ug = *reinterpret_cast<const uint4*>(gate + b * gs.v[0] + tok * gs.v[1] + h * gs.v[2] + c8 * 8);
      const __nv_bfloat162* g2 = reinterpret_cast<const __nv_bfloat162*>(&ug);
      float gv[8];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float2 f = __bfloat1622float2(g2[i]);
        gv[2 * i] = f.x;
        gv[2 * i + 1] = f.y;
      }
      if (d_gate != nullptr) {
        uint4 o = make_uint4(0, 0, 0, 0);
        if (r < len) {
          o.x = pack_bf16x2(__fmul_rn(dv[0], oc[0]), __fmul_rn(dv[1], oc[1]));
          o.y = pack_bf16x2(__fmul_rn(dv[2], oc[2]), __fmul_rn(dv[3], oc[3]));
          o.z = pack_bf16x2(__fmul_rn(dv[4], oc[4]), __fmul_rn(dv[5], oc[5]));
          o.w = pack_bf16x2(__fmul_rn(dv[6], oc[6]), __fmul_rn(dv[7], oc[7]));
        }
        *reinterpret_cast<uint4*>(d_gate + b * dgs.v[0] + tok * dgs.v[1] + h * dgs.v[2] + c8 * 8) = o;
      }
      if (r < len) {
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[i] = __fadd_rn(acc[i], __fmul_rn(dv[i], gv[i]));
      }
    } else if (r < len) {
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] = __fadd_rn(acc[i], dv[i]);
    }
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) red[rg][c8 * 8 + i] = acc[i];
  __syncthreads();
  if (threadIdx.x < 128) {
    const int c = threadIdx.x;
    float s = 0.f;
#pragma unroll
    for (int g = 0; g < 16; ++g) s = __fadd_rn(s, red[g][c]);
    const __nv_bfloat16 sb = __float2bfloat16_rn(s);
    d_out_c[(bh * nblk + blk) * 128 + c] = sb;
    if (d_out_c_t != nullptr) d_out_c_t[(bh * 128 + c) * ldt + blk] = sb;
  }
}

// Softmax backward over square [n, n] blocks of rows (batch b at base + b * n * ld). One CTA (256 threads) per 32 rows of one
// batch: each warp reduces rowsum(dp * p) of 4 rows (lane-strided partials, then a shuffle tree: a fixed order), then the CTA
// walks 64-column tiles: thread t computes 8 elements of row t >> 3, stores them row-major and stages the bf16 results in shared
// memory, from where the transposed tiles are stored as 16-byte rows of 8 consecutive source rows.
constexpr int SMB_ROWS = 32;
constexpr int SMB_COLS = 64;
constexpr int SMB_LDS = SMB_COLS + 2;  // bf16 pitch of the staging tiles: 33 words, so neither access pattern conflicts

FVB_DEVICE void load8_bf16(const __nv_bfloat16* p, int valid, float* f) {
  if (valid >= 8) {
    const uint4 u = __ldg(reinterpret_cast<const uint4*>(p));
    const __nv_bfloat162* h2 = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 v = __bfloat1622float2(h2[i]);
      f[2 * i] = v.x;
      f[2 * i + 1] = v.y;
    }
  } else {
#pragma unroll
    for (int i = 0; i < 8; ++i) f[i] = i < valid ? __bfloat162float(p[i]) : 0.f;
  }
}

__global__ void __launch_bounds__(256) softmax_rows_bwd_kernel(const __nv_bfloat16* __restrict__ p,
                                                               const __nv_bfloat16* __restrict__ dp, int64_t ld, int n,
                                                               float scale, __nv_bfloat16* __restrict__ ds,
                                                               __nv_bfloat16* __restrict__ ds_t,
                                                               __nv_bfloat16* __restrict__ p_t) {
  __shared__ float rowsum[SMB_ROWS];
  __shared__ __align__(16) __nv_bfloat16 sds[SMB_ROWS * SMB_LDS];
  __shared__ __align__(16) __nv_bfloat16 sp[SMB_ROWS * SMB_LDS];
  const int64_t base = int64_t(blockIdx.y) * n * ld;
  const int i0 = blockIdx.x * SMB_ROWS;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int rr = 0; rr < SMB_ROWS / 8; ++rr) {
    const int r = warp * (SMB_ROWS / 8) + rr;
    float s = 0.f;
    if (i0 + r < n) {
      const int64_t row = base + int64_t(i0 + r) * ld;
      for (int c = lane * 8; c < n; c += 256) {
        float a[8], g[8];
        load8_bf16(p + row + c, n - c, a);
        load8_bf16(dp + row + c, n - c, g);
#pragma unroll
        for (int i = 0; i < 8; ++i) s = __fmaf_rn(a[i], g[i], s);
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) rowsum[r] = s;
  }
  __syncthreads();
  const int r = threadIdx.x >> 3, c8 = (threadIdx.x & 7) * 8;
  const bool row_ok = i0 + r < n;
  const float rs = rowsum[r];
  // transposed stores: thread t covers column jj = t >> 2 of the tile and source rows ii .. ii + 7
  const int jj = threadIdx.x >> 2, ii = (threadIdx.x & 3) * 8;
  for (int j0 = 0; j0 < n; j0 += SMB_COLS) {
    const int c = j0 + c8;
    float a[8], g[8];
    uint32_t dsp[4], pp[4];
    if (row_ok && c < n) {
      const int64_t off = base + int64_t(i0 + r) * ld + c;
      load8_bf16(p + off, n - c, a);
      load8_bf16(dp + off, n - c, g);
      float o[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) o[i] = __fmul_rn(__fmul_rn(a[i], __fsub_rn(g[i], rs)), scale);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        dsp[i] = pack_bf16x2(o[2 * i], o[2 * i + 1]);
        pp[i] = pack_bf16x2(a[2 * i], a[2 * i + 1]);
      }
      if (n - c >= 8) {
        *reinterpret_cast<uint4*>(ds + off) = make_uint4(dsp[0], dsp[1], dsp[2], dsp[3]);
      } else {
#pragma unroll
        for (int i = 0; i < 8; ++i)
          if (i < n - c) ds[off + i] = __float2bfloat16_rn(o[i]);
      }
    } else {
#pragma unroll
      for (int i = 0; i < 4; ++i) dsp[i] = pp[i] = 0u;
    }
    if (ds_t == nullptr && p_t == nullptr) continue;
    __syncthreads();  // the previous tile's transposed stores have read the staging tiles
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      reinterpret_cast<uint32_t*>(sds + r * SMB_LDS + c8)[i] = dsp[i];
      reinterpret_cast<uint32_t*>(sp + r * SMB_LDS + c8)[i] = pp[i];
    }
    __syncthreads();
    const int j = j0 + jj;
    if (j < n && i0 + ii < n) {
      const int nv = min(8, n - (i0 + ii));
      const int64_t off = base + int64_t(j) * ld + i0 + ii;
#pragma unroll
      for (int t = 0; t < 2; ++t) {
        __nv_bfloat16* dst = t ? p_t : ds_t;
        if (dst == nullptr) continue;
        const unsigned short* src = reinterpret_cast<const unsigned short*>(t ? sp : sds);
        uint32_t w[4];
#pragma unroll
        for (int i = 0; i < 4; ++i)
          w[i] = uint32_t(src[(ii + 2 * i) * SMB_LDS + jj]) | (uint32_t(src[(ii + 2 * i + 1) * SMB_LDS + jj]) << 16);
        if (nv == 8) {
          *reinterpret_cast<uint4*>(dst + off) = make_uint4(w[0], w[1], w[2], w[3]);
        } else {
          unsigned short* d16 = reinterpret_cast<unsigned short*>(dst + off);
#pragma unroll
          for (int i = 0; i < 8; ++i)
            if (i < nv) d16[i] = (unsigned short)(w[i >> 1] >> (16 * (i & 1)));
        }
      }
    }
  }
}

// dx[b, tok, h, :] = bf16(dx_s + d_mean[b, h, tile, :] / len[tile]) for tok % 64 < len[tile], else 0. One thread per 8
// elements; dx may be dx_s (in place). COMPACT: block_len is block_off [nblk + 1], tile = row_block[tok], every row valid.
template <bool COMPACT>
__global__ void block_mean_bwd_kernel(const __nv_bfloat16* dx_s, BwdStrides3 ss, const __nv_bfloat16* __restrict__ d_mean,
                                      const int32_t* __restrict__ block_len, __nv_bfloat16* dx, BwdStrides3 os, int B, int S,
                                      int H, int nblk, const int32_t* __restrict__ row_block) {
  const int64_t idx = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  const int64_t total = int64_t(B) * H * S * 16;
  if (idx >= total) return;
  const int c8 = int(idx & 15);
  const int tok = int((idx >> 4) % S);
  const int64_t bh = (idx >> 4) / S;
  const int h = int(bh % H), b = int(bh / H);
  const int blk = COMPACT ? __ldg(row_block + tok) : tok / VSA_TILE;
  const int len = COMPACT ? __ldg(block_len + blk + 1) - __ldg(block_len + blk) : __ldg(block_len + blk);
  uint4 o = make_uint4(0, 0, 0, 0);
  if (COMPACT || tok - blk * VSA_TILE < len) {
    const uint4 us = *reinterpret_cast<const uint4*>(dx_s + b * ss.v[0] + int64_t(tok) * ss.v[1] + h * ss.v[2] + c8 * 8);
    const uint4 um = __ldg(reinterpret_cast<const uint4*>(d_mean + (bh * nblk + blk) * 128 + c8 * 8));
    const __nv_bfloat162* s2 = reinterpret_cast<const __nv_bfloat162*>(&us);
    const __nv_bfloat162* m2 = reinterpret_cast<const __nv_bfloat162*>(&um);
    const float fl = float(len);
    uint32_t* o32 = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 fs = __bfloat1622float2(s2[i]), fm = __bfloat1622float2(m2[i]);
      o32[i] = pack_bf16x2(__fadd_rn(fs.x, __fdiv_rn(fm.x, fl)), __fadd_rn(fs.y, __fdiv_rn(fm.y, fl)));
    }
  }
  *reinterpret_cast<uint4*>(dx + b * os.v[0] + int64_t(tok) * os.v[1] + h * os.v[2] + c8 * 8) = o;
}

static bool strides_ok(const int64_t* s) { return s[0] % 8 == 0 && s[1] % 8 == 0 && s[2] % 8 == 0; }

}  // namespace fvb

using namespace fvb;

template <bool COMPACT>
static int combine_bwd(const void* dO, const int64_t* do_strides, const void* gate, const int64_t* g_strides, const void* out_c,
                       const int32_t* block_tab, int B, int S, int H, int nblk, void* d_gate, const int64_t* dg_strides,
                       void* d_out_c, void* d_out_c_t, int64_t ldt, void* stream) {
  FVB_CHECK_ARG(dO && do_strides && out_c && block_tab && d_out_c, "null pointer");
  if (COMPACT)
    FVB_CHECK_ARG(B > 0 && H > 0 && nblk > 0 && S > 0, "empty problem");
  else
    FVB_CHECK_ARG(B > 0 && H > 0 && nblk > 0 && S == nblk * VSA_TILE, "S must be 64 * nblk (padded layout)");
  FVB_CHECK_ARG(gate == nullptr || g_strides != nullptr, "gate strides missing");
  FVB_CHECK_ARG(d_gate == nullptr || (gate != nullptr && dg_strides != nullptr), "d_gate needs gate and its strides");
  FVB_CHECK_ARG(d_out_c_t == nullptr || ldt >= nblk, "ldt too small");
  FVB_CHECK_ARG(strides_ok(do_strides) && (gate == nullptr || strides_ok(g_strides)) && (d_gate == nullptr || strides_ok(dg_strides)),
                "strides must be multiples of 8");
  BwdStrides3 ds{}, gs{}, dgs{};
  for (int i = 0; i < 3; ++i) {
    ds.v[i] = do_strides[i];
    gs.v[i] = gate ? g_strides[i] : 0;
    dgs.v[i] = d_gate ? dg_strides[i] : 0;
  }
  vsa_combine_bwd_kernel<COMPACT><<<dim3(nblk, H, B), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const __nv_bfloat16*>(dO), ds, reinterpret_cast<const __nv_bfloat16*>(gate), gs,
      reinterpret_cast<const __nv_bfloat16*>(out_c), block_tab, reinterpret_cast<__nv_bfloat16*>(d_gate), dgs,
      reinterpret_cast<__nv_bfloat16*>(d_out_c), reinterpret_cast<__nv_bfloat16*>(d_out_c_t), ldt, nblk, H);
  FVB_CHECK_CUDA(cudaGetLastError());
  return FVB_OK;
}

extern "C" int fvb_vsa_combine_bwd(const void* dO, const int64_t* do_strides, const void* gate, const int64_t* g_strides,
                                   const void* out_c, const int32_t* block_len, int B, int S, int H, int nblk, void* d_gate,
                                   const int64_t* dg_strides, void* d_out_c, void* d_out_c_t, int64_t ldt, void* stream) {
  return combine_bwd<false>(dO, do_strides, gate, g_strides, out_c, block_len, B, S, H, nblk, d_gate, dg_strides, d_out_c,
                            d_out_c_t, ldt, stream);
}

extern "C" int fvb_vsa_combine_bwd_compact(const void* dO, const int64_t* do_strides, const void* gate,
                                           const int64_t* g_strides, const void* out_c, const int32_t* block_off, int B, int S,
                                           int H, int nblk, void* d_gate, const int64_t* dg_strides, void* d_out_c,
                                           void* d_out_c_t, int64_t ldt, void* stream) {
  return combine_bwd<true>(dO, do_strides, gate, g_strides, out_c, block_off, B, S, H, nblk, d_gate, dg_strides, d_out_c,
                           d_out_c_t, ldt, stream);
}

extern "C" int fvb_softmax_rows_bwd(const void* p, const void* dp, int64_t ld, int batch, int n, float scale, void* ds,
                                    void* ds_t, void* p_t, void* stream) {
  FVB_CHECK_ARG(p && dp && ds && batch > 0 && n > 0 && n <= 8192, "bad arguments (n <= 8192)");
  FVB_CHECK_ARG(ld >= n && ld % 8 == 0, "ld must be >= n and a multiple of 8");
  const uintptr_t al = reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(dp) | reinterpret_cast<uintptr_t>(ds) |
                       reinterpret_cast<uintptr_t>(ds_t) | reinterpret_cast<uintptr_t>(p_t);
  FVB_CHECK_ARG((al & 15) == 0, "buffers must be 16-byte aligned");
  softmax_rows_bwd_kernel<<<dim3((n + SMB_ROWS - 1) / SMB_ROWS, batch), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const __nv_bfloat16*>(p), reinterpret_cast<const __nv_bfloat16*>(dp), ld, n, scale,
      reinterpret_cast<__nv_bfloat16*>(ds), reinterpret_cast<__nv_bfloat16*>(ds_t), reinterpret_cast<__nv_bfloat16*>(p_t));
  FVB_CHECK_CUDA(cudaGetLastError());
  return FVB_OK;
}

template <bool COMPACT>
static int mean_bwd(const void* dx_s, const int64_t* s_strides, const void* d_mean, const int32_t* block_tab,
                    const int32_t* row_block, int B, int H, int S, int nblk, void* dx, const int64_t* dx_strides, void* stream) {
  FVB_CHECK_ARG(dx_s && s_strides && d_mean && block_tab && dx && dx_strides && (!COMPACT || row_block), "null pointer");
  if (COMPACT)
    FVB_CHECK_ARG(B > 0 && H > 0 && nblk > 0 && S > 0, "empty problem");
  else
    FVB_CHECK_ARG(B > 0 && H > 0 && nblk > 0 && S == nblk * VSA_TILE, "S must be 64 * nblk (padded layout)");
  FVB_CHECK_ARG(strides_ok(s_strides) && strides_ok(dx_strides), "strides must be multiples of 8");
  const int64_t total = int64_t(B) * H * S * 16;
  block_mean_bwd_kernel<COMPACT><<<(unsigned)((total + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const __nv_bfloat16*>(dx_s), BwdStrides3{{s_strides[0], s_strides[1], s_strides[2]}},
      reinterpret_cast<const __nv_bfloat16*>(d_mean), block_tab, reinterpret_cast<__nv_bfloat16*>(dx),
      BwdStrides3{{dx_strides[0], dx_strides[1], dx_strides[2]}}, B, S, H, nblk, row_block);
  FVB_CHECK_CUDA(cudaGetLastError());
  return FVB_OK;
}

extern "C" int fvb_block_mean_bwd(const void* dx_s, const int64_t* s_strides, const void* d_mean, const int32_t* block_len,
                                  int B, int H, int S, int nblk, void* dx, const int64_t* dx_strides, void* stream) {
  return mean_bwd<false>(dx_s, s_strides, d_mean, block_len, nullptr, B, H, S, nblk, dx, dx_strides, stream);
}

extern "C" int fvb_block_mean_bwd_compact(const void* dx_s, const int64_t* s_strides, const void* d_mean,
                                          const int32_t* block_off, const int32_t* row_block, int B, int H, int S, int nblk,
                                          void* dx, const int64_t* dx_strides, void* stream) {
  return mean_bwd<true>(dx_s, s_strides, d_mean, block_off, row_block, B, H, S, nblk, dx, dx_strides, stream);
}
