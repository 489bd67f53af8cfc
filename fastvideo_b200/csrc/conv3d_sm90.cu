// conv3d_sm90.cu -- causal Conv3d / Conv2d of the Wan VAE decoder as a TMA-staged implicit GEMM on wgmma.
//
// Replaces WanCausalConv3d.forward (fastvideo/models/vaes/wanvae.py:160-207: causal time padding 2*pt, the
// <=2-frame feature cache prepended, then nn.Conv3d) and the nn.Conv2d of WanResample (wanvae.py:303-356).
//
// Layout: activations are channels-last frames, x[t][h][w][c] bf16, so the im2col matrix never exists:
//   M = output pixels of one frame (tile = 16 wide x 8 high = 128 GEMM rows),
//   K = (tap dt,dh,dw) x input channels, N = output channels.
// For every tap the A tile is ONE TMA box {BK channels, 16 w, 8 h, 1 frame} of the input at the shifted
// coordinate (c0, w0+dw-pw, h0+dh-ph, t+dt-(kt-1)); out-of-range coordinates (spatial "same" padding, causal
// time padding, an absent feature cache) are zero-filled by the TMA unit, and taps whose frame lies wholly before
// the start of the stream are skipped. Weights are pre-packed [Cout][tap][Cin_pad] (K-major), loaded by a 2D TMA.
// Pipeline / warp roles as in gemm_sm90.cu: warpgroup 0 TMA, warpgroups 1 and 2 wgmma on GEMM rows [0, 64) and [64, 128)
// with the epilogue (fused bias, + residual add, bf16 channels-last stores) straight from the accumulator registers.
// NORM instantiation (one N block covers every output channel): the epilogue also applies the CONSUMER's WanRMS_norm
// (+ SiLU) to the finished row -- the four threads of a quad hold one pixel's whole channel row -- and writes the normalised
// tensor next to (or instead of) the raw output, so the separate RMS-norm pass (a read + a write of the whole activation)
// disappears (wanvae.py:383-462: conv1 -> norm2 -> SiLU -> conv2; conv2 + shortcut -> next norm1).
// NORM == 2 writes that normalised tensor as e4m3 with a static per-tensor scale (the input of an FP8 convolution).
// FP8 instantiation: e4m3 activations and packed weights (one byte per channel), wgmma m64nNk32 .e4m3.e4m3 with both
// operands K-major; a k-block is one 32 / 64 / 128-byte swizzle row (32 / 64 / 128 channels). The MMAs accumulate straight
// into the fp32 accumulators (no second promotion set: it does not fit next to 96 accumulators at N = 192); the epilogue
// applies (acc * x_scale) * w_scale[n] before the bias, then runs the bf16 epilogue unchanged.
#include <cuda_fp8.h>

#include <type_traits>

#include "fvb_host.cuh"
#include "fvb_ptx.cuh"

namespace fvb {

constexpr int CONV_TW = 16, CONV_TH = 8;  // spatial tile -> 128 GEMM rows
constexpr int CONV_THREADS = 384;
constexpr int CONV_TAB_FLOATS = 512;  // per-CTA shared-memory table: the bias (and, fused norm, gamma) as fp32
// FP8: w_scale follows the bias, [512, 1024); with the fused norm at [2 BN, 3 BN)
template <bool FP8>
constexpr int conv_tab_floats() { return FP8 ? 2 * CONV_TAB_FLOATS : CONV_TAB_FLOATS; }

struct ConvParams {
  const __nv_bfloat16* bias;   // [Cout] or NULL
  const __nv_bfloat16* resid;  // [T_out][H][W][Cout] or NULL
  __nv_bfloat16* out;          // [T_out][H][W][out_ld] (channels-last, out_ld >= Cout)
  int64_t out_ld, resid_ld;
  int H, W, Cout, Cin_pad;
  int kt, kh, kw;      // kernel extent
  int interleave_c;    // > 0: output channel col goes to frame 2t + col / interleave_c, channel col % interleave_c
                       //      (the reshape/stack of WanResample upsample3d, wanvae.py:343-345)
  // fused consumer norm (NORM instantiation): normed = silu?(y / max(||y||, 1e-12) * sqrt(Cout) * gamma), y = the bf16 output row
  const float* norm_gamma;     // [Cout] fp32
  void* norm_out;              // [T_out][H][W][norm_ld] bf16 (NORM == 1) or e4m3 (NORM == 2)
  int64_t norm_ld;
  int norm_silu;
  int T_out;           // frames to produce
  int t_off;           // input buffer frame index of output frame 0's LAST tap (= number of cached frames present)
  int tiles_w, tiles_h, num_n, cblocks;
  float norm_qscale;   // NORM == 2: e4m3 norm output = satfinite(v * norm_qscale), norm_qscale = 448 / bound (0 when bound == 0)
};
// The FP8 instantiation's parameters: acc * x_scale * w_scale[n] dequantises the e4m3 products. (A separate type, so the
// bf16 kernels keep the parameter block -- and the code -- they had before the FP8 path existed.)
struct ConvParamsFp8 : ConvParams {
  const float* w_scale;  // [Cout] fp32
  float x_scale;
};
template <bool FP8>
using ConvParamsOf = std::conditional_t<FP8, ConvParamsFp8, ConvParams>;

// ROWB: bytes of one k-block row (BK channels) -> the swizzle mode of its TMA box and wgmma descriptor
template <int ROWB>
FVB_DEVICE uint64_t conv_desc(uint32_t smem_addr) {
  return ROWB == 128 ? make_desc_kmajor_sw128(smem_addr) : (ROWB == 64 ? make_desc_kmajor_sw64(smem_addr) : make_desc_kmajor_sw32(smem_addr));
}

// KSUB: channel blocks (BK channels each) of one tap that share a pipeline stage and ONE full/empty barrier pair. With
// Cin = 96 a k-block is 32 channels = two M=128, N=96 MMAs = 96 tensor-pipe cycles, less than the issuing thread needs for
// a barrier round trip: three sub-tiles per stage give the issuer 288 cycles of MMA work per wait.
template <bool FP8, int BN, int BK, int KSUB = 1>
struct ConvCfg {
  static constexpr int ESZ = FP8 ? 1 : 2;  // bytes per element
  static constexpr int ROWB = BK * ESZ;    // bytes per k-block row
  static constexpr int A_BYTES = 128 * ROWB;
  static constexpr int B_BYTES = BN * ROWB;
  static constexpr int B_BYTES_AL = (B_BYTES + 1023) / 1024 * 1024;
  static constexpr int SUB_BYTES = A_BYTES + B_BYTES_AL;
  static constexpr int STAGE_BYTES = KSUB * SUB_BYTES;
  static constexpr int STAGES = (200 * 1024 / STAGE_BYTES) > 8 ? 8 : (200 * 1024 / STAGE_BYTES);
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 + 256 + conv_tab_floats<FP8>() * 4;
};

// Fill the epilogue's table once per CTA (before the first __syncthreads): bias[0, min(Cout, 512)) as fp32, zero where there is
// none; with the fused norm (one N block, Cout <= 192) gamma follows at [BN, 2 BN). The epilogue reads it with broadcast
// LDS.128 instead of one LDG + convert per element under a per-element branch.
template <bool FP8, int BN, int NORM>
FVB_DEVICE void conv_fill_table(const ConvParamsOf<FP8>& p, float* tab) {
  if constexpr (NORM != 0) {
    for (int i = threadIdx.x; i < BN; i += blockDim.x) {
      tab[i] = (p.bias != nullptr && i < p.Cout) ? __bfloat162float(p.bias[i]) : 0.f;
      tab[BN + i] = i < p.Cout ? p.norm_gamma[i] : 0.f;
      if constexpr (FP8) tab[2 * BN + i] = i < p.Cout ? p.w_scale[i] : 0.f;
    }
  } else {
    for (int i = threadIdx.x; i < CONV_TAB_FLOATS; i += blockDim.x) {
      tab[i] = (p.bias != nullptr && i < p.Cout) ? __bfloat162float(p.bias[i]) : 0.f;
      if constexpr (FP8) tab[CONV_TAB_FLOATS + i] = i < p.Cout ? p.w_scale[i] : 0.f;
    }
  }
}

FVB_DEVICE float bf16_lo(uint32_t pk) { return __uint_as_float(pk << 16); }
FVB_DEVICE float bf16_hi(uint32_t pk) { return __uint_as_float(pk & 0xffff0000u); }

// The two accumulator rows of this thread (GEMM rows 16 warp + lane / 4 + 8 i of its warpgroup's 64) to global memory:
// bias, bf16 rounding (the conv's own output under autocast), residual, optional fused consumer norm. A thread holds the
// column pairs 8 j + 2 (lane % 4) of both rows; the four threads of a quad hold the whole row.
template <bool FP8, int BN, int NORM>
FVB_DEVICE void conv_epilogue(const ConvParamsOf<FP8>& p, const float* tab, float (&acc)[BN / 2], int n_blk, int t, const int (&ys)[2],
                              const int (&xs)[2], int lane) {
  const int tq = lane & 3;
  const bool pair_ok = (p.out == nullptr || ((p.out_ld & 1) == 0 && (reinterpret_cast<uintptr_t>(p.out) & 3) == 0)) &&
                       (p.interleave_c & 1) == 0;
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const bool ok = ys[i] < p.H && xs[i] < p.W;
    const int64_t pix = (int64_t(t) * p.H + ys[i]) * p.W + xs[i];
    float ss = 0.f;
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      const int lc = 8 * j + 2 * tq;  // column inside the N block
      const int col = n_blk * BN + lc;
      float y[2];
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        float b = 0.f;
        if (NORM || col + c < CONV_TAB_FLOATS) b = tab[NORM ? lc + c : col + c];
        else if (p.bias != nullptr && col + c < p.Cout) b = __bfloat162float(p.bias[col + c]);
        float a = acc[4 * j + 2 * i + c];
        if constexpr (FP8) {
          float ws = 0.f;
          if (NORM || col + c < CONV_TAB_FLOATS) ws = tab[NORM ? 2 * BN + lc + c : CONV_TAB_FLOATS + col + c];
          else if (col + c < p.Cout) ws = p.w_scale[col + c];
          a = __fmul_rn(__fmul_rn(a, p.x_scale), ws);
        }
        float v = bf16_round(__fadd_rn(a, b));
        if (p.resid != nullptr && ok && col + c < p.Cout) v = bf16_round(__fadd_rn(v, __bfloat162float(p.resid[pix * p.resid_ld + col + c])));
        y[c] = v;
      }
      acc[4 * j + 2 * i] = y[0];
      acc[4 * j + 2 * i + 1] = y[1];
      if constexpr (NORM != 0) {
        if (col < p.Cout) ss = fmaf(y[0], y[0], fmaf(y[1], y[1], ss));  // Cout % 8 == 0: both or neither
      }
      if (!ok || p.out == nullptr || col >= p.Cout) continue;
      __nv_bfloat16* op = p.out + pix * p.out_ld + col;
      if (p.interleave_c > 0) {
        const int hf = col / p.interleave_c;
        op = p.out + ((int64_t(2 * t + hf) * p.H + ys[i]) * p.W + xs[i]) * p.out_ld + (col - hf * p.interleave_c);
      }
      if (pair_ok && col + 1 < p.Cout) {
        *reinterpret_cast<uint32_t*>(op) = pack_bf16x2(y[0], y[1]);
      } else {
        op[0] = __float2bfloat16_rn(y[0]);
        if (col + 1 < p.Cout) op[1] = __float2bfloat16_rn(y[1]);
      }
    }
    if constexpr (NORM != 0) {
      ss += __shfl_xor_sync(0xffffffffu, ss, 1);
      ss += __shfl_xor_sync(0xffffffffu, ss, 2);
      if (!ok) continue;
      // y / max(||y||, 1e-12) * sqrt(C) as ONE multiplier per pixel instead of an IEEE division per element
      const float rn = __fmul_rn(__frcp_rn(fmaxf(sqrtf(ss), 1e-12f)), sqrtf(float(p.Cout)));
      __nv_bfloat16* np = static_cast<__nv_bfloat16*>(p.norm_out) + pix * p.norm_ld;
      uint8_t* nq = static_cast<uint8_t*>(p.norm_out) + pix * p.norm_ld;
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int col = 8 * j + 2 * tq;
        if (col >= p.Cout) continue;
        float r2[2];
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          float vv = __fmul_rn(__fmul_rn(acc[4 * j + 2 * i + c], rn), tab[BN + col + c]);
          if (p.norm_silu) vv = __fdividef(vv, 1.0f + __expf(-vv));
          r2[c] = vv;
        }
        if constexpr (NORM == 2) {
          *reinterpret_cast<__nv_fp8x2_storage_t*>(nq + col) = __nv_cvt_float2_to_fp8x2(
              make_float2(__fmul_rn(r2[0], p.norm_qscale), __fmul_rn(r2[1], p.norm_qscale)), __NV_SATFINITE, __NV_E4M3);
        } else {
          *reinterpret_cast<uint32_t*>(np + col) = pack_bf16x2(r2[0], r2[1]);
        }
      }
    }
  }
}

template <bool FP8, int BN, int BK, int NORM, int KSUB>
__global__ void __launch_bounds__(CONV_THREADS, 1)
conv3d_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmW, const ConvParamsOf<FP8> p) {
  using Cfg = ConvCfg<FP8, BN, BK, KSUB>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + Cfg::STAGES * Cfg::STAGE_BYTES);
  uint64_t* full = bars;
  uint64_t* empty = bars + Cfg::STAGES;
  float* tab = reinterpret_cast<float*>(bars) + 64;  // 256 bytes of barriers, then the epilogue's bias / gamma table

  const int wg = threadIdx.x >> 7;
  const int tiles_sp = p.tiles_w * p.tiles_h;
  const int num_tiles = tiles_sp * p.T_out * p.num_n;
  const int taps_sp = p.kh * p.kw;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmX);
    tma_prefetch_desc(&tmW);
    for (int i = 0; i < Cfg::STAGES; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], 8);  // lane 0 of each of the eight consumer warps
    }
    fence_mbar_init();
  }
  conv_fill_table<FP8, BN, NORM>(p, tab);
  __syncthreads();

  // tile -> (n block, frame, spatial tile); n fastest so neighbouring CTAs share the activation tile in L2
  auto decode = [&](int tile, int& n_blk, int& t, int& th, int& tw) {
    n_blk = tile % p.num_n;
    int r = tile / p.num_n;
    tw = r % p.tiles_w;
    r /= p.tiles_w;
    th = r % p.tiles_h;
    t = r / p.tiles_h;
  };
  // first time tap that can touch a real frame for output frame t (frames before the stream start are zeros)
  auto dt_first = [&](int t) { return max(0, (p.kt - 1) - (p.t_off + t)); };

  if (wg == 0) {
    reg_dealloc<40>();
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        int n_blk, t, th, tw;
        decode(tile, n_blk, t, th, tw);
        for (int dt = dt_first(t); dt < p.kt; ++dt) {
          const int tf = p.t_off + t + dt - (p.kt - 1);  // frame index inside the input buffer
          for (int sp = 0; sp < taps_sp; ++sp) {
            const int dh = sp / p.kw, dw = sp % p.kw;
            const int tap = dt * taps_sp + sp;
            for (int cb = 0; cb < p.cblocks; cb += KSUB) {
              mbar_wait(&empty[stage], phase ^ 1);
              mbar_expect_tx(&full[stage], KSUB * (Cfg::A_BYTES + Cfg::B_BYTES));
#pragma unroll
              for (int u = 0; u < KSUB; ++u) {
                uint8_t* sa = smem + stage * Cfg::STAGE_BYTES + u * Cfg::SUB_BYTES;
                uint8_t* sb = sa + Cfg::A_BYTES;
                tma_load_4d(sa, &tmX, &full[stage], (cb + u) * BK, tw * CONV_TW + dw - p.kw / 2, th * CONV_TH + dh - p.kh / 2, tf);
                tma_load_2d(sb, &tmW, &full[stage], tap * p.Cin_pad + (cb + u) * BK, n_blk * BN);
              }
              if (++stage == Cfg::STAGES) {
                stage = 0;
                phase ^= 1;
              }
            }
          }
        }
      }
    }
    return;
  }
  reg_alloc<232>();
  const int half = wg - 1;  // GEMM rows [64 half, 64 half + 64) of the tile
  const int warp = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  int stage = 0;
  uint32_t phase = 0;
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    int n_blk, t, th, tw;
    decode(tile, n_blk, t, th, tw);
    const int nkb = (p.kt - dt_first(t)) * taps_sp * (p.cblocks / KSUB);
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    int prev = -1;
    for (int kb = 0; kb < nkb; ++kb) {
      mbar_wait(&full[stage], phase);
      const uint32_t sa0 = smem_u32(smem + stage * Cfg::STAGE_BYTES);
      wgmma_fence();
#pragma unroll
      for (int u = 0; u < KSUB; ++u) {
        const uint64_t da = conv_desc<Cfg::ROWB>(sa0 + u * Cfg::SUB_BYTES + half * (64 * Cfg::ROWB));
        const uint64_t db = conv_desc<Cfg::ROWB>(sa0 + u * Cfg::SUB_BYTES + Cfg::A_BYTES);
        // one MMA per 32 B of the row (k16 bf16 / k32 e4m3): +2 on the descriptor = 32 B = 2 x 16 B
#pragma unroll
        for (int k = 0; k < Cfg::ROWB / 32; ++k) {
          if constexpr (FP8) wgmma_ss_e4m3<BN>(acc, da + uint64_t(2 * k), db + uint64_t(2 * k), 1);
          else wgmma_ss<BN>(acc, da + uint64_t(2 * k), db + uint64_t(2 * k));
        }
      }
      wgmma_commit();
      wgmma_wait<1>();
      if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);
      prev = stage;
      if (++stage == Cfg::STAGES) {
        stage = 0;
        phase ^= 1;
      }
    }
    wgmma_wait<0>();
    wgmma_fence_regs(acc);
    if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);
    int ys[2], xs[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int r = half * 64 + warp * 16 + (lane >> 2) + 8 * i;
      ys[i] = th * CONV_TH + r / CONV_TW;
      xs[i] = tw * CONV_TW + r % CONV_TW;
    }
    conv_epilogue<FP8, BN, NORM>(p, tab, acc, n_blk, t, ys, xs, lane);
  }
}

template <bool FP8, int BN, int BK, int NORM, int KSUB>
static int launch_conv_k(const CUtensorMap& tmX, const CUtensorMap& tmW, const ConvParamsOf<FP8>& p, cudaStream_t st) {
  using Cfg = ConvCfg<FP8, BN, BK, KSUB>;
  auto kern = conv3d_kernel<FP8, BN, BK, NORM, KSUB>;
  static bool configured = false;
  if (!configured) {
    FVB_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
    configured = true;
  }
  const int tiles = p.tiles_w * p.tiles_h * p.T_out * p.num_n;
  const int grid = tiles < sm_count() ? tiles : sm_count();
  kern<<<grid, CONV_THREADS, Cfg::SMEM_BYTES, st>>>(tmX, tmW, p);
  FVB_CHECK_CUDA(cudaGetLastError());
  return FVB_OK;
}

// 32-channel bf16 k-blocks (Cin not a multiple of 64): three of them per stage when the channel count allows (Cin = 96).
// e4m3 k-blocks shorter than 128 B (Cin = 96: 32 B, Cin = 192: 64 B) likewise.
template <bool FP8, int BN, int BK, int NORM = 0>
static int launch_conv(const CUtensorMap& tmX, const CUtensorMap& tmW, const ConvParamsOf<FP8>& p, cudaStream_t st) {
  if constexpr (FP8 ? BK < 128 : (BK == 32 && BN <= 128)) {
    if (p.cblocks % 3 == 0) return launch_conv_k<FP8, BN, BK, NORM, 3>(tmX, tmW, p, st);
  }
  return launch_conv_k<FP8, BN, BK, NORM, 1>(tmX, tmW, p, st);
}

}  // namespace fvb

using namespace fvb;

// fp8: x / w_packed are e4m3 with x_scale / w_scale. norm_e4m3: the fused norm output is e4m3 with the static bound.
static int conv3d_impl(const void* x, int T_in, int H, int W, int Cin, const void* w_packed, int Cin_pad, int Cout,
                       int kt, int kh, int kw, const void* bias, const void* resid, int64_t resid_ld, void* out,
                       int64_t out_ld, int T_out, int t_off, int interleave_c, const float* norm_gamma, void* norm_out,
                       int64_t norm_ld, int norm_silu, void* stream, bool fp8 = false, float x_scale = 1.f,
                       const float* w_scale = nullptr, bool norm_e4m3 = false, float norm_bound = 0.f) {
  FVB_CHECK_ARG(x && w_packed && (out || norm_out), "null pointer");
  if (norm_gamma != nullptr || norm_out != nullptr) {
    FVB_CHECK_ARG(norm_gamma && norm_out, "norm_gamma and norm_out come together");
    FVB_CHECK_ARG(Cout > 16 && Cout <= 192 && Cout % 8 == 0, "fused norm needs 16 < Cout <= 192 (one N block), Cout % 8 == 0");
    FVB_CHECK_ARG(interleave_c == 0, "fused norm cannot be combined with interleave_c");
    FVB_CHECK_ARG(norm_ld >= Cout && norm_ld % 8 == 0 && (out == nullptr || out_ld % 8 == 0) && (resid == nullptr || resid_ld % 8 == 0),
                  "fused norm needs 16-byte aligned rows");
    FVB_CHECK_ARG((reinterpret_cast<uintptr_t>(out) & 15) == 0 && (reinterpret_cast<uintptr_t>(norm_out) & 15) == 0 &&
                      (reinterpret_cast<uintptr_t>(resid) & 15) == 0,
                  "fused norm needs 16-byte aligned base pointers");
    FVB_CHECK_ARG(!norm_e4m3 || (norm_bound >= 0.f && norm_ld % 16 == 0), "e4m3 norm output needs bound >= 0 and norm_ld % 16 == 0");
  }
  FVB_CHECK_ARG(T_in > 0 && H > 0 && W > 0 && Cin > 0 && Cout > 0 && T_out > 0, "bad shape");
  if (fp8) {
    FVB_CHECK_ARG(w_scale != nullptr, "fp8 convolution needs w_scale");
    FVB_CHECK_ARG(Cin % 16 == 0, "fp8 convolution needs Cin % 16 == 0 (16-byte e4m3 channel rows)");
    FVB_CHECK_ARG(interleave_c == 0, "fp8 convolution has no interleave_c");
  }
  FVB_CHECK_ARG(Cin % 8 == 0, "Cin must be a multiple of 8 (16-byte channel rows)");
  FVB_CHECK_ARG((kt == 1 || kt == 3) && (kh == 1 || kh == 3) && kh == kw, "kernel must be (1|3) x (1x1|3x3)");
  FVB_CHECK_ARG(t_off >= 0 && t_off + T_out <= T_in, "t_off + T_out must fit in the input buffer");
  // k-block = one swizzle row: bf16 64 channels (128 B) or 32 (64 B); e4m3 128, 64 or 32 channels (128 / 64 / 32 B)
  const int BK = fp8 ? (Cin_pad % 128 == 0 ? 128 : (Cin_pad % 64 == 0 ? 64 : 32)) : ((Cin_pad % 64 == 0) ? 64 : 32);
  const int ROWB = fp8 ? BK : 2 * BK;
  const CUtensorMapSwizzle swz = ROWB == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : (ROWB == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B);
  const uint64_t esz = fp8 ? 1 : 2;
  FVB_CHECK_ARG(Cin_pad % 32 == 0 && Cin_pad >= Cin, "Cin_pad must be a multiple of 32 covering Cin");
  FVB_CHECK_ARG((out == nullptr || out_ld >= (interleave_c > 0 ? interleave_c : Cout)) && (resid == nullptr || resid_ld >= Cout), "leading dimensions too small");
  const int ntaps = kt * kh * kw;
  // N tile: one block of up to 192 columns (wgmma N = 192: 96 fp32 accumulator registers per thread)
  const int BN = Cout > 128 ? 192 : (Cout > 96 ? 128 : (Cout > 16 ? 96 : 16));

  CUtensorMap tmX, tmW;
  {
    uint64_t dims[4] = {(uint64_t)Cin, (uint64_t)W, (uint64_t)H, (uint64_t)T_in};
    uint64_t str[4] = {esz, (uint64_t)Cin * esz, (uint64_t)W * Cin * esz, (uint64_t)H * W * Cin * esz};
    uint32_t box[4] = {(uint32_t)BK, CONV_TW, CONV_TH, 1};
    int r = fp8 ? make_tmap_u8(&tmX, x, 4, dims, str, box, swz) : make_tmap_bf16(&tmX, x, 4, dims, str, box, swz);
    if (r) return r;
  }
  {
    uint64_t dims[2] = {(uint64_t)ntaps * Cin_pad, (uint64_t)Cout};
    uint64_t str[2] = {esz, (uint64_t)ntaps * Cin_pad * esz};
    uint32_t box[2] = {(uint32_t)BK, (uint32_t)BN};
    int r = fp8 ? make_tmap_u8(&tmW, w_packed, 2, dims, str, box, swz) : make_tmap_bf16(&tmW, w_packed, 2, dims, str, box, swz);
    if (r) return r;
  }
  ConvParamsFp8 p;
  p.bias = reinterpret_cast<const __nv_bfloat16*>(bias);
  p.resid = reinterpret_cast<const __nv_bfloat16*>(resid);
  p.out = reinterpret_cast<__nv_bfloat16*>(out);
  p.out_ld = out_ld;
  p.resid_ld = resid_ld;
  p.H = H;
  p.W = W;
  p.Cout = Cout;
  p.Cin_pad = Cin_pad;
  p.kt = kt;
  p.kh = kh;
  p.kw = kw;
  p.T_out = T_out;
  p.t_off = t_off;
  p.interleave_c = interleave_c;
  p.norm_gamma = norm_gamma;
  p.norm_out = norm_out;
  p.norm_ld = norm_ld;
  p.norm_silu = norm_silu;
  p.w_scale = w_scale;
  p.x_scale = x_scale;
  p.norm_qscale = norm_bound > 0.f ? 448.0f / norm_bound : 0.f;
  FVB_CHECK_ARG(interleave_c == 0 || (interleave_c % 32 == 0 && Cout == 2 * interleave_c && resid == nullptr),
                "interleave_c must be Cout/2, a multiple of 32, without residual");
  p.tiles_w = (W + CONV_TW - 1) / CONV_TW;
  p.tiles_h = (H + CONV_TH - 1) / CONV_TH;
  p.num_n = (Cout + BN - 1) / BN;
  p.cblocks = Cin_pad / BK;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int norm = norm_gamma == nullptr ? 0 : (norm_e4m3 ? 2 : 1);
  if (fp8) {
#define FVB_CONV8_NORM_CASE(bn, nm)                                           \
  if (BN == bn && norm == nm) {                                               \
    if (BK == 128) return launch_conv<true, bn, 128, nm>(tmX, tmW, p, st);    \
    if (BK == 64) return launch_conv<true, bn, 64, nm>(tmX, tmW, p, st);      \
    return launch_conv<true, bn, 32, nm>(tmX, tmW, p, st);                    \
  }
    FVB_CONV8_NORM_CASE(192, 1)
    FVB_CONV8_NORM_CASE(128, 1)
    FVB_CONV8_NORM_CASE(96, 1)
    FVB_CONV8_NORM_CASE(192, 2)
    FVB_CONV8_NORM_CASE(128, 2)
    FVB_CONV8_NORM_CASE(96, 2)
    FVB_CONV8_NORM_CASE(192, 0)
    FVB_CONV8_NORM_CASE(128, 0)
    FVB_CONV8_NORM_CASE(96, 0)
    FVB_CONV8_NORM_CASE(16, 0)
#undef FVB_CONV8_NORM_CASE
    return set_error(FVB_ERR_UNSUPPORTED, "no fp8 conv tile for this Cout%s");
  }
#define FVB_CONV_NORM_CASE(bn)                                              \
  if (BN == bn && norm == 1) {                                              \
    if (BK == 64) return launch_conv<false, bn, 64, 1>(tmX, tmW, p, st);    \
    return launch_conv<false, bn, 32, 1>(tmX, tmW, p, st);                  \
  }                                                                         \
  if (BN == bn && norm == 2) {                                              \
    if (BK == 64) return launch_conv<false, bn, 64, 2>(tmX, tmW, p, st);    \
    return launch_conv<false, bn, 32, 2>(tmX, tmW, p, st);                  \
  }
  FVB_CONV_NORM_CASE(192)
  FVB_CONV_NORM_CASE(128)
  FVB_CONV_NORM_CASE(96)
#undef FVB_CONV_NORM_CASE
#define FVB_CONV_CASE(bn)                                            \
  if (BN == bn) {                                                    \
    if (BK == 64) return launch_conv<false, bn, 64>(tmX, tmW, p, st); \
    return launch_conv<false, bn, 32>(tmX, tmW, p, st);              \
  }
  FVB_CONV_CASE(192)
  FVB_CONV_CASE(128)
  FVB_CONV_CASE(96)
  FVB_CONV_CASE(16)
#undef FVB_CONV_CASE
  return set_error(FVB_ERR_UNSUPPORTED, "no conv tile for this Cout%s");
}

extern "C" int fvb_conv3d_cl(const void* x, int T_in, int H, int W, int Cin, const void* w_packed, int Cin_pad, int Cout,
                             int kt, int kh, int kw, const void* bias, const void* resid, int64_t resid_ld, void* out,
                             int64_t out_ld, int T_out, int t_off, int interleave_c, void* stream) {
  FVB_CHECK_ARG(out != nullptr, "null pointer");
  return conv3d_impl(x, T_in, H, W, Cin, w_packed, Cin_pad, Cout, kt, kh, kw, bias, resid, resid_ld, out, out_ld, T_out, t_off,
                     interleave_c, nullptr, nullptr, 0, 0, stream);
}

extern "C" int fvb_conv3d_cl_norm(const void* x, int T_in, int H, int W, int Cin, const void* w_packed, int Cin_pad, int Cout,
                                  int kt, int kh, int kw, const void* bias, const void* resid, int64_t resid_ld, void* out,
                                  int64_t out_ld, int T_out, int t_off, const float* norm_gamma, void* norm_out,
                                  int64_t norm_ld, int norm_silu, void* stream) {
  FVB_CHECK_ARG(norm_gamma && norm_out, "null pointer");
  return conv3d_impl(x, T_in, H, W, Cin, w_packed, Cin_pad, Cout, kt, kh, kw, bias, resid, resid_ld, out, out_ld, T_out, t_off, 0,
                     norm_gamma, norm_out, norm_ld, norm_silu, stream);
}

extern "C" int fvb_conv3d_cl_norm_e4m3(const void* x, int T_in, int H, int W, int Cin, const void* w_packed, int Cin_pad,
                                       int Cout, int kt, int kh, int kw, const void* bias, const void* resid, int64_t resid_ld,
                                       void* out, int64_t out_ld, int T_out, int t_off, const float* norm_gamma, void* norm_out,
                                       int64_t norm_ld, int norm_silu, float norm_bound, void* stream) {
  FVB_CHECK_ARG(norm_gamma && norm_out, "null pointer");
  return conv3d_impl(x, T_in, H, W, Cin, w_packed, Cin_pad, Cout, kt, kh, kw, bias, resid, resid_ld, out, out_ld, T_out, t_off, 0,
                     norm_gamma, norm_out, norm_ld, norm_silu, stream, false, 1.f, nullptr, true, norm_bound);
}

extern "C" int fvb_conv3d_cl_fp8(const void* x, int T_in, int H, int W, int Cin, float x_scale, const void* w_packed,
                                 const float* w_scale, int Cin_pad, int Cout, int kt, int kh, int kw, const void* bias,
                                 const void* resid, int64_t resid_ld, void* out, int64_t out_ld, int T_out, int t_off,
                                 void* stream) {
  FVB_CHECK_ARG(out != nullptr, "null pointer");
  return conv3d_impl(x, T_in, H, W, Cin, w_packed, Cin_pad, Cout, kt, kh, kw, bias, resid, resid_ld, out, out_ld, T_out, t_off, 0,
                     nullptr, nullptr, 0, 0, stream, true, x_scale, w_scale);
}

extern "C" int fvb_conv3d_cl_fp8_norm(const void* x, int T_in, int H, int W, int Cin, float x_scale, const void* w_packed,
                                      const float* w_scale, int Cin_pad, int Cout, int kt, int kh, int kw, const void* bias,
                                      const void* resid, int64_t resid_ld, void* out, int64_t out_ld, int T_out, int t_off,
                                      const float* norm_gamma, void* norm_out, int64_t norm_ld, int norm_silu, int norm_e4m3,
                                      float norm_bound, void* stream) {
  FVB_CHECK_ARG(norm_gamma && norm_out, "null pointer");
  return conv3d_impl(x, T_in, H, W, Cin, w_packed, Cin_pad, Cout, kt, kh, kw, bias, resid, resid_ld, out, out_ld, T_out, t_off, 0,
                     norm_gamma, norm_out, norm_ld, norm_silu, stream, true, x_scale, w_scale, norm_e4m3 != 0, norm_bound);
}
