// gemm_sm90.cu -- persistent, warp-specialised GEMM for sm_90a, bf16, fp8 (e4m3), int8-weight or int8 x int8 operands:
//   out = epilogue(x[M,K] @ w[N,K]^T + bias)                                   (bf16)
//   out = epilogue((x_q[M,K] @ w_q[N,K]^T) * x_scale[m] * w_scale[n] + bias)   (e4m3, per-row / per-channel scales)
//   out = epilogue((x[M,K] @ w_q[N,K]^T) * w_scale[n] + bias)                  (bf16 x, int8 w, per-channel scales)
//   out = epilogue((x_q[M,K] @ w_q[N,K]^T) * x_scale[m] * w_scale[n] + bias)   (int8 x and w, s32 accumulators)
// TMA (128B swizzle) -> shared-memory ring -> wgmma (two warpgroups, 64 rows x BN each, fp32 accumulators in registers)
// -> epilogue straight from the accumulator registers with fused bias / GELU(tanh) / gated residual.
// A k-block is one 128-byte swizzle row of both operands: 64 bf16 or 128 e4m3 elements, so a stage holds the same bytes
// for both types. The e4m3 tensor-core accumulator keeps fewer bits than fp32, so the fp8 path lets each k-block's MMAs
// accumulate into a second register set and adds that into the fp32 accumulators once per k-block (every 128 elements).
// The int8-weight path (W8) runs the bf16 MMAs: each k-block's BN x 64 int8 weight tile lands, unswizzled, in the second
// half of the stage's bf16 B region, and warps 1-3 of the producer warpgroup widen it in place to the 128B-swizzled
// bf16 tile the B descriptor reads. int8 -> bf16 is exact, so the products are those of a bf16 GEMM on integer weights.
// The int8 x int8 path (I8, W8A8) loads both operands like the fp8 path (128-element k-blocks, 128B swizzle) and runs
// s8 MMAs into s32 accumulators. |acc| <= 127^2 K fits in s32 for K <= FVB_I8_MAX_K, so the sums are exact and need no
// promotion registers: the tile widths and the one-k-block-in-flight mainloop are the bf16 path's.
// Transposed operands (TA / TB, bf16 only: the backward of the bf16 linear): an MN-major operand is stored [K][MN] with MN
// contiguous and lands as 64-element x 64-row TMA boxes (128B swizzle), one 8 KB box per 64-wide MN chunk, chunk-major in
// the stage, so a stage holds the same bytes as the K-major tile. wgmma reads it with imm-trans set:
//   dgrad dx[M,K] = dy[M,N] . w[N,K]  -> A = dy (K-major), B = w (MN-major)              (TB)
//   wgrad dw[N,K] = dy^T . x           -> A = dy^T (MN-major), B = x (MN-major), over M  (TA, TB)
//
// Stands behind fastvideo/layers/linear.py:146-156 (F.linear) and the elementwise op that follows
// each linear in fastvideo/models/dits/wanvideo.py:394-431; rounding points mirror the reference's
// eager bf16 path (see include/fvb200.h).
//
// Warp roles (384 threads): warpgroup 0 = TMA producer (one thread issues; on the W8 path warps 1-3 widen the weights),
// warpgroups 1 and 2 = MMA + epilogue for rows [0, 64) and [64, 128) of the 128-row tile. The producer runs ahead into the next tile while the consumers finish the
// epilogue of the current one.
// Persistent CTAs walk the tiles in weight-stripe order (tile_coords): a stripe of 8 column tiles stays in L2 while
// the row-blocks stream past it. Output column blocks may be redirected by an offset table (out_col_offsets), which
// is how the sequence-parallel paths write heads straight into send / peer receive buffers.
#include <cstdlib>
#include <type_traits>
#include "fvb_host.cuh"
#include "fvb_ptx.cuh"

namespace fvb {

constexpr int GEMM_BM = 128;
constexpr int GEMM_BK = 64;   // 64 bf16 = one 128B swizzle row
constexpr int GEMM_BK_FP8 = 128;  // 128 e4m3 / int8 = one 128B swizzle row
constexpr int FVB_I8_MAX_K = 133144;  // 127^2 * 133144 < 2^31
constexpr int GEMM_THREADS = 384;
constexpr int GEMM_GROUP_M = 8;
constexpr int GEMM_MN_CHUNK = 64;                         // MN-major operands: elements per 128B swizzle row
constexpr int GEMM_MN_CHUNK_BYTES = GEMM_MN_CHUNK * GEMM_BK * 2;  // one 64 x 64 bf16 box: 8 KB

struct GemmParams {
  const __nv_bfloat16* bias;
  void* out;
  const __nv_bfloat16* resid;
  const float* gate;
  int gate_rows;        // 0: one gate vector; > 0: rows [i*gate_rows, (i+1)*gate_rows) use gate + i*gate_stride
  int64_t gate_stride;
  int64_t ldo, ldr;
  int64_t out_batch_stride;  // elements between batches of `out`
  const int64_t* out_col_offsets;  // optional: element offset of each 128-column block of `out` (row stride ldo)
  int a_seg_len;                   // K is split in segments of this many elements (== K: plain row-major A)
  float div;                 // FVB_EPI_DIV divisor
  int M, N, K;
  int num_m, num_n, num_k;
  int batch;
  int stripe_n;  // > 0: weight-stripe raster with this many column tiles per stripe (see tile_coords)
};

// e4m3 / int8 operands: the per-row / per-channel scales (a_scale: e4m3 and int8 x int8 only). The bf16 kernels keep
// taking the plain GemmParams.
struct GemmParamsFp8 : GemmParams {
  const float* a_scale;  // [M]
  const float* b_scale;  // [N_valid]
  int N_valid;           // columns with a b_scale entry (N before rounding up to 8)
};
template <bool SCALED>
using GemmParamsT = std::conditional_t<SCALED, GemmParamsFp8, GemmParams>;

template <int BN>
struct GemmCfg {
  static constexpr int A_BYTES = GEMM_BM * GEMM_BK * 2;  // 16 KB
  static constexpr int B_BYTES = BN * GEMM_BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int STAGES = (BN == 256) ? 4 : (BN == 128 ? 6 : 8);
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
};

FVB_DEVICE void tile_coords(int tile, int num_m, int num_n, int stripe_n, int& m_blk, int& n_blk) {
  if (stripe_n > 0) {
    // weight-stripe raster: sweep every row-block against a stripe of `stripe_n` weight tiles before moving to the next
    // stripe. The stripe (stripe_n x BN x K) is re-touched by every wave and stays in L2 while activations stream
    // through once per stripe; with the row-group raster below, the streaming output / residual traffic kept evicting
    // the weights and each wave re-read them from HBM.
    const int per_stripe = stripe_n * num_m;
    const int sidx = tile / per_stripe;
    const int first_n = sidx * stripe_n;
    const int ssz = min(stripe_n, num_n - first_n);
    const int r = tile - sidx * per_stripe;
    n_blk = first_n + r % ssz;
    m_blk = r / ssz;
    return;
  }
  // grouped raster: GEMM_GROUP_M row-blocks share the same stripe of weight tiles in L2
  const int per_group = GEMM_GROUP_M * num_n;
  const int g = tile / per_group;
  const int first_m = g * GEMM_GROUP_M;
  const int gsz = min(GEMM_GROUP_M, num_m - first_m);
  const int r = tile - g * per_group;
  m_blk = first_m + r % gsz;
  n_blk = r / gsz;
}

FVB_DEVICE float gelu_tanh_f(float x) {
  // 0.5 x (1 + tanh(sqrt(2/pi) (x + 0.044715 x^3))), tanh(u) = 1 - 2/(exp(2u)+1)
  const float k0 = 0.7978845608028654f, k1 = 0.044715f;
  float u = k0 * (x + k1 * x * x * x);
  float e = ex2(u * 2.885390081777927f);  // exp(2u)
  float t = 1.0f - __fdividef(2.0f, e + 1.0f);
  return 0.5f * x * (1.0f + t);
}

FVB_DEVICE float gelu_tanh_grad_f(float x) {
  // d/dx of gelu_tanh_f, with the same t: 0.5 (1 + t) + 0.5 x (1 - t^2) sqrt(2/pi) (1 + 3 * 0.044715 x^2)
  const float k0 = 0.7978845608028654f, k1 = 0.044715f;
  float u = k0 * (x + k1 * x * x * x);
  float e = ex2(u * 2.885390081777927f);
  float t = 1.0f - __fdividef(2.0f, e + 1.0f);
  return 0.5f * (1.0f + t) + 0.5f * x * (1.0f - t * t) * k0 * (1.0f + 3.0f * k1 * x * x);
}

// W8: the int8 weight tile (BN rows of 64 bytes) sits in the upper half of the stage's bf16 B region
template <int BN>
constexpr int W8_STAGING_OFFSET = BN * GEMM_BK;
constexpr int W8_CONVERT_THREADS = 96;  // warps 1-3 of the producer warpgroup

FVB_DEVICE uint4 lds128(uint32_t addr) {
  uint4 v;
  asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr) : "memory");
  return v;
}
FVB_DEVICE void sts128(uint32_t addr, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
  asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}

// Widen one stage's int8 weight tile into the 128B-swizzled bf16 K-major tile the wgmma B descriptor reads, in place.
// Unit u = 16 int8 weights (row u / 4, k [16 (u % 4), +16)) -> two 16-byte bf16 chunks of that row. Output row r covers
// staging rows 2r - BN and 2r - BN + 1, which are <= r, so rows are processed in ascending batches: every thread loads its
// units of the batch, the 96 threads meet at a named barrier, then they store; a batch never overwrites staging rows of
// a later batch. sb: shared-space address of the stage's B region.
template <int BN>
FVB_DEVICE void w8_widen_tile(uint32_t sb, int t) {
  constexpr int UNITS = BN * 4, PER = 2;  // units per thread per batch
  const uint32_t stg = sb + W8_STAGING_OFFSET<BN>;
#pragma unroll 1  // the producer warpgroup runs with 40 registers
  for (int u0 = 0; u0 < UNITS; u0 += PER * W8_CONVERT_THREADS) {
    uint4 v[PER];
#pragma unroll
    for (int p = 0; p < PER; ++p) {
      const int u = u0 + p * W8_CONVERT_THREADS + t;
      if (u < UNITS) v[p] = lds128(stg + u * 16);
    }
    named_bar_sync(1, W8_CONVERT_THREADS);
#pragma unroll
    for (int p = 0; p < PER; ++p) {
      const int u = u0 + p * W8_CONVERT_THREADS + t;
      if (u >= UNITS) continue;
      const int r = u >> 2, q = u & 3;
      const uint32_t w[4] = {v[p].x, v[p].y, v[p].z, v[p].w};
      uint32_t o[8];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        // int8 b -> fp32 exactly: the float with bits 0x4B0000uu (u = b ^ 0x80) is 2^23 + b + 128. |b| <= 128 has at
        // most 8 significant bits, so its bf16 is the upper half of the fp32 bits (no rounding needed)
        const uint32_t x = w[i] ^ 0x80808080u;
        uint32_t f[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) f[j] = __float_as_uint(__uint_as_float(__byte_perm(x, 0x4B000000u, 0x7440 + j)) - 8388736.f);
        o[2 * i] = __byte_perm(f[0], f[1], 0x7632);
        o[2 * i + 1] = __byte_perm(f[2], f[3], 0x7632);
      }
      const uint32_t row = sb + r * 128;
      sts128(row + (((2 * q) ^ (r & 7)) << 4), o[0], o[1], o[2], o[3]);
      sts128(row + (((2 * q + 1) ^ (r & 7)) << 4), o[4], o[5], o[6], o[7]);
    }
  }
}

FVB_DEVICE float acc_f32(float v) { return v; }
FVB_DEVICE float acc_f32(int32_t v) { return __int2float_rn(v); }

// FP8: e4m3 x e4m3 operands; W8: bf16 x int8 (weight-only); I8: int8 x int8 (W8A8); none: bf16 x bf16.
// TA / TB: A / B is MN-major (bf16 x bf16 only).
// Epilogue of the dgrad GEMM only (fvb_linear_dgrad_gelu_bf16): dx = bf16(bf16(acc) * gelu_tanh'(h)), h read through resid.
constexpr int EPI_DGELU_TANH = 100;

// fvb_linear_bf16_aux: the bf16 y = bf16(acc + bias) of every element is also stored to aux[row * ldaux + col]. A template
// so that the kernel body's e4m3 / int8 branches, discarded for it, stay dependent.
template <bool SCALED = false>
struct GemmParamsAuxT : GemmParams {
  __nv_bfloat16* aux;
  int64_t ldaux;
};
using GemmParamsAux = GemmParamsAuxT<>;

template <int BN, int EPI, bool FP8, bool W8 = false, bool I8 = false, bool TA = false, bool TB = false>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GemmParamsT<FP8 || W8 || I8> p) {
  constexpr bool AUX = false;
#include "gemm_kernel_body.cuh"
}

template <int BN, int EPI, bool FP8 = false, bool W8 = false, bool I8 = false, bool TA = false, bool TB = false>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_aux_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                const GemmParamsAuxT<FP8 || W8 || I8> p) {
  static_assert(!(FP8 || W8 || I8 || TA || TB), "the aux epilogues are bf16 forward GEMMs");
  constexpr bool AUX = true;
#include "gemm_kernel_body.cuh"
}

template <int BN, int EPI, bool FP8, bool W8 = false, bool I8 = false, bool TA = false, bool TB = false>
static int launch_gemm(const CUtensorMap& tmA, const CUtensorMap& tmB, const GemmParamsT<FP8 || W8 || I8>& p, cudaStream_t st) {
  using Cfg = GemmCfg<BN>;
  auto kern = gemm_kernel<BN, EPI, FP8, W8, I8, TA, TB>;
  static bool configured = false;
  if (!configured) {
    FVB_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
    configured = true;
  }
  const int tiles = p.num_m * p.num_n * p.batch;
  const int grid = tiles < sm_count() ? tiles : sm_count();
  kern<<<grid, GEMM_THREADS, Cfg::SMEM_BYTES, st>>>(tmA, tmB, p);
  FVB_CHECK_CUDA(cudaGetLastError());
  return FVB_OK;
}

template <int BN>
static int dispatch_epi(int epi, const CUtensorMap& a, const CUtensorMap& b, const GemmParams& p, cudaStream_t st) {
  switch (epi) {
    case FVB_EPI_BIAS: return launch_gemm<BN, FVB_EPI_BIAS, false>(a, b, p, st);
    case FVB_EPI_BIAS_GELU_TANH: return launch_gemm<BN, FVB_EPI_BIAS_GELU_TANH, false>(a, b, p, st);
    case FVB_EPI_RESID_GATE_F32: return launch_gemm<BN, FVB_EPI_RESID_GATE_F32, false>(a, b, p, st);
    case FVB_EPI_RESID_GATE_BF16: return launch_gemm<BN, FVB_EPI_RESID_GATE_BF16, false>(a, b, p, st);
    case FVB_EPI_RESID_GATE_BF16R: return launch_gemm<BN, FVB_EPI_RESID_GATE_BF16R, false>(a, b, p, st);
    case FVB_EPI_RESID_BF16: return launch_gemm<BN, FVB_EPI_RESID_BF16, false>(a, b, p, st);
    case FVB_EPI_DIV: return launch_gemm<BN, FVB_EPI_DIV, false>(a, b, p, st);
    case FVB_EPI_SCALE_F32: return launch_gemm<BN, FVB_EPI_SCALE_F32, false>(a, b, p, st);
  }
  return set_error(FVB_ERR_INVALID_ARG, "unknown epilogue%s");
}

template <int BN, int EPI>
static int launch_gemm_aux(const CUtensorMap& tmA, const CUtensorMap& tmB, const GemmParamsAux& p, cudaStream_t st) {
  using Cfg = GemmCfg<BN>;
  auto kern = gemm_aux_kernel<BN, EPI>;
  static bool configured = false;
  if (!configured) {
    FVB_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
    configured = true;
  }
  const int tiles = p.num_m * p.num_n;
  const int grid = tiles < sm_count() ? tiles : sm_count();
  kern<<<grid, GEMM_THREADS, Cfg::SMEM_BYTES, st>>>(tmA, tmB, p);
  FVB_CHECK_CUDA(cudaGetLastError());
  return FVB_OK;
}

// bf16 operands with the pre-epilogue y also stored (fvb_linear_bf16_aux): the epilogues whose y the block backward needs
template <int BN>
static int dispatch_epi_aux(int epi, const CUtensorMap& a, const CUtensorMap& b, const GemmParamsAux& p, cudaStream_t st) {
  switch (epi) {
    case FVB_EPI_BIAS_GELU_TANH: return launch_gemm_aux<BN, FVB_EPI_BIAS_GELU_TANH>(a, b, p, st);
    case FVB_EPI_RESID_GATE_F32: return launch_gemm_aux<BN, FVB_EPI_RESID_GATE_F32>(a, b, p, st);
    case FVB_EPI_RESID_GATE_BF16: return launch_gemm_aux<BN, FVB_EPI_RESID_GATE_BF16>(a, b, p, st);
    case FVB_EPI_RESID_GATE_BF16R: return launch_gemm_aux<BN, FVB_EPI_RESID_GATE_BF16R>(a, b, p, st);
  }
  return set_error(FVB_ERR_INVALID_ARG,
                   "fvb_linear_bf16_aux takes FVB_EPI_BIAS_GELU_TANH, _RESID_GATE_F32, _RESID_GATE_BF16 or _RESID_GATE_BF16R%s");
}

// fp8 / int8 operands: the public linear epilogues only (DIV / SCALE_F32 belong to bf16-only entry points)
template <int BN, bool FP8, bool W8, bool I8 = false>
static int dispatch_epi_scaled(int epi, const CUtensorMap& a, const CUtensorMap& b, const GemmParamsFp8& p, cudaStream_t st) {
  switch (epi) {
    case FVB_EPI_BIAS: return launch_gemm<BN, FVB_EPI_BIAS, FP8, W8, I8>(a, b, p, st);
    case FVB_EPI_BIAS_GELU_TANH: return launch_gemm<BN, FVB_EPI_BIAS_GELU_TANH, FP8, W8, I8>(a, b, p, st);
    case FVB_EPI_RESID_GATE_F32: return launch_gemm<BN, FVB_EPI_RESID_GATE_F32, FP8, W8, I8>(a, b, p, st);
    case FVB_EPI_RESID_GATE_BF16: return launch_gemm<BN, FVB_EPI_RESID_GATE_BF16, FP8, W8, I8>(a, b, p, st);
    case FVB_EPI_RESID_GATE_BF16R: return launch_gemm<BN, FVB_EPI_RESID_GATE_BF16R, FP8, W8, I8>(a, b, p, st);
    case FVB_EPI_RESID_BF16: return launch_gemm<BN, FVB_EPI_RESID_BF16, FP8, W8, I8>(a, b, p, st);
  }
  return set_error(FVB_ERR_INVALID_ARG, "unknown epilogue for fvb_linear_fp8 / fvb_linear_w8_sp / fvb_linear_w8a8_sp%s");
}

}  // namespace fvb

using namespace fvb;

static int gemm_impl(const void* x, int64_t ldx, int64_t x_batch, int a_seg_len, int64_t a_seg_stride, const void* w, int64_t ldw, int64_t w_batch,
                     const void* bias, void* out, int64_t ldo, int64_t o_batch, const int64_t* out_col_offsets,
                     const void* resid, int64_t ldr,
                     const float* gate, int gate_rows, int64_t gate_stride, float div, int M, int N, int K, int batch,
                     int epilogue, void* stream, const float* x_scale = nullptr, const float* w_scale = nullptr,
                     bool int8_operands = false, void* aux = nullptr, int64_t ldaux = 0) {
  // x_scale / w_scale set: x and w are e4m3 (one byte per element) with per-row / per-output-channel fp32 scales, or
  // int8 with the same scales when int8_operands is set.
  // w_scale alone: x is bf16 and w is int8 with per-output-channel fp32 scales.
  const bool i8 = x_scale != nullptr && int8_operands;
  const bool fp8 = x_scale != nullptr && !i8;
  const bool w8 = x_scale == nullptr && w_scale != nullptr;
  FVB_CHECK_ARG(x && w && out, "null pointer");
  FVB_CHECK_ARG(M > 0 && N > 0 && K > 0 && batch > 0, "empty problem");
  if (fp8) {
    FVB_CHECK_ARG(w_scale != nullptr, "w_scale required");
    FVB_CHECK_ARG(batch == 1 && a_seg_len <= 0 && out_col_offsets == nullptr, "fp8 operands: plain row-major, unbatched");
    FVB_CHECK_ARG(ldx % 16 == 0 && ldw % 16 == 0, "fp8 ldx/ldw must be multiples of 16 (16-byte rows)");
  }
  if (i8) {
    FVB_CHECK_ARG(w_scale != nullptr, "w_scale required");
    FVB_CHECK_ARG(batch == 1 && a_seg_len <= 0, "int8 operands: plain row-major, unbatched");
    FVB_CHECK_ARG(ldx % 16 == 0 && ldw % 16 == 0, "int8 ldx/ldw must be multiples of 16 (16-byte rows)");
    FVB_CHECK_ARG(K <= FVB_I8_MAX_K, "int8 operands: K > 133144 could overflow the s32 accumulator");
  }
  if (w8) {
    FVB_CHECK_ARG(batch == 1, "int8 weights: unbatched");
    FVB_CHECK_ARG(ldw % 16 == 0, "int8 ldw must be a multiple of 16 (16-byte rows)");
  }
  FVB_CHECK_ARG(ldx % 8 == 0 && ldw % 8 == 0 && ldo % 8 == 0, "ldx/ldw/ldo must be multiples of 8");
  // N not a multiple of 8: the tail columns up to the next multiple of 8 are written as zeros (they must fit in ldo)
  const int N_store = (N + 7) & ~7;
  FVB_CHECK_ARG(N_store <= ldo || N_store == N, "ldo must cover N rounded up to 8");
  if (N_store != N) FVB_CHECK_ARG(bias == nullptr && resid == nullptr && out_col_offsets == nullptr, "N must be a multiple of 8 when bias/residual/offsets are used");
  FVB_CHECK_ARG(x_batch % 8 == 0 && w_batch % 8 == 0 && o_batch % 8 == 0, "batch strides must be multiples of 8");
  const bool needs_resid = epilogue == FVB_EPI_RESID_GATE_F32 || epilogue == FVB_EPI_RESID_GATE_BF16 ||
                           epilogue == FVB_EPI_RESID_GATE_BF16R ||
                           epilogue == FVB_EPI_RESID_BF16;
  if (needs_resid) {
    FVB_CHECK_ARG(batch == 1, "residual epilogues are not batched");
    FVB_CHECK_ARG(resid != nullptr && ldr % 8 == 0, "residual required (ldr multiple of 8)");
    if (epilogue != FVB_EPI_RESID_BF16) {
      FVB_CHECK_ARG(gate != nullptr, "gate required");
      FVB_CHECK_ARG(gate_rows >= 0 && (gate_rows == 0 || gate_stride % 4 == 0), "bad gate grouping (stride must be a multiple of 4)");
    }
  }
  if (epilogue == FVB_EPI_DIV) FVB_CHECK_ARG(div != 0.f, "divisor must be non-zero");
  // fp8: the promotion registers double the accumulator footprint, so 128 columns is the widest tile that fits
  const int BN = fp8 ? (N >= 128 ? 128 : 64)
                     : (N >= 256 && N % 256 == 0) ? 256 : (N >= 128 && N % 128 == 0 ? 128 : (N >= 192 ? 256 : 64));
  const int BK = fp8 || i8 ? GEMM_BK_FP8 : GEMM_BK;
  const int esz = fp8 || i8 ? 1 : 2;  // operand element bytes
  const int wsz = fp8 || w8 || i8 ? 1 : 2;

  CUtensorMap tmA, tmB;
  if (a_seg_len <= 0 || a_seg_len >= K) {
    a_seg_len = K;
    a_seg_stride = 16;  // unused (single segment); any multiple of 16 elements
  }
  FVB_CHECK_ARG(a_seg_len % GEMM_BK == 0 || a_seg_len == K, "A segment length must be a multiple of 64");
  FVB_CHECK_ARG(K % a_seg_len == 0 && a_seg_stride % 8 == 0, "bad A segmentation");
  {
    uint64_t dims[4] = {(uint64_t)a_seg_len, (uint64_t)M, (uint64_t)(K / a_seg_len), (uint64_t)batch};
    uint64_t str[4] = {(uint64_t)esz, (uint64_t)ldx * esz, (uint64_t)a_seg_stride * esz,
                       batch > 1 ? (uint64_t)x_batch * esz : 16};  // unused dimension (size 1): any 16-byte multiple
    uint32_t box[4] = {(uint32_t)BK, GEMM_BM, 1, 1};
    int r = fp8 || i8 ? make_tmap_u8(&tmA, x, 4, dims, str, box) : make_tmap_bf16(&tmA, x, 4, dims, str, box);
    if (r) return r;
  }
  {
    uint64_t dims[3] = {(uint64_t)K, (uint64_t)N, (uint64_t)batch};
    uint64_t str[3] = {(uint64_t)wsz, (uint64_t)ldw * wsz, (uint64_t)(batch > 1 ? w_batch : ldw * (int64_t)N) * wsz};
    uint32_t box[3] = {(uint32_t)BK, (uint32_t)BN, 1};
    // int8 weights land unswizzled in a staging area and are widened into the swizzled bf16 layout in shared memory
    int r = fp8 || i8 ? make_tmap_u8(&tmB, w, 3, dims, str, box)
            : w8 ? make_tmap_u8(&tmB, w, 3, dims, str, box, CU_TENSOR_MAP_SWIZZLE_NONE)
                 : make_tmap_bf16(&tmB, w, 3, dims, str, box);
    if (r) return r;
  }
  GemmParamsFp8 p;  // the bf16 kernels receive its GemmParams part
  p.bias = reinterpret_cast<const __nv_bfloat16*>(bias);
  p.out = out;
  p.resid = reinterpret_cast<const __nv_bfloat16*>(resid);
  p.gate = gate;
  p.gate_rows = gate_rows;
  p.gate_stride = gate_stride;
  p.ldo = ldo;
  p.ldr = ldr;
  p.out_batch_stride = o_batch;
  p.out_col_offsets = out_col_offsets;
  p.a_seg_len = a_seg_len;
  p.div = div;
  p.a_scale = x_scale;
  p.b_scale = w_scale;
  p.N_valid = N;
  p.M = M;
  p.N = N_store;
  p.K = K;
  p.batch = batch;
  p.num_m = (M + GEMM_BM - 1) / GEMM_BM;
  p.num_n = (N + BN - 1) / BN;
  p.num_k = (K + BK - 1) / BK;
  static const int stripe_env = [] { const char* e = getenv("FVB_GEMM_STRIPE_N"); return e ? atoi(e) : -1; }();
  // default: stripes of 8 column tiles once the problem is tall enough for a stripe sweep to fill several waves
  p.stripe_n = stripe_env >= 0 ? stripe_env : 8;
  if (stripe_env > 0) {  // explicit setting (A/B runs): clamp to the column-tile count instead of falling back to the row-group raster
    p.stripe_n = p.num_m < 16 ? 0 : (stripe_env < p.num_n ? stripe_env : p.num_n);
  } else if (p.stripe_n > 0 && (p.num_m < 16 || p.num_n <= p.stripe_n)) {
    p.stripe_n = 0;
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (aux != nullptr) {
    GemmParamsAux pa;
    static_cast<GemmParams&>(pa) = p;
    pa.aux = reinterpret_cast<__nv_bfloat16*>(aux);
    pa.ldaux = ldaux;
    if (BN == 256) return dispatch_epi_aux<256>(epilogue, tmA, tmB, pa, st);
    if (BN == 128) return dispatch_epi_aux<128>(epilogue, tmA, tmB, pa, st);
    return dispatch_epi_aux<64>(epilogue, tmA, tmB, pa, st);
  }
  if (fp8)
    return BN == 128 ? dispatch_epi_scaled<128, true, false>(epilogue, tmA, tmB, p, st)
                     : dispatch_epi_scaled<64, true, false>(epilogue, tmA, tmB, p, st);
  if (i8) {
    if (BN == 256) return dispatch_epi_scaled<256, false, false, true>(epilogue, tmA, tmB, p, st);
    if (BN == 128) return dispatch_epi_scaled<128, false, false, true>(epilogue, tmA, tmB, p, st);
    return dispatch_epi_scaled<64, false, false, true>(epilogue, tmA, tmB, p, st);
  }
  if (w8) {
    if (BN == 256) return dispatch_epi_scaled<256, false, true>(epilogue, tmA, tmB, p, st);
    if (BN == 128) return dispatch_epi_scaled<128, false, true>(epilogue, tmA, tmB, p, st);
    return dispatch_epi_scaled<64, false, true>(epilogue, tmA, tmB, p, st);
  }
  if (BN == 256) return dispatch_epi<256>(epilogue, tmA, tmB, p, st);
  if (BN == 128) return dispatch_epi<128>(epilogue, tmA, tmB, p, st);
  return dispatch_epi<64>(epilogue, tmA, tmB, p, st);
}

extern "C" int fvb_linear_bf16(const void* x, int64_t ldx, const void* w, int64_t ldw, const void* bias, void* out,
                               int64_t ldo, const void* resid, int64_t ldr, const float* gate, int gate_rows,
                               int64_t gate_stride, int M, int N, int K, int epilogue, void* stream) {
  if (epilogue == FVB_EPI_DIV) return set_error(FVB_ERR_INVALID_ARG, "use fvb_gemm_batched_bf16 for FVB_EPI_DIV%s");
  return gemm_impl(x, ldx, 0, 0, 0, w, ldw, 0, bias, out, ldo, 0, nullptr, resid, ldr, gate, gate_rows, gate_stride, 1.0f,
                   M, N, K, 1, epilogue, stream);
}

extern "C" int fvb_linear_bf16_aux(const void* x, int64_t ldx, const void* w, int64_t ldw, const void* bias, void* out,
                                   int64_t ldo, const void* resid, int64_t ldr, const float* gate, int gate_rows,
                                   int64_t gate_stride, void* aux, int64_t ldaux, int M, int N, int K, int epilogue, void* stream) {
  FVB_CHECK_ARG(aux != nullptr && ldaux % 8 == 0 && ldaux >= N, "aux required (ldaux a multiple of 8, >= N)");
  FVB_CHECK_ARG(N % 8 == 0, "N must be a multiple of 8");
  return gemm_impl(x, ldx, 0, 0, 0, w, ldw, 0, bias, out, ldo, 0, nullptr, resid, ldr, gate, gate_rows, gate_stride, 1.0f,
                   M, N, K, 1, epilogue, stream, nullptr, nullptr, false, aux, ldaux);
}

extern "C" int fvb_linear_bf16_sp(const void* x, int64_t ldx, int x_seg_len, int64_t x_seg_stride, const void* w,
                                  int64_t ldw, const void* bias, void* out, int64_t ldo, const int64_t* out_col_offsets,
                                  const void* resid, int64_t ldr, const float* gate, int gate_rows, int64_t gate_stride,
                                  int M, int N, int K, int epilogue, void* stream) {
  if (epilogue == FVB_EPI_DIV) return set_error(FVB_ERR_INVALID_ARG, "use fvb_gemm_batched_bf16 for FVB_EPI_DIV%s");
  if (out_col_offsets != nullptr && N % 128 != 0) return set_error(FVB_ERR_INVALID_ARG, "column-block offsets need N %% 128 == 0%s");
  return gemm_impl(x, ldx, 0, x_seg_len, x_seg_stride, w, ldw, 0, bias, out, ldo, 0, out_col_offsets, resid, ldr, gate, gate_rows,
                   gate_stride, 1.0f, M, N, K, 1, epilogue, stream);
}

extern "C" int fvb_gemm_batched_bf16(const void* a, int64_t lda, int64_t a_batch_stride, const void* b, int64_t ldb,
                                     int64_t b_batch_stride, void* out, int64_t ldo, int64_t out_batch_stride, int M,
                                     int N, int K, int batch, float div, void* stream) {
  return gemm_impl(a, lda, a_batch_stride, 0, 0, b, ldb, b_batch_stride, nullptr, out, ldo, out_batch_stride, nullptr,
                   nullptr, 0, nullptr, 0, 0, div, M, N, K, batch, div != 0.f && div != 1.f ? FVB_EPI_DIV : FVB_EPI_BIAS, stream);
}

extern "C" int fvb_gemm_f32out(const void* a, int64_t lda, const void* b, int64_t ldb, float* out, int64_t ldo, int M, int N,
                               int K, float scale, void* stream) {
  return gemm_impl(a, lda, 0, 0, 0, b, ldb, 0, nullptr, out, ldo, 0, nullptr, nullptr, 0, nullptr, 0, 0, scale, M, N, K, 1,
                   FVB_EPI_SCALE_F32, stream);
}

extern "C" int fvb_linear_fp8(const void* xq, int64_t ldx, const float* x_scale, const void* wq, int64_t ldw,
                              const float* w_scale, const void* bias, void* out, int64_t ldo, const void* resid, int64_t ldr,
                              const float* gate, int gate_rows, int64_t gate_stride, int M, int N, int K, int epilogue,
                              void* stream) {
  if (x_scale == nullptr || w_scale == nullptr) return set_error(FVB_ERR_INVALID_ARG, "invalid argument: x_scale and w_scale are required%s");
  return gemm_impl(xq, ldx, 0, 0, 0, wq, ldw, 0, bias, out, ldo, 0, nullptr, resid, ldr, gate, gate_rows, gate_stride, 1.0f,
                   M, N, K, 1, epilogue, stream, x_scale, w_scale);
}

extern "C" int fvb_linear_w8_sp(const void* x, int64_t ldx, int x_seg_len, int64_t x_seg_stride, const void* wq, int64_t ldw,
                                const float* w_scale, const void* bias, void* out, int64_t ldo, const int64_t* out_col_offsets,
                                const void* resid, int64_t ldr, const float* gate, int gate_rows, int64_t gate_stride, int M,
                                int N, int K, int epilogue, void* stream) {
  if (w_scale == nullptr) return set_error(FVB_ERR_INVALID_ARG, "invalid argument: w_scale is required%s");
  if (out_col_offsets != nullptr && N % 128 != 0) return set_error(FVB_ERR_INVALID_ARG, "column-block offsets need N %% 128 == 0%s");
  return gemm_impl(x, ldx, 0, x_seg_len, x_seg_stride, wq, ldw, 0, bias, out, ldo, 0, out_col_offsets, resid, ldr, gate,
                   gate_rows, gate_stride, 1.0f, M, N, K, 1, epilogue, stream, nullptr, w_scale);
}

extern "C" int fvb_linear_w8a8_sp(const void* xq, int64_t ldx, const float* x_scale, const void* wq, int64_t ldw,
                                  const float* w_scale, const void* bias, void* out, int64_t ldo, const int64_t* out_col_offsets,
                                  const void* resid, int64_t ldr, const float* gate, int gate_rows, int64_t gate_stride, int M,
                                  int N, int K, int epilogue, void* stream) {
  if (x_scale == nullptr || w_scale == nullptr) return set_error(FVB_ERR_INVALID_ARG, "invalid argument: x_scale and w_scale are required%s");
  if (out_col_offsets != nullptr && N % 128 != 0) return set_error(FVB_ERR_INVALID_ARG, "column-block offsets need N %% 128 == 0%s");
  return gemm_impl(xq, ldx, 0, 0, 0, wq, ldw, 0, bias, out, ldo, 0, out_col_offsets, resid, ldr, gate, gate_rows, gate_stride,
                   1.0f, M, N, K, 1, epilogue, stream, x_scale, w_scale, true);
}

// ------------------------------------------------------------------------------------------------------------------------
// Backward of the bf16 linear y = x w^T + b (fvb_linear_dgrad_bf16 / fvb_linear_wgrad_bf16; arithmetic in include/fvb200.h).
// out[Mo, No] = bf16(sum_r A(mo, r) * B(r, no)) with fp32 accumulation, the plain FVB_EPI_BIAS store without bias. A is
// K-major [Mo][R] (a_mn_major = false) or MN-major [R][Mo] (true); B is always MN-major [R][No]. R tails are zero-filled by
// TMA, Mo tails are the epilogue's row check; No must be a multiple of 8 (whole bf16x2 column pairs, 16-byte rows).
// No split-K: every output element is one CTA's sum in k-block order, so two calls give the same bits.
// ------------------------------------------------------------------------------------------------------------------------
template <bool TA>
static int dispatch_bwd(int BN, const CUtensorMap& a, const CUtensorMap& b, const GemmParams& p, cudaStream_t st) {
  if (p.resid != nullptr) {  // dgrad with the GELU-backward epilogue
    if (BN == 256) return launch_gemm<256, EPI_DGELU_TANH, false, false, false, false, true>(a, b, p, st);
    if (BN == 128) return launch_gemm<128, EPI_DGELU_TANH, false, false, false, false, true>(a, b, p, st);
    return launch_gemm<64, EPI_DGELU_TANH, false, false, false, false, true>(a, b, p, st);
  }
  if (BN == 256) return launch_gemm<256, FVB_EPI_BIAS, false, false, false, TA, true>(a, b, p, st);
  if (BN == 128) return launch_gemm<128, FVB_EPI_BIAS, false, false, false, TA, true>(a, b, p, st);
  return launch_gemm<64, FVB_EPI_BIAS, false, false, false, TA, true>(a, b, p, st);
}

static int gemm_bwd_impl(bool a_mn_major, const void* a, int64_t lda, const void* b, int64_t ldb, void* out, int64_t ldo,
                         int Mo, int No, int R, bool weight_stripes, void* stream, const void* h = nullptr, int64_t ldh = 0) {
  FVB_CHECK_ARG(a && b && out, "null pointer");
  FVB_CHECK_ARG(Mo > 0 && No > 0 && R > 0, "empty problem");
  FVB_CHECK_ARG(No % 8 == 0, "output columns (K of the forward) must be a multiple of 8");
  FVB_CHECK_ARG(lda % 8 == 0 && ldb % 8 == 0 && ldo % 8 == 0, "row strides must be multiples of 8");
  FVB_CHECK_ARG(ldo >= No, "output row stride must cover the output columns");
  const int BN = (No >= 256 && No % 256 == 0) ? 256 : (No >= 128 && No % 128 == 0 ? 128 : (No >= 192 ? 256 : 64));
  // bind the device's primary context to this thread before the driver-API encode: autograd runs the backward on its own
  // worker thread, where no runtime call may have made it current yet (the encode then fails with CUDA_ERROR_INVALID_CONTEXT)
  FVB_CHECK_CUDA(cudaFree(nullptr));
  CUtensorMap tmA, tmB;
  if (a_mn_major) {
    uint64_t dims[2] = {(uint64_t)Mo, (uint64_t)R};
    uint64_t str[2] = {2, (uint64_t)lda * 2};
    uint32_t box[2] = {(uint32_t)GEMM_MN_CHUNK, (uint32_t)GEMM_BK};
    if (int r = make_tmap_bf16(&tmA, a, 2, dims, str, box)) return r;
  } else {  // the forward's A map: [batch 1][segment 1][Mo][R]
    uint64_t dims[4] = {(uint64_t)R, (uint64_t)Mo, 1, 1};
    uint64_t str[4] = {2, (uint64_t)lda * 2, 32, 16};  // unused dimensions (size 1): any 16-byte multiple
    uint32_t box[4] = {(uint32_t)GEMM_BK, GEMM_BM, 1, 1};
    if (int r = make_tmap_bf16(&tmA, a, 4, dims, str, box)) return r;
  }
  {
    uint64_t dims[2] = {(uint64_t)No, (uint64_t)R};
    uint64_t str[2] = {2, (uint64_t)ldb * 2};
    uint32_t box[2] = {(uint32_t)GEMM_MN_CHUNK, (uint32_t)GEMM_BK};
    if (int r = make_tmap_bf16(&tmB, b, 2, dims, str, box)) return r;
  }
  GemmParams p{};
  p.out = out;
  p.ldo = ldo;
  p.resid = reinterpret_cast<const __nv_bfloat16*>(h);
  p.ldr = ldh;
  p.a_seg_len = R;
  p.div = 1.f;
  p.M = Mo;
  p.N = No;
  p.K = R;
  p.batch = 1;
  p.num_m = (Mo + GEMM_BM - 1) / GEMM_BM;
  p.num_n = (No + BN - 1) / BN;
  p.num_k = (R + GEMM_BK - 1) / GEMM_BK;
  // dgrad: the forward's weight-stripe raster (a stripe of w's columns stays in L2 while dy streams past it). wgrad: the
  // row-group raster -- the ~132 resident tiles cover 8 row-blocks x ~16 column tiles and walk the token axis in step, so
  // each k-block of dy and x is read from HBM once per wave and shared through L2 by 16 resp. 8 CTAs.
  p.stripe_n = weight_stripes && p.num_m >= 16 && p.num_n > 8 ? 8 : 0;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (a_mn_major) return dispatch_bwd<true>(BN, tmA, tmB, p, st);
  return dispatch_bwd<false>(BN, tmA, tmB, p, st);
}

extern "C" int fvb_linear_dgrad_bf16(const void* dy, int64_t lddy, const void* w, int64_t ldw, void* dx, int64_t lddx, int M,
                                     int N, int K, void* stream) {
  // dx[M, K] = dy[M, N] . w[N, K]: A = dy (K-major over n), B = w (MN-major: row n holds the K output columns)
  return gemm_bwd_impl(false, dy, lddy, w, ldw, dx, lddx, M, K, N, true, stream);
}

extern "C" int fvb_linear_wgrad_bf16(const void* dy, int64_t lddy, const void* x, int64_t ldx, void* dw, int64_t lddw, int M,
                                     int N, int K, void* stream) {
  // dw[N, K] = dy^T . x over the M tokens: A = dy^T (MN-major: token row m holds the N output rows), B = x (MN-major)
  return gemm_bwd_impl(true, dy, lddy, x, ldx, dw, lddw, N, K, M, false, stream);
}

extern "C" int fvb_linear_dgrad_gelu_bf16(const void* dy, int64_t lddy, const void* w, int64_t ldw, const void* h, int64_t ldh,
                                          void* dh, int64_t lddh, int M, int N, int K, void* stream) {
  // fvb_linear_dgrad_bf16 with h[M, K] (the fc_in output before its GELU) read in the epilogue
  FVB_CHECK_ARG(h != nullptr && ldh % 8 == 0, "h required (ldh a multiple of 8)");
  return gemm_bwd_impl(false, dy, lddy, w, ldw, dh, lddh, M, K, N, true, stream, h, ldh);
}
