// gemm_sm90.cu -- persistent, warp-specialised bf16 GEMM for sm_90a:
//   out = epilogue(x[M,K] @ w[N,K]^T + bias)
// TMA (128B swizzle) -> shared-memory ring -> wgmma (two warpgroups, 64 rows x BN each, fp32 accumulators in registers)
// -> epilogue straight from the accumulator registers with fused bias / GELU(tanh) / gated residual.
//
// Stands behind fastvideo/layers/linear.py:146-156 (F.linear) and the elementwise op that follows
// each linear in fastvideo/models/dits/wanvideo.py:394-431; rounding points mirror the reference's
// eager bf16 path (see include/fvb200.h).
//
// Warp roles (384 threads): warpgroup 0 = TMA producer (one thread issues), warpgroups 1 and 2 = MMA + epilogue for rows
// [0, 64) and [64, 128) of the 128-row tile. The producer runs ahead into the next tile while the consumers finish the
// epilogue of the current one.
// Persistent CTAs walk the tiles in weight-stripe order (tile_coords): a stripe of 8 column tiles stays in L2 while
// the row-blocks stream past it. Output column blocks may be redirected by an offset table (out_col_offsets), which
// is how the sequence-parallel paths write heads straight into send / peer receive buffers.
#include <cstdlib>
#include "fvb_host.cuh"
#include "fvb_ptx.cuh"

namespace fvb {

constexpr int GEMM_BM = 128;
constexpr int GEMM_BK = 64;   // 64 bf16 = one 128B swizzle row
constexpr int GEMM_THREADS = 384;
constexpr int GEMM_GROUP_M = 8;

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

template <int BN, int EPI>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_bf16_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                 const GemmParams p) {
  using Cfg = GemmCfg<BN>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + Cfg::STAGES * Cfg::STAGE_BYTES);
  uint64_t* full = bars;
  uint64_t* empty = bars + Cfg::STAGES;

  const int wg = threadIdx.x >> 7;
  const int tiles_per_batch = p.num_m * p.num_n;
  const int num_tiles = tiles_per_batch * p.batch;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int i = 0; i < Cfg::STAGES; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], 8);  // lane 0 of each of the eight consumer warps
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (wg == 0) {
    // ------------------------------ TMA producer ------------------------------
    reg_dealloc<40>();
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        int m_blk, n_blk;
        const int bt = tile / tiles_per_batch;
        tile_coords(tile - bt * tiles_per_batch, p.num_m, p.num_n, p.stripe_n, m_blk, n_blk);
        for (int kb = 0; kb < p.num_k; ++kb) {
          mbar_wait(&empty[stage], phase ^ 1);
          uint8_t* sa = smem + stage * Cfg::STAGE_BYTES;
          uint8_t* sb = sa + Cfg::A_BYTES;
          mbar_expect_tx(&full[stage], Cfg::STAGE_BYTES);
          {
            const int k0 = kb * GEMM_BK;
            const int seg = k0 / p.a_seg_len;
            tma_load_4d(sa, &tmA, &full[stage], k0 - seg * p.a_seg_len, m_blk * GEMM_BM, seg, bt);
          }
          tma_load_3d(sb, &tmB, &full[stage], kb * GEMM_BK, n_blk * BN, bt);
          if (++stage == Cfg::STAGES) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    }
    return;
  }
  // ------------------------------ MMA + epilogue (rows [64 (wg - 1), 64 wg) of the tile) ------------------------------
  reg_alloc<232>();  // 128 x 40 + 256 x 232 = 64 512 of 65 536 registers
  const int half = wg - 1;
  const int warp = (threadIdx.x >> 5) & 3;
  const int lane = threadIdx.x & 31;
  int stage = 0;
  uint32_t phase = 0;
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    int m_blk, n_blk;
    const int bt = tile / tiles_per_batch;
    tile_coords(tile - bt * tiles_per_batch, p.num_m, p.num_n, p.stripe_n, m_blk, n_blk);
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    int prev = -1;
    for (int kb = 0; kb < p.num_k; ++kb) {
      mbar_wait(&full[stage], phase);
      const uint32_t sa = smem_u32(smem + stage * Cfg::STAGE_BYTES) + half * (64 * 128);
      const uint32_t sb = smem_u32(smem + stage * Cfg::STAGE_BYTES + Cfg::A_BYTES);
      const uint64_t da = make_desc_kmajor_sw128(sa);
      const uint64_t db = make_desc_kmajor_sw128(sb);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < GEMM_BK / 16; ++k) wgmma_ss<BN>(acc, da + uint64_t(2 * k), db + uint64_t(2 * k));
      wgmma_commit();
      // keep one k-block of MMAs in flight: the stage read by the previous group is free once it completes
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

    // ------------------------------ epilogue ------------------------------
    const int row0 = m_blk * GEMM_BM + half * 64 + warp * 16 + (lane >> 2);
    const float* gate_rows_p[2] = {p.gate, p.gate};
    if constexpr (EPI != FVB_EPI_RESID_BF16)
      if (p.gate_rows > 0)
        for (int i = 0; i < 2; ++i) gate_rows_p[i] += int64_t((row0 + 8 * i) / p.gate_rows) * p.gate_stride;
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      const int col = n_blk * BN + 8 * j + 2 * (lane & 3);
      if (col >= p.N) continue;  // N is a multiple of 8: the pair (col, col + 1) is inside or outside together
      const int64_t out_col = p.out_col_offsets ? __ldg(p.out_col_offsets + (col >> 7)) + (col & 127) : int64_t(col);
      float2 bf = make_float2(0.f, 0.f);
      if (p.bias != nullptr) bf = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(p.bias + col));
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int row = row0 + 8 * i;
        if (row >= p.M) continue;
        float f0 = acc[4 * j + 2 * i], f1 = acc[4 * j + 2 * i + 1];
        if (p.bias != nullptr) {
          f0 = __fadd_rn(f0, bf.x);
          f1 = __fadd_rn(f1, bf.y);
        }
        // y = bf16(acc + bias) in every mode (the reference's F.linear output dtype)
        if constexpr (EPI == FVB_EPI_BIAS_GELU_TANH) {
          f0 = gelu_tanh_f(bf16_round(f0));
          f1 = gelu_tanh_f(bf16_round(f1));
        } else if constexpr (EPI == FVB_EPI_DIV) {
          f0 = __fdiv_rn(bf16_round(f0), p.div);
          f1 = __fdiv_rn(bf16_round(f1), p.div);
        } else if constexpr (EPI == FVB_EPI_SCALE_F32) {
          f0 = __fmul_rn(f0, p.div);
          f1 = __fmul_rn(f1, p.div);
        } else if constexpr (EPI == FVB_EPI_RESID_GATE_F32 || EPI == FVB_EPI_RESID_GATE_BF16 ||
                             EPI == FVB_EPI_RESID_GATE_BF16R || EPI == FVB_EPI_RESID_BF16) {
          const float2 rf = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(p.resid + int64_t(row) * p.ldr + col));
          const float y0 = bf16_round(f0), y1 = bf16_round(f1);
          if constexpr (EPI == FVB_EPI_RESID_BF16) {
            f0 = __fadd_rn(rf.x, y0);
            f1 = __fadd_rn(rf.y, y1);
          } else {
            const float2 g = *reinterpret_cast<const float2*>(gate_rows_p[i] + col);
            if constexpr (EPI == FVB_EPI_RESID_GATE_BF16R) {
              f0 = __fadd_rn(rf.x, bf16_round(__fmul_rn(y0, g.x)));
              f1 = __fadd_rn(rf.y, bf16_round(__fmul_rn(y1, g.y)));
            } else {
              f0 = __fadd_rn(rf.x, __fmul_rn(y0, g.x));
              f1 = __fadd_rn(rf.y, __fmul_rn(y1, g.y));
            }
          }
        }
        if constexpr (EPI == FVB_EPI_RESID_GATE_F32 || EPI == FVB_EPI_SCALE_F32) {
          float* op = reinterpret_cast<float*>(p.out) + int64_t(bt) * p.out_batch_stride + int64_t(row) * p.ldo + out_col;
          *reinterpret_cast<float2*>(op) = make_float2(f0, f1);
        } else {
          __nv_bfloat16* op = reinterpret_cast<__nv_bfloat16*>(p.out) + int64_t(bt) * p.out_batch_stride + int64_t(row) * p.ldo + out_col;
          *reinterpret_cast<uint32_t*>(op) = pack_bf16x2(f0, f1);
        }
      }
    }
  }
}

template <int BN, int EPI>
static int launch_gemm(const CUtensorMap& tmA, const CUtensorMap& tmB, const GemmParams& p, cudaStream_t st) {
  using Cfg = GemmCfg<BN>;
  auto kern = gemm_bf16_kernel<BN, EPI>;
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
    case FVB_EPI_BIAS: return launch_gemm<BN, FVB_EPI_BIAS>(a, b, p, st);
    case FVB_EPI_BIAS_GELU_TANH: return launch_gemm<BN, FVB_EPI_BIAS_GELU_TANH>(a, b, p, st);
    case FVB_EPI_RESID_GATE_F32: return launch_gemm<BN, FVB_EPI_RESID_GATE_F32>(a, b, p, st);
    case FVB_EPI_RESID_GATE_BF16: return launch_gemm<BN, FVB_EPI_RESID_GATE_BF16>(a, b, p, st);
    case FVB_EPI_RESID_GATE_BF16R: return launch_gemm<BN, FVB_EPI_RESID_GATE_BF16R>(a, b, p, st);
    case FVB_EPI_RESID_BF16: return launch_gemm<BN, FVB_EPI_RESID_BF16>(a, b, p, st);
    case FVB_EPI_DIV: return launch_gemm<BN, FVB_EPI_DIV>(a, b, p, st);
    case FVB_EPI_SCALE_F32: return launch_gemm<BN, FVB_EPI_SCALE_F32>(a, b, p, st);
  }
  return set_error(FVB_ERR_INVALID_ARG, "unknown epilogue%s");
}

}  // namespace fvb

using namespace fvb;

static int gemm_impl(const void* x, int64_t ldx, int64_t x_batch, int a_seg_len, int64_t a_seg_stride, const void* w, int64_t ldw, int64_t w_batch,
                     const void* bias, void* out, int64_t ldo, int64_t o_batch, const int64_t* out_col_offsets,
                     const void* resid, int64_t ldr,
                     const float* gate, int gate_rows, int64_t gate_stride, float div, int M, int N, int K, int batch,
                     int epilogue, void* stream) {
  FVB_CHECK_ARG(x && w && out, "null pointer");
  FVB_CHECK_ARG(M > 0 && N > 0 && K > 0 && batch > 0, "empty problem");
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
  const int BN = (N >= 256 && N % 256 == 0) ? 256 : (N >= 128 && N % 128 == 0 ? 128 : (N >= 192 ? 256 : 64));

  CUtensorMap tmA, tmB;
  if (a_seg_len <= 0 || a_seg_len >= K) {
    a_seg_len = K;
    a_seg_stride = 16;  // unused (single segment); any 16B multiple
  }
  FVB_CHECK_ARG(a_seg_len % GEMM_BK == 0 || a_seg_len == K, "A segment length must be a multiple of 64");
  FVB_CHECK_ARG(K % a_seg_len == 0 && a_seg_stride % 8 == 0, "bad A segmentation");
  {
    uint64_t dims[4] = {(uint64_t)a_seg_len, (uint64_t)M, (uint64_t)(K / a_seg_len), (uint64_t)batch};
    uint64_t str[4] = {2, (uint64_t)ldx * 2, (uint64_t)a_seg_stride * 2,
                       (uint64_t)(batch > 1 ? x_batch : 8) * 2};
    uint32_t box[4] = {GEMM_BK, GEMM_BM, 1, 1};
    int r = make_tmap_bf16(&tmA, x, 4, dims, str, box);
    if (r) return r;
  }
  {
    uint64_t dims[3] = {(uint64_t)K, (uint64_t)N, (uint64_t)batch};
    uint64_t str[3] = {2, (uint64_t)ldw * 2, (uint64_t)(batch > 1 ? w_batch : ldw * (int64_t)N) * 2};
    uint32_t box[3] = {GEMM_BK, (uint32_t)BN, 1};
    int r = make_tmap_bf16(&tmB, w, 3, dims, str, box);
    if (r) return r;
  }
  GemmParams p;
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
  p.M = M;
  p.N = N_store;
  p.K = K;
  p.batch = batch;
  p.num_m = (M + GEMM_BM - 1) / GEMM_BM;
  p.num_n = (N + BN - 1) / BN;
  p.num_k = (K + GEMM_BK - 1) / GEMM_BK;
  static const int stripe_env = [] { const char* e = getenv("FVB_GEMM_STRIPE_N"); return e ? atoi(e) : -1; }();
  // default: stripes of 8 column tiles once the problem is tall enough for a stripe sweep to fill several waves
  p.stripe_n = stripe_env >= 0 ? stripe_env : 8;
  if (stripe_env > 0) {  // explicit setting (A/B runs): clamp to the column-tile count instead of falling back to the row-group raster
    p.stripe_n = p.num_m < 16 ? 0 : (stripe_env < p.num_n ? stripe_env : p.num_n);
  } else if (p.stripe_n > 0 && (p.num_m < 16 || p.num_n <= p.stripe_n)) {
    p.stripe_n = 0;
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
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
