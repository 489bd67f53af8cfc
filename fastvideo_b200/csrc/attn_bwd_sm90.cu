// attn_bwd_sm90.cu -- backward of block-sparse attention (64-token blocks, per-q-block key lists): dQ, dK, dV.
// Contract: fastvideo-kernel/python/fastvideo_kernel/block_sparse_attn.py:138-243 (block_sparse_attn_backward_triton and its
// autograd glue) over triton_kernels/block_sparse_attn_triton.py:165-694 (_attn_bwd_preprocess / _attn_bwd_dkdv / _attn_bwd_dq)
// and triton_kernels/index.py:147-250 (invert_indices). Same inputs as the reference: q, k, v, o, the forward's LSE
// M = max(qk * scale * log2 e) + log2(sum) (what fvb_attention_blocklist_fwd writes), dO, the q->kv lists and their inverse.
//
//   delta_i = rowsum(dO_i * O_i)                                   (preprocess, one row kernel)
//   P = exp2(Q_i K_j^T * scale * log2 e - M_i)   (keys >= variable_block_sizes[j] masked to 0)
//   dV_j += P^T dO_i       dP = dO_i V_j^T       dS = P * (dP - delta_i) * scale
//   dQ_i += dS K_j         dK_j += dS^T Q_i
//
// Correctness-first on warp-level mma.sync tiles (nvcuda::wmma, bf16 inputs, fp32 accumulation; P and dS rounded to bf16
// before their second GEMM exactly like the Triton kernels do), not the wgmma / TMA pipeline of the forward. One CTA per (q block, head) for dQ walking the q->kv list, one CTA per
// (kv block, head) for dK / dV walking the kv->q list; K/V (resp. Q/dO) tiles staged through shared memory.
#include <mma.h>

#include <type_traits>

#include "fvb_host.cuh"
#include "fvb_ptx.cuh"

namespace fvb {
using namespace nvcuda;

constexpr int BW_THREADS = 128;  // 4 warps, 16 rows each
constexpr int BW_LD = 136;       // bf16 row pitch of the 64 x 128 tiles (+8: bank spread)
constexpr int BW_LDS = 68;       // fp32 row pitch of the 64 x 64 score tiles
constexpr int BW_LDP = 72;       // bf16 row pitch of the 64 x 64 P / dS tiles
constexpr int BW_TILE = 64 * BW_LD;
constexpr int BW_SMEM = 4 * BW_TILE * 2 + 2 * 64 * BW_LDS * 4 + 2 * 64 * BW_LDP * 2 + 4 * 64 * 4;

struct BwdStr {
  int64_t b, s, h;
};

struct BwdParams {
  const __nv_bfloat16 *q, *k, *v, *o, *dO;
  __nv_bfloat16 *dq, *dk, *dv;
  BwdStr sq, sk, sv, so, sdo, sdq, sdk, sdv;
  const float* lse;   // [B, H, Sq] log2 domain
  float* delta;       // [B, H, Sq]
  int Sq, Skv, H;
  float scale, scale_log2;
  const int32_t *q2k_idx, *q2k_num, *k2q_idx, *k2q_num;  // [B?, H?, nqb, capq] / [.., nqb] ; [B?, H?, nkb, capk] / [.., nkb]
  int64_t idx_stride_b, idx_stride_h;                      // in rows of the respective index tensors (0 = broadcast)
  int capq, capk, nqb, nkb;
  const int32_t* kv_len;  // variable_block_sizes [nkb]
};

// 64 x 128 bf16 tile global -> shared (rows past `rows_valid` are zero filled)
FVB_DEVICE void bw_load_tile(__nv_bfloat16* dst, const __nv_bfloat16* base, int64_t row_stride, int row0, int rows_valid) {
  for (int i = threadIdx.x; i < 64 * 16; i += BW_THREADS) {
    const int r = i >> 4, c = i & 15;
    uint4 val = make_uint4(0, 0, 0, 0);
    if (r < rows_valid) val = *reinterpret_cast<const uint4*>(base + int64_t(row0 + r) * row_stride + c * 8);
    *reinterpret_cast<uint4*>(dst + r * BW_LD + c * 8) = val;
  }
}

// S[64 x 64] (fp32, shared) = A[64 x 128] B[64 x 128]^T ; warp w computes rows 16w .. 16w+15
FVB_DEVICE void bw_abt(float* S, const __nv_bfloat16* A, const __nv_bfloat16* Bm, int warp) {
  wmma::fragment<wmma::accumulator, 16, 16, 16, float> acc[4];
#pragma unroll
  for (int n = 0; n < 4; ++n) wmma::fill_fragment(acc[n], 0.f);
#pragma unroll
  for (int kk = 0; kk < 8; ++kk) {
    wmma::fragment<wmma::matrix_a, 16, 16, 16, __nv_bfloat16, wmma::row_major> a;
    wmma::load_matrix_sync(a, A + warp * 16 * BW_LD + kk * 16, BW_LD);
#pragma unroll
    for (int n = 0; n < 4; ++n) {
      wmma::fragment<wmma::matrix_b, 16, 16, 16, __nv_bfloat16, wmma::col_major> bf;
      wmma::load_matrix_sync(bf, Bm + n * 16 * BW_LD + kk * 16, BW_LD);  // B^T: element (k, n) = Bm[n][k]
      wmma::mma_sync(acc[n], a, bf, acc[n]);
    }
  }
#pragma unroll
  for (int n = 0; n < 4; ++n) wmma::store_matrix_sync(S + warp * 16 * BW_LDS + n * 16, acc[n], BW_LDS, wmma::mem_row_major);
}

// per-warp elementwise stage on its 16 rows: P = exp2(S * scale_log2 - M) (masked), dS = P * (dP - delta) * scale
FVB_DEVICE void bw_p_ds(const float* S, const float* dP, __nv_bfloat16* P, __nv_bfloat16* dS, const float* rowM, const float* rowD,
                        int vlen, float scale, float scale_log2, int warp, int lane) {
  for (int e = lane; e < 16 * 64; e += 32) {
    const int r = warp * 16 + (e >> 6), c = e & 63;
    const float m = rowM[r];
    float pv = 0.f;
    if (c < vlen && m != -INFINITY) pv = exp2f(fmaf(S[r * BW_LDS + c], scale_log2, -m));
    P[r * BW_LDP + c] = __float2bfloat16_rn(pv);
    dS[r * BW_LDP + c] = __float2bfloat16_rn(pv * (dP[r * BW_LDS + c] - rowD[r]) * scale);
  }
}

__global__ void bwd_delta_kernel(BwdParams p, int B) {
  // one warp per row: delta = sum_d dO * O
  const int64_t row = int64_t(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  const int64_t total = int64_t(B) * p.H * p.Sq;
  if (row >= total) return;
  const int s = int(row % p.Sq), h = int((row / p.Sq) % p.H), b = int(row / (int64_t(p.Sq) * p.H));
  const __nv_bfloat16* o = p.o + b * p.so.b + int64_t(s) * p.so.s + h * p.so.h;
  const __nv_bfloat16* d = p.dO + b * p.sdo.b + int64_t(s) * p.sdo.s + h * p.sdo.h;
  float acc = 0.f;
  for (int c = lane * 4; c < 128; c += 128) {
#pragma unroll
    for (int j = 0; j < 4; ++j) acc += __bfloat162float(o[c + j]) * __bfloat162float(d[c + j]);
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
  if (lane == 0) p.delta[row] = acc;
}

// ---------------------------------------------------------------- dQ: CTA = (q block, head, batch)
__global__ void __launch_bounds__(BW_THREADS) bwd_dq_kernel(BwdParams p) {
  extern __shared__ __align__(128) uint8_t smem[];
  __nv_bfloat16* sQ = reinterpret_cast<__nv_bfloat16*>(smem);
  __nv_bfloat16* sdO = sQ + BW_TILE;
  __nv_bfloat16* sK = sdO + BW_TILE;
  __nv_bfloat16* sV = sK + BW_TILE;
  float* sS = reinterpret_cast<float*>(sV + BW_TILE);
  float* sdP = sS + 64 * BW_LDS;
  __nv_bfloat16* sP = reinterpret_cast<__nv_bfloat16*>(sdP + 64 * BW_LDS);
  __nv_bfloat16* sdS = sP + 64 * BW_LDP;
  float* rowM = reinterpret_cast<float*>(sdS + 64 * BW_LDP);
  float* rowD = rowM + 64;
  const int qb = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q0 = qb * 64;
  const int q_valid = max(0, min(64, p.Sq - q0));
  bw_load_tile(sQ, p.q + b * p.sq.b + h * p.sq.h, p.sq.s, q0, q_valid);
  bw_load_tile(sdO, p.dO + b * p.sdo.b + h * p.sdo.h, p.sdo.s, q0, q_valid);
  if (threadIdx.x < 64) {
    const int64_t r = (int64_t(b) * p.H + h) * p.Sq + q0 + threadIdx.x;
    rowM[threadIdx.x] = threadIdx.x < q_valid ? p.lse[r] : -INFINITY;
    rowD[threadIdx.x] = threadIdx.x < q_valid ? p.delta[r] : 0.f;
  }
  const int64_t ir = int64_t(b) * p.idx_stride_b + int64_t(h) * p.idx_stride_h + qb;
  const int32_t* list = p.q2k_idx + ir * p.capq;
  const int n = min(p.q2k_num[ir], p.capq);
  wmma::fragment<wmma::accumulator, 16, 16, 16, float> dq[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) wmma::fill_fragment(dq[i], 0.f);
  for (int e = 0; e < n; ++e) {
    const int kb = list[e];
    const int k0 = kb * 64;
    const int vlen = min(p.kv_len ? p.kv_len[kb] : 64, max(0, p.Skv - k0));
    __syncthreads();  // previous iteration's readers of sK / sV / sdS are done
    bw_load_tile(sK, p.k + b * p.sk.b + h * p.sk.h, p.sk.s, k0, min(64, max(0, p.Skv - k0)));
    bw_load_tile(sV, p.v + b * p.sv.b + h * p.sv.h, p.sv.s, k0, min(64, max(0, p.Skv - k0)));
    __syncthreads();
    bw_abt(sS, sQ, sK, warp);    // S  = Q K^T
    bw_abt(sdP, sdO, sV, warp);  // dP = dO V^T
    __syncwarp();
    bw_p_ds(sS, sdP, sP, sdS, rowM, rowD, vlen, p.scale, p.scale_log2, warp, lane);
    __syncwarp();
    // dQ[16 rows of this warp] += dS[16 x 64] K[64 x 128]
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      wmma::fragment<wmma::matrix_a, 16, 16, 16, __nv_bfloat16, wmma::row_major> a;
      wmma::load_matrix_sync(a, sdS + warp * 16 * BW_LDP + kk * 16, BW_LDP);
#pragma unroll
      for (int nn = 0; nn < 8; ++nn) {
        wmma::fragment<wmma::matrix_b, 16, 16, 16, __nv_bfloat16, wmma::row_major> bf;
        wmma::load_matrix_sync(bf, sK + kk * 16 * BW_LD + nn * 16, BW_LD);
        wmma::mma_sync(dq[nn], a, bf, dq[nn]);
      }
    }
  }
  __syncthreads();
  // stage fp32 dQ through shared memory (reuse the K / V tiles: 64 x 128 fp32 = 32 KB) and write bf16 rows
  float* stage = reinterpret_cast<float*>(sK);
#pragma unroll
  for (int nn = 0; nn < 8; ++nn) wmma::store_matrix_sync(stage + warp * 16 * 128 + nn * 16, dq[nn], 128, wmma::mem_row_major);
  __syncthreads();
  __nv_bfloat16* dst = p.dq + b * p.sdq.b + h * p.sdq.h;
  for (int i = threadIdx.x; i < 64 * 16; i += BW_THREADS) {
    const int r = i >> 4, c = i & 15;
    if (r >= q_valid) continue;
    const float* s = stage + r * 128 + c * 8;
    uint4 o;
    o.x = pack_bf16x2(s[0], s[1]);
    o.y = pack_bf16x2(s[2], s[3]);
    o.z = pack_bf16x2(s[4], s[5]);
    o.w = pack_bf16x2(s[6], s[7]);
    *reinterpret_cast<uint4*>(dst + int64_t(q0 + r) * p.sdq.s + c * 8) = o;
  }
}

// ---------------------------------------------------------------- dK, dV: CTA = (kv block, head, batch)
__global__ void __launch_bounds__(BW_THREADS) bwd_dkdv_kernel(BwdParams p) {
  extern __shared__ __align__(128) uint8_t smem[];
  __nv_bfloat16* sQ = reinterpret_cast<__nv_bfloat16*>(smem);
  __nv_bfloat16* sdO = sQ + BW_TILE;
  __nv_bfloat16* sK = sdO + BW_TILE;
  __nv_bfloat16* sV = sK + BW_TILE;
  float* sS = reinterpret_cast<float*>(sV + BW_TILE);
  float* sdP = sS + 64 * BW_LDS;
  __nv_bfloat16* sP = reinterpret_cast<__nv_bfloat16*>(sdP + 64 * BW_LDS);
  __nv_bfloat16* sdS = sP + 64 * BW_LDP;
  float* rowM = reinterpret_cast<float*>(sdS + 64 * BW_LDP);
  float* rowD = rowM + 64;
  const int kb = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int k0 = kb * 64;
  const int k_rows = min(64, max(0, p.Skv - k0));
  const int vlen = min(p.kv_len ? p.kv_len[kb] : 64, k_rows);
  bw_load_tile(sK, p.k + b * p.sk.b + h * p.sk.h, p.sk.s, k0, k_rows);
  bw_load_tile(sV, p.v + b * p.sv.b + h * p.sv.h, p.sv.s, k0, k_rows);
  const int64_t ir = int64_t(b) * p.idx_stride_b + int64_t(h) * p.idx_stride_h + kb;
  const int32_t* list = p.k2q_idx + ir * p.capk;
  const int n = min(p.k2q_num[ir], p.capk);
  wmma::fragment<wmma::accumulator, 16, 16, 16, float> dk[8], dv[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    wmma::fill_fragment(dk[i], 0.f);
    wmma::fill_fragment(dv[i], 0.f);
  }
  for (int e = 0; e < n; ++e) {
    const int qb = list[e];
    const int q0 = qb * 64;
    const int q_valid = max(0, min(64, p.Sq - q0));
    __syncthreads();
    bw_load_tile(sQ, p.q + b * p.sq.b + h * p.sq.h, p.sq.s, q0, q_valid);
    bw_load_tile(sdO, p.dO + b * p.sdo.b + h * p.sdo.h, p.sdo.s, q0, q_valid);
    if (threadIdx.x < 64) {
      const int64_t r = (int64_t(b) * p.H + h) * p.Sq + q0 + threadIdx.x;
      rowM[threadIdx.x] = threadIdx.x < q_valid ? p.lse[r] : -INFINITY;
      rowD[threadIdx.x] = threadIdx.x < q_valid ? p.delta[r] : 0.f;
    }
    __syncthreads();
    bw_abt(sS, sQ, sK, warp);
    bw_abt(sdP, sdO, sV, warp);
    __syncwarp();
    bw_p_ds(sS, sdP, sP, sdS, rowM, rowD, vlen, p.scale, p.scale_log2, warp, lane);
    __syncthreads();  // every warp reads all 64 q rows of P / dS below
    // dV[16 keys of this warp] += P^T[16 x 64 q] dO[64 q x 128] ; dK likewise with dS and Q
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      wmma::fragment<wmma::matrix_a, 16, 16, 16, __nv_bfloat16, wmma::col_major> ap, as;
      wmma::load_matrix_sync(ap, sP + kk * 16 * BW_LDP + warp * 16, BW_LDP);   // A(m = key, k = q) = P[q][key]
      wmma::load_matrix_sync(as, sdS + kk * 16 * BW_LDP + warp * 16, BW_LDP);
#pragma unroll
      for (int nn = 0; nn < 8; ++nn) {
        wmma::fragment<wmma::matrix_b, 16, 16, 16, __nv_bfloat16, wmma::row_major> bo, bq;
        wmma::load_matrix_sync(bo, sdO + kk * 16 * BW_LD + nn * 16, BW_LD);
        wmma::load_matrix_sync(bq, sQ + kk * 16 * BW_LD + nn * 16, BW_LD);
        wmma::mma_sync(dv[nn], ap, bo, dv[nn]);
        wmma::mma_sync(dk[nn], as, bq, dk[nn]);
      }
    }
  }
  __syncthreads();
  float* stage = reinterpret_cast<float*>(sQ);  // 64 x 128 fp32 = Q + dO tiles' space (2 x 17 KB >= 32 KB)
  for (int pass = 0; pass < 2; ++pass) {
#pragma unroll
    for (int nn = 0; nn < 8; ++nn)
      wmma::store_matrix_sync(stage + warp * 16 * 128 + nn * 16, pass ? dv[nn] : dk[nn], 128, wmma::mem_row_major);
    __syncthreads();
    __nv_bfloat16* dst = pass ? p.dv + b * p.sdv.b + h * p.sdv.h : p.dk + b * p.sdk.b + h * p.sdk.h;
    const int64_t rs = pass ? p.sdv.s : p.sdk.s;
    for (int i = threadIdx.x; i < 64 * 16; i += BW_THREADS) {
      const int r = i >> 4, c = i & 15;
      if (r >= k_rows) continue;
      const float* s = stage + r * 128 + c * 8;
      uint4 o;
      o.x = pack_bf16x2(s[0], s[1]);
      o.y = pack_bf16x2(s[2], s[3]);
      o.z = pack_bf16x2(s[4], s[5]);
      o.w = pack_bf16x2(s[6], s[7]);
      *reinterpret_cast<uint4*>(dst + int64_t(k0 + r) * rs + c * 8) = o;
    }
    __syncthreads();
  }
}

// ---------------------------------------------------------------- dense backward (fvb_attention_bwd): wgmma + TMA
// Two kernels, no float atomics:
//   KV = true : a CTA owns two 64-key tiles (one per consumer warpgroup) and walks every 64-row q tile:
//               S^T = K Q^T, dP^T = V dO^T (SS, m64n64k16), dV += P^T dO, dK += dS^T Q (RS, m64n128k16, dO / Q as the
//               transposed B operand, as the forward reads V). lse and delta are per column here: the producer warp stages
//               them in shared memory with each q tile (+inf / 0 for rows >= Sq, so those columns give P = dS = 0).
//   KV = false: a CTA owns two 64-row q tiles and walks every 64-key tile: S = Q K^T, dP = dO V^T (SS), dQ += dS K (RS).
// Warp roles as in the forward: warpgroup 0 is the producer (one TMA warp; setmaxnreg 24), warpgroups 1 and 2 consume
// (setmaxnreg 240: the KV kernel holds two 64 x 128 fp32 accumulators next to the 64 x 64 S^T and dP^T).
// Keys >= Skv get P = 0 explicitly (TMA zero fill gives S = 0 there, and exp2(0 - lse) is not 0).
//
// Block-list mode (LIST = true, fvb_attention_sparse_bwd), same arithmetic: the two owned 64-row boxes are tiles 2 x and
// 2 x + 1 of their layout, and the CTA walks the ascending union of those tiles' two lists (KV: kv -> q lists, else q -> kv),
// merged on the fly as the forward merges its q-block lists (KeyWalk mode 2). Only the producer walks: with each stage it
// publishes the item (2-bit "which warpgroup takes part" flags, the walked tile's valid rows) in shared memory, and after the
// last one an end marker. A warpgroup whose flag bit is clear does no MMA for the item and only releases the stage. Tile i starts at row off[i] (64 i without off) and has len[i] valid rows
// (the forward's rule, tile_rows); a box starting there also reads the next tile's first rows, so keys past the walked kv
// tile's length get P = 0, q rows past the walked q tile's length get lse = +inf / delta = 0 (KV) or are not loaded (dQ), and
// the epilogue stores only the owned tile's valid rows.
constexpr int DB_THREADS = 384;
constexpr int DB_STAGES = 3;
constexpr int DB_TILE = 64 * 128 * 2;  // 16 KB: [d half (2)][64 rows][128 B], the forward's tile
constexpr int DB_HALF = 64 * 128;
constexpr int DB_SMEM = 1024 + 4 * DB_TILE + DB_STAGES * 2 * DB_TILE + DB_STAGES * 2 * 64 * 4 + 256;

struct DenseBwdParams {
  __nv_bfloat16 *out0, *out1;  // KV: dk, dv; else dq
  BwdStr so0, so1;
  const float* lse;
  int64_t lse_stride_b, lse_stride_h;
  const float* delta;  // [B, H, Sq]
  int Sq, Skv, H;
  float scale, scale_log2;
};

struct SparseBwdParams : DenseBwdParams {
  const int32_t *list_idx, *list_num;     // KV: k2q lists, else q2k: [B?, H?, n_own, cap] ascending / [.., n_own]
  int64_t list_stride_b, list_stride_h;   // in list rows (0 = broadcast)
  int cap, n_own;
  const int32_t *own_off, *own_len;       // tiles a CTA owns (KV: kv tiles, else q tiles); NULL = the padded rule
  const int32_t *walk_off, *walk_len;     // tiles it walks (KV: q tiles, else kv tiles)
};

// first row and valid rows of tile i, the forward's rule: row0 = off[i] (64 i without off), rows = len[i] (without len:
// off[i + 1] - off[i], else 64), at most 64 and never past S
FVB_DEVICE void tile_rows(const int32_t* off, const int32_t* len, int i, int S, int& row0, int& rows) {
  row0 = off ? __ldg(off + i) : 64 * i;
  const int l = len ? __ldg(len + i) : (off ? __ldg(off + i + 1) - row0 : 64);
  rows = min(min(l, 64), max(0, S - row0));
}

// owned tile s of the CTA (block-list mode): its first row and valid rows; a missing second tile has none
template <bool KV>
FVB_DEVICE void own_tile(const SparseBwdParams& p, int s, int& row0, int& rows) {
  const int t = 2 * blockIdx.x + s, S = KV ? p.Skv : p.Sq;
  if (t < p.n_own) {
    tile_rows(p.own_off, p.own_len, t, S, row0, rows);
  } else {
    row0 = S;
    rows = 0;
  }
}

template <bool KV, bool LIST>
__global__ void __launch_bounds__(DB_THREADS, 1)
attn_bwd_dense_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                      const __grid_constant__ CUtensorMap tmV, const __grid_constant__ CUtensorMap tmdO,
                      const std::conditional_t<LIST, SparseBwdParams, DenseBwdParams> p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  // resident: [warpgroup (2)][operand (2)][tile] -- KV: (K, V), else (Q, dO); ring: [stage][operand (2)][tile] -- KV:
  // (Q, dO), else (K, V)
  uint8_t* sRes = smem;
  uint8_t* sRing = smem + 4 * DB_TILE;
  float* sLse = reinterpret_cast<float*>(sRing + DB_STAGES * 2 * DB_TILE);  // [stage][64] (KV only)
  float* sDelta = sLse + DB_STAGES * 64;
  uint64_t* res_full = reinterpret_cast<uint64_t*>(sDelta + DB_STAGES * 64);
  uint64_t* full = res_full + 1;
  uint64_t* empty = full + DB_STAGES;
  // LIST: int [stage] after the barriers, the walk item of each stage: flags | walked rows << 2, or -1 = end of walk

  const int h = blockIdx.y, b = blockIdx.z;
  const int n_walk = KV ? (p.Sq + 63) / 64 : (p.Skv + 63) / 64;
  const int64_t bh = int64_t(b) * p.H + h;
  if (threadIdx.x == 0) {
    mbar_init(res_full, 1);
    for (int i = 0; i < DB_STAGES; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], 8);  // lane 0 of each consumer warp
    }
    fence_mbar_init();
  }
  __syncthreads();

  const int wg = threadIdx.x >> 7, warp = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  if (wg == 0) {
    // ------------------------------ producer: warp 0 (all lanes wait; lane 0 issues TMA) ------------------------------
    reg_dealloc<24>();
    if (warp != 0) return;
    const CUtensorMap* res0 = KV ? &tmK : &tmQ;
    const CUtensorMap* res1 = KV ? &tmV : &tmdO;
    const CUtensorMap* ring0 = KV ? &tmQ : &tmK;
    const CUtensorMap* ring1 = KV ? &tmdO : &tmV;
    if (lane == 0) {
      tma_prefetch_desc(ring0);
      tma_prefetch_desc(ring1);
      mbar_expect_tx(res_full, 4 * DB_TILE);
      for (int s = 0; s < 2; ++s)
        for (int hf = 0; hf < 2; ++hf) {
          int row0 = (2 * blockIdx.x + s) * 64, rows;
          if constexpr (LIST) own_tile<KV>(p, s, row0, rows);
          tma_load_4d(sRes + (2 * s) * DB_TILE + hf * DB_HALF, res0, res_full, hf * 64, row0, h, b);
          tma_load_4d(sRes + (2 * s + 1) * DB_TILE + hf * DB_HALF, res1, res_full, hf * 64, row0, h, b);
        }
    }
    KeyWalk walk;  // LIST: the union of the two owned tiles' lists
    if constexpr (LIST) {
      const int64_t r0 = int64_t(b) * p.list_stride_b + int64_t(h) * p.list_stride_h + 2 * blockIdx.x;
      walk.mode = 2;
      walk.i0 = walk.i1 = 0;
      walk.l0 = p.list_idx + r0 * p.cap;
      walk.l1 = walk.l0 + p.cap;
      walk.n0 = min(__ldg(p.list_num + r0), p.cap);
      walk.n1 = 2 * int(blockIdx.x) + 1 < p.n_own ? min(__ldg(p.list_num + r0 + 1), p.cap) : 0;
    }
    int stage = 0;
    uint32_t phase = 0;
    int flags;
    for (int t = 0; LIST ? walk.next(t, flags) : t < n_walk; ++t) {  // LIST: next() sets t
      mbar_wait(&empty[stage], phase ^ 1);
      int row0 = t * 64, rows = 64;
      if constexpr (LIST) {
        tile_rows(p.walk_off, p.walk_len, t, KV ? p.Sq : p.Skv, row0, rows);
        if (lane == 0) reinterpret_cast<int*>(empty + DB_STAGES)[stage] = flags | rows << 2;
      }
      if constexpr (KV) {
        for (int r = lane; r < 64; r += 32) {
          const int q = row0 + r;
          const bool valid = LIST ? r < rows : q < p.Sq;
          sLse[stage * 64 + r] = valid ? __ldg(p.lse + int64_t(b) * p.lse_stride_b + int64_t(h) * p.lse_stride_h + q) : INFINITY;
          sDelta[stage * 64 + r] = valid ? __ldg(p.delta + bh * p.Sq + q) : 0.f;
        }
        __syncwarp();
      }
      if (lane == 0) {
        uint8_t* dst = sRing + stage * 2 * DB_TILE;
        mbar_expect_tx(&full[stage], 2 * DB_TILE);  // also the arrive that publishes the staged lse / delta
        for (int hf = 0; hf < 2; ++hf) {
          tma_load_4d(dst + hf * DB_HALF, ring0, &full[stage], hf * 64, row0, h, b);
          tma_load_4d(dst + DB_TILE + hf * DB_HALF, ring1, &full[stage], hf * 64, row0, h, b);
        }
      }
      if (++stage == DB_STAGES) {
        stage = 0;
        phase ^= 1;
      }
    }
    if constexpr (LIST) {
      mbar_wait(&empty[stage], phase ^ 1);
      if (lane == 0) {
        reinterpret_cast<int*>(empty + DB_STAGES)[stage] = -1;
        mbar_arrive(&full[stage]);
      }
    }
    return;
  }

  // ------------------------------ consumers: warpgroup s owns 64 rows (KV: keys, else q rows) ------------------------------
  reg_alloc<240>();  // 128 x 24 + 256 x 240 = 64 512 of 65 536 registers
  const int s = wg - 1;
  const int tq = lane & 3;
  int own0 = (2 * blockIdx.x + s) * 64;
  int own_rows = max(0, min(64, (KV ? p.Skv : p.Sq) - own0));
  if constexpr (LIST) own_tile<KV>(p, s, own0, own_rows);
  const uint32_t ra0 = smem_u32(sRes + (2 * s) * DB_TILE), ra1 = smem_u32(sRes + (2 * s + 1) * DB_TILE);
  // KV: lse / delta come per column from shared memory; else per row, from global once
  float row_lse[2] = {INFINITY, INFINITY}, row_delta[2] = {0.f, 0.f};
  if constexpr (!KV) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int r = 16 * warp + (lane >> 2) + 8 * i;
      if (r < own_rows) {
        row_lse[i] = __ldg(p.lse + int64_t(b) * p.lse_stride_b + int64_t(h) * p.lse_stride_h + own0 + r);
        row_delta[i] = __ldg(p.delta + bh * p.Sq + own0 + r);
      }
    }
  }
  float acc0[64], acc1[64];  // KV: dV, dK; else dQ (acc1 unused)
#pragma unroll
  for (int i = 0; i < 64; ++i) acc0[i] = acc1[i] = 0.f;
  mbar_wait(res_full, 0);
  int stage = 0;
  uint32_t phase = 0;
  for (int t = 0; LIST || t < n_walk; ++t) {  // LIST: until the end marker
    mbar_wait(&full[stage], phase);
    int item = 3;
    if constexpr (LIST) {
      item = reinterpret_cast<const int*>(empty + DB_STAGES)[stage];
      if (item < 0) break;
    }
    if (own_rows > 0 && (!LIST || ((item >> s) & 1))) {
      const uint32_t ga0 = smem_u32(sRing + stage * 2 * DB_TILE), ga1 = ga0 + DB_TILE;
      float sc[32], dp[32];  // KV: S^T, dP^T (rows = keys, columns = q rows); else S, dP
#pragma unroll
      for (int i = 0; i < 32; ++i) sc[i] = dp[i] = 0.f;
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const uint32_t off = (k >> 2) * DB_HALF;
        wgmma_ss<64>(sc, make_desc_kmajor_sw128(ra0 + off) + uint64_t(2 * (k & 3)), make_desc_kmajor_sw128(ga0 + off) + uint64_t(2 * (k & 3)));
      }
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const uint32_t off = (k >> 2) * DB_HALF;
        wgmma_ss<64>(dp, make_desc_kmajor_sw128(ra1 + off) + uint64_t(2 * (k & 3)), make_desc_kmajor_sw128(ga1 + off) + uint64_t(2 * (k & 3)));
      }
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(sc);
      wgmma_fence_regs(dp);
      // P = exp2(S scale log2e - lse), dS = P (dP - delta) scale on rows (16 warp + lane / 4 + 8 i), columns (8 j + 2 tq + c)
      const int col_valid = KV ? 64 : LIST ? item >> 2 : min(64, p.Skv - t * 64);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        float2 cl = make_float2(0.f, 0.f), cd = make_float2(0.f, 0.f);
        if constexpr (KV) {
          cl = *reinterpret_cast<const float2*>(sLse + stage * 64 + 8 * j + 2 * tq);
          cd = *reinterpret_cast<const float2*>(sDelta + stage * 64 + 8 * j + 2 * tq);
        }
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const int row = 16 * warp + (lane >> 2) + 8 * i;
#pragma unroll
          for (int c = 0; c < 2; ++c) {
            const int col = 8 * j + 2 * tq + c;
            const float l = KV ? (c ? cl.y : cl.x) : row_lse[i];
            const float dl = KV ? (c ? cd.y : cd.x) : row_delta[i];
            const bool valid = KV ? row < own_rows : col < col_valid;
            const int e = 4 * j + 2 * i + c;
            const float pv = valid ? ex2(fmaf(sc[e], p.scale_log2, -l)) : 0.f;
            sc[e] = pv;
            dp[e] = pv * (dp[e] - dl) * p.scale;
          }
        }
      }
      // P / dS (bf16) as the register A operand, 16 columns per MMA
      uint32_t pa[4][4], da[4][4];
#pragma unroll
      for (int kk = 0; kk < 4; ++kk)
#pragma unroll
        for (int r = 0; r < 4; ++r) {
          pa[kk][r] = pack_bf16x2(sc[8 * kk + 2 * r], sc[8 * kk + 2 * r + 1]);
          da[kk][r] = pack_bf16x2(dp[8 * kk + 2 * r], dp[8 * kk + 2 * r + 1]);
        }
      wgmma_fence();
      if constexpr (KV) {
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) wgmma_rs_n128_tb(acc0, pa[kk], make_desc_mnmajor_sw128(ga1 + kk * 16 * 128, DB_HALF));
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) wgmma_rs_n128_tb(acc1, da[kk], make_desc_mnmajor_sw128(ga0 + kk * 16 * 128, DB_HALF));
      } else {
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) wgmma_rs_n128_tb(acc0, da[kk], make_desc_mnmajor_sw128(ga0 + kk * 16 * 128, DB_HALF));
      }
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(acc0);
      if constexpr (KV) wgmma_fence_regs(acc1);
    }
    if (lane == 0) mbar_arrive(&empty[stage]);
    if (++stage == DB_STAGES) {
      stage = 0;
      phase ^= 1;
    }
  }

  // ------------------------------ epilogue: bf16 rows < own_rows ------------------------------
  auto store = [&](const float(&acc)[64], __nv_bfloat16* base, const BwdStr& st) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int r = 16 * warp + (lane >> 2) + 8 * i;
      if (r >= own_rows) continue;
      __nv_bfloat16* op = base + int64_t(b) * st.b + int64_t(own0 + r) * st.s + int64_t(h) * st.h;
#pragma unroll
      for (int j = 0; j < 16; ++j)
        *reinterpret_cast<uint32_t*>(op + 8 * j + 2 * tq) = pack_bf16x2(acc[4 * j + 2 * i], acc[4 * j + 2 * i + 1]);
    }
  };
  if constexpr (KV) {
    store(acc1, p.out0, p.so0);  // dK
    store(acc0, p.out1, p.so1);  // dV
  } else {
    store(acc0, p.out0, p.so0);  // dQ
  }
}

}  // namespace fvb

using namespace fvb;

// delta = rowsum(dO * O) (the block-list backward's row kernel), the four TMA maps and the parameters both wgmma backward
// kernels share
static int wgmma_bwd_setup(const void* q, const void* k, const void* v, const void* o, const void* dO, const float* lse,
                           int64_t lse_stride_b, int64_t lse_stride_h, float* delta_ws, const int64_t* const (&st8)[8], int B,
                           int H, int Sq, int Skv, float softmax_scale, cudaStream_t st, CUtensorMap (&tm)[4],
                           DenseBwdParams& p) {
  for (auto s : st8)
    for (int i = 0; i < 3; ++i) FVB_CHECK_ARG(s[i] % 8 == 0, "strides must be multiples of 8 elements");
  auto S3 = [](const int64_t* s) { return BwdStr{s[0], s[1], s[2]}; };
  BwdParams dp = {};
  dp.o = reinterpret_cast<const __nv_bfloat16*>(o);
  dp.dO = reinterpret_cast<const __nv_bfloat16*>(dO);
  dp.so = S3(st8[3]);
  dp.sdo = S3(st8[4]);
  dp.delta = delta_ws;
  dp.Sq = Sq;
  dp.H = H;
  const int64_t rows = int64_t(B) * H * Sq;
  bwd_delta_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, st>>>(dp, B);
  FVB_CHECK_CUDA(cudaGetLastError());

  int r;
  if ((r = make_qkv_tmap(&tm[0], q, Sq, H, B, st8[0][1], st8[0][2], st8[0][0]))) return r;
  if ((r = make_qkv_tmap(&tm[1], k, Skv, H, B, st8[1][1], st8[1][2], st8[1][0]))) return r;
  if ((r = make_qkv_tmap(&tm[2], v, Skv, H, B, st8[2][1], st8[2][2], st8[2][0]))) return r;
  if ((r = make_qkv_tmap(&tm[3], dO, Sq, H, B, st8[4][1], st8[4][2], st8[4][0]))) return r;
  p = {};
  p.lse = lse;
  p.lse_stride_b = lse_stride_b;
  p.lse_stride_h = lse_stride_h;
  p.delta = delta_ws;
  p.Sq = Sq;
  p.Skv = Skv;
  p.H = H;
  p.scale = softmax_scale;
  p.scale_log2 = softmax_scale * 1.4426950408889634f;
  return FVB_OK;
}

template <bool KV, bool LIST, typename P>
static int launch_wgmma_bwd(const CUtensorMap (&tm)[4], const P& p, int n_own, int H, int B, cudaStream_t st) {
  static bool configured = false;
  if (!configured) {
    FVB_CHECK_CUDA(cudaFuncSetAttribute(attn_bwd_dense_kernel<KV, LIST>, cudaFuncAttributeMaxDynamicSharedMemorySize, DB_SMEM));
    configured = true;
  }
  attn_bwd_dense_kernel<KV, LIST><<<dim3((n_own + 1) / 2, H, B), DB_THREADS, DB_SMEM, st>>>(tm[0], tm[1], tm[2], tm[3], p);
  FVB_CHECK_CUDA(cudaGetLastError());
  return FVB_OK;
}

extern "C" int fvb_attention_bwd(const void* q, const void* k, const void* v, const void* o, const void* dO, const float* lse,
                                 int64_t lse_stride_b, int64_t lse_stride_h, void* dq, void* dk, void* dv, float* delta_ws,
                                 const int64_t* q_strides, const int64_t* k_strides, const int64_t* v_strides,
                                 const int64_t* o_strides, const int64_t* do_strides, const int64_t* dq_strides,
                                 const int64_t* dk_strides, const int64_t* dv_strides, int B, int H, int Sq, int Skv,
                                 int head_dim, float softmax_scale, void* stream) {
  FVB_CHECK_ARG(q && k && v && o && dO && lse && dq && dk && dv && delta_ws, "null pointer");
  FVB_CHECK_ARG(head_dim == 128, "head_dim must be 128");
  FVB_CHECK_ARG(B > 0 && H > 0 && Sq > 0 && Skv > 0, "empty problem");
  FVB_CHECK_ARG(H <= 65535 && B <= 65535, "too many heads / batches");
  const int64_t* const all[8] = {q_strides, k_strides, v_strides, o_strides, do_strides, dq_strides, dk_strides, dv_strides};
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  CUtensorMap tm[4];
  DenseBwdParams p;
  int r;
  if ((r = wgmma_bwd_setup(q, k, v, o, dO, lse, lse_stride_b, lse_stride_h, delta_ws, all, B, H, Sq, Skv, softmax_scale, st, tm, p)))
    return r;
  auto S3 = [](const int64_t* s) { return BwdStr{s[0], s[1], s[2]}; };
  p.out0 = reinterpret_cast<__nv_bfloat16*>(dk);
  p.out1 = reinterpret_cast<__nv_bfloat16*>(dv);
  p.so0 = S3(dk_strides);
  p.so1 = S3(dv_strides);
  if ((r = launch_wgmma_bwd<true, false>(tm, p, (Skv + 63) / 64, H, B, st))) return r;
  p.out0 = reinterpret_cast<__nv_bfloat16*>(dq);
  p.out1 = nullptr;
  p.so0 = S3(dq_strides);
  return launch_wgmma_bwd<false, false>(tm, p, (Sq + 63) / 64, H, B, st);
}

extern "C" int fvb_attention_sparse_bwd(const void* q, const void* k, const void* v, const void* o, const void* dO,
                                        const float* lse, int64_t lse_stride_b, int64_t lse_stride_h, void* dq, void* dk,
                                        void* dv, float* delta_ws, const int64_t* q_strides, const int64_t* k_strides,
                                        const int64_t* v_strides, const int64_t* o_strides, const int64_t* do_strides,
                                        const int64_t* dq_strides, const int64_t* dk_strides, const int64_t* dv_strides, int B,
                                        int H, int Sq, int Skv, int head_dim, float softmax_scale, const int32_t* q2k_idx,
                                        const int32_t* q2k_num, int capq, const int32_t* k2q_idx, const int32_t* k2q_num,
                                        int capk, int64_t idx_stride_b, int64_t idx_stride_h, int64_t kidx_stride_b,
                                        int64_t kidx_stride_h, const int32_t* q_off, const int32_t* q_len, int nqb,
                                        const int32_t* kv_off, const int32_t* kv_len, int nkb, void* stream) {
  FVB_CHECK_ARG(q && k && v && o && dO && lse && dq && dk && dv && delta_ws && q2k_idx && q2k_num && k2q_idx && k2q_num,
                "null pointer");
  FVB_CHECK_ARG(head_dim == 128, "head_dim must be 128");
  FVB_CHECK_ARG(B > 0 && H > 0 && Sq > 0 && Skv > 0 && nqb > 0 && nkb > 0 && capq > 0 && capk > 0, "empty problem");
  FVB_CHECK_ARG(H <= 65535 && B <= 65535, "too many heads / batches");
  FVB_CHECK_ARG((idx_stride_h == 0 || idx_stride_h == nqb) &&
                    (idx_stride_b == 0 || idx_stride_b == (idx_stride_h ? int64_t(H) * nqb : int64_t(nqb))),
                "q2k index tensors must be contiguous [B or 1, H or 1, nqb, capq]");
  FVB_CHECK_ARG((kidx_stride_h == 0 || kidx_stride_h == nkb) &&
                    (kidx_stride_b == 0 || kidx_stride_b == (kidx_stride_h ? int64_t(H) * nkb : int64_t(nkb))),
                "k2q index tensors must be contiguous [B or 1, H or 1, nkb, capk]");
  const int64_t* const all[8] = {q_strides, k_strides, v_strides, o_strides, do_strides, dq_strides, dk_strides, dv_strides};
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  CUtensorMap tm[4];
  SparseBwdParams p;
  int r;
  if ((r = wgmma_bwd_setup(q, k, v, o, dO, lse, lse_stride_b, lse_stride_h, delta_ws, all, B, H, Sq, Skv, softmax_scale, st, tm, p)))
    return r;
  auto S3 = [](const int64_t* s) { return BwdStr{s[0], s[1], s[2]}; };
  // dK, dV: kv tiles owned, q tiles walked (the k2q lists)
  p.out0 = reinterpret_cast<__nv_bfloat16*>(dk);
  p.out1 = reinterpret_cast<__nv_bfloat16*>(dv);
  p.so0 = S3(dk_strides);
  p.so1 = S3(dv_strides);
  p.list_idx = k2q_idx;
  p.list_num = k2q_num;
  p.list_stride_b = kidx_stride_b;
  p.list_stride_h = kidx_stride_h;
  p.cap = capk;
  p.n_own = nkb;
  p.own_off = kv_off;
  p.own_len = kv_len;
  p.walk_off = q_off;
  p.walk_len = q_len;
  if ((r = launch_wgmma_bwd<true, true>(tm, p, nkb, H, B, st))) return r;
  // dQ: q tiles owned, kv tiles walked (the q2k lists)
  p.out0 = reinterpret_cast<__nv_bfloat16*>(dq);
  p.out1 = nullptr;
  p.so0 = S3(dq_strides);
  p.list_idx = q2k_idx;
  p.list_num = q2k_num;
  p.list_stride_b = idx_stride_b;
  p.list_stride_h = idx_stride_h;
  p.cap = capq;
  p.n_own = nqb;
  p.own_off = q_off;
  p.own_len = q_len;
  p.walk_off = kv_off;
  p.walk_len = kv_len;
  return launch_wgmma_bwd<false, true>(tm, p, nqb, H, B, st);
}

extern "C" int fvb_attention_blocklist_bwd(const void* q, const void* k, const void* v, const void* o, const void* dO,
                                           const float* lse, void* dq, void* dk, void* dv, float* delta_ws,
                                           const int64_t* q_strides, const int64_t* k_strides, const int64_t* v_strides,
                                           const int64_t* o_strides, const int64_t* do_strides, const int64_t* dq_strides,
                                           const int64_t* dk_strides, const int64_t* dv_strides, int B, int H, int Sq, int Skv,
                                           int head_dim, float softmax_scale, const int32_t* q2k_idx, const int32_t* q2k_num,
                                           int capq, const int32_t* k2q_idx, const int32_t* k2q_num, int capk,
                                           int64_t idx_stride_b, int64_t idx_stride_h, int64_t kidx_stride_b,
                                           int64_t kidx_stride_h, const int32_t* kv_len, void* stream) {
  FVB_CHECK_ARG(q && k && v && o && dO && lse && dq && dk && dv && delta_ws && q2k_idx && q2k_num && k2q_idx && k2q_num,
                "null pointer");
  FVB_CHECK_ARG(head_dim == 128, "head_dim must be 128");
  FVB_CHECK_ARG(B > 0 && H > 0 && Sq > 0 && Skv > 0 && Sq % 64 == 0 && Skv % 64 == 0, "sequence lengths must be multiples of 64");
  const int64_t* all[8] = {q_strides, k_strides, v_strides, o_strides, do_strides, dq_strides, dk_strides, dv_strides};
  for (auto st : all)
    for (int i = 0; i < 3; ++i) FVB_CHECK_ARG(st[i] % 8 == 0, "strides must be multiples of 8 elements");
  BwdParams p;
  auto S3 = [](const int64_t* s) { return BwdStr{s[0], s[1], s[2]}; };
  p.q = reinterpret_cast<const __nv_bfloat16*>(q);
  p.k = reinterpret_cast<const __nv_bfloat16*>(k);
  p.v = reinterpret_cast<const __nv_bfloat16*>(v);
  p.o = reinterpret_cast<const __nv_bfloat16*>(o);
  p.dO = reinterpret_cast<const __nv_bfloat16*>(dO);
  p.dq = reinterpret_cast<__nv_bfloat16*>(dq);
  p.dk = reinterpret_cast<__nv_bfloat16*>(dk);
  p.dv = reinterpret_cast<__nv_bfloat16*>(dv);
  p.sq = S3(q_strides); p.sk = S3(k_strides); p.sv = S3(v_strides); p.so = S3(o_strides); p.sdo = S3(do_strides);
  p.sdq = S3(dq_strides); p.sdk = S3(dk_strides); p.sdv = S3(dv_strides);
  p.lse = lse;
  p.delta = delta_ws;
  p.Sq = Sq; p.Skv = Skv; p.H = H;
  p.scale = softmax_scale;
  p.scale_log2 = softmax_scale * 1.4426950408889634f;
  p.q2k_idx = q2k_idx; p.q2k_num = q2k_num; p.k2q_idx = k2q_idx; p.k2q_num = k2q_num;
  p.capq = capq; p.capk = capk; p.nqb = Sq / 64; p.nkb = Skv / 64;
  p.kv_len = kv_len;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  static bool configured = false;
  if (!configured) {
    FVB_CHECK_CUDA(cudaFuncSetAttribute(bwd_dq_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, BW_SMEM));
    FVB_CHECK_CUDA(cudaFuncSetAttribute(bwd_dkdv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, BW_SMEM));
    configured = true;
  }
  const int64_t rows = int64_t(B) * H * Sq;
  bwd_delta_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, st>>>(p, B);
  FVB_CHECK_CUDA(cudaGetLastError());
  p.idx_stride_b = idx_stride_b; p.idx_stride_h = idx_stride_h;
  bwd_dq_kernel<<<dim3(p.nqb, H, B), BW_THREADS, BW_SMEM, st>>>(p);
  FVB_CHECK_CUDA(cudaGetLastError());
  p.idx_stride_b = kidx_stride_b; p.idx_stride_h = kidx_stride_h;
  bwd_dkdv_kernel<<<dim3(p.nkb, H, B), BW_THREADS, BW_SMEM, st>>>(p);
  FVB_CHECK_CUDA(cudaGetLastError());
  return FVB_OK;
}
