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

}  // namespace fvb

using namespace fvb;

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
