// attn_sm90.cu -- fused multi-head attention forward for sm_90a (head_dim 128, bf16), one kernel, three key sources:
//   dense        : every key tile                      (SDPAImpl.forward, fastvideo/attention/backends/sdpa.py:122-147;
//                                                       cross-attention, fastvideo/models/dits/wanvideo.py:188-222)
//   pair lists   : the ascending union of two q blocks' 64-key block lists with a 2-bit "who attends" flag per entry
//                  (fvb_attention_fwd with a schedule from fvb_pair_schedule; STA tile windows,
//                  fastvideo-kernel/tests/support_flex_sta.py:11-58)
//   q-block lists: each q block's own ascending list (fvb_attention_blocklist_fwd; VSA,
//                  fastvideo-kernel/python/fastvideo_kernel/block_sparse_attn.py:347-393); the CTA merges the lists of its
//                  two q blocks on the fly, so a key block both select is loaded once.
// Keys past a block's valid length are masked (variable_block_sizes); rows whose list is empty produce exact zeros and
// LSE = -inf, as the reference kernels do. LSE is in the log2 domain: max(qk*scale*log2e) + log2(sum), the format of
// block_sparse_attn_triton.py:160-163.
//
// Design (one CTA = two 64-row q blocks, 288 threads):
//   warpgroups 0, 1  one q block each: S = Q K^T (wgmma m64n64k16, both operands in shared memory), online softmax in
//                    registers, O += P V (wgmma m64n128k16, P from registers, V in shared memory as the transposed operand)
//   warp 8           TMA producer: Q once, then a ring of 64-key K and V tiles (each an arbitrary 64-row window)
// A warpgroup whose q block does not attend a tile of the shared walk skips its MMAs and only releases the stage.
//
// The kernel is a template over its operands. attn_fwd_kernel<false> is the bf16 kernel above; attn_fwd_kernel<true> is
// the 8-bit one of fvb_attention_8bit_fwd (arithmetic in include/fvb200.h), with the same CTA shape, key walk and
// schedule: S = Q8 K8^T by wgmma m64n64k32 s32.s8.s8 (both from 128B-swizzled shared memory, rows of exactly 128 B), the
// logits scaled by the per-row q / k scales, P quantised to e4m3 straight from the S accumulator registers into the
// A-operand registers of wgmma m64n128k32 f32.e4m3.e4m3 (the vt8 key-slot permutation makes the two layouts agree), B =
// the vt8 tile (128 channel rows of 64 key slots, 64B swizzle). Each tile's P V goes into its own register set, which is
// added into the running O in fp32 after O is rescaled.
#include <cuda_fp8.h>

#include "fvb_host.cuh"
#include "fvb_ptx.cuh"

namespace fvb {

constexpr int ATT_D = 128;
constexpr int ATT_THREADS = 288;
constexpr int ATT_STAGES = 4;
constexpr int ATT_TILE_BYTES = 64 * ATT_D * 2;  // 16 KB: [d half (2)][64 rows][128 B]
constexpr int ATT_HALF_BYTES = 64 * 128;        // 8 KB

struct AttnParams {
  __nv_bfloat16* o;
  float* lse;  // [B, H, lse_stride_h rows] or NULL
  int64_t o_stride_b, o_stride_s, o_stride_h;
  int64_t lse_stride_b, lse_stride_h;
  int Sq, Skv, H, B;
  float scale_log2;
  // pair lists (fvb_attention_fwd with a schedule)
  const int32_t* sched;      // [B?, H?, npairs, sched_cap] entries kv_block | flags << 24, ascending
  const int32_t* sched_cnt;  // [B?, H?, npairs]
  int64_t sched_stride_b, sched_stride_h;  // in pairs (0 = broadcast)
  int sched_cap;
  // q-block lists (fvb_attention_blocklist_fwd)
  const int32_t* q2k_idx;  // [B?, H?, nqb, cap] ascending kv block ids
  const int32_t* q2k_num;  // [B?, H?, nqb]
  int64_t idx_stride_b, idx_stride_h;  // in q blocks (0 = broadcast)
  int cap;
  const int32_t* q_off;   // [nqb+1] first row of each q block, or NULL (64*b)
  const int32_t* kv_off;  // [nkb+1] first row of each kv block, or NULL (64*b)
  const int32_t* kv_len;  // [nkb] valid keys per kv block, or NULL (from kv_off, else 64)
  const int32_t* q_len;   // [nqb] rows to write per q block, or NULL (from q_off, else 64)
  int nqb, nkb;
  // 8-bit operands only (fvb_attention_8bit_fwd)
  const float* q_scale;  // [B, H, Sq]
  const float* k_scale;  // [B, H, Skv]
  const float* v_scale;  // [B, H, 128]
};

// byte sizes of one 64-row operand tile and of the kernel's shared memory
template <bool Q8>
struct AttnSmem {
  static constexpr int TILE = Q8 ? 64 * ATT_D : ATT_TILE_BYTES;  // Q / K: 64 rows of 128 B (8-bit) or 2 x [64][128 B]
  static constexpr int BYTES = TILE * (2 + 2 * ATT_STAGES) + 1024 + 256;
};

// The CTA's walk over key blocks (KeyWalk, fvb_ptx.cuh): flags bit s = q block s attends.
FVB_DEVICE void kv_rows(const AttnParams& p, bool dense, int kb, int& row0, int& vlen) {
  if (dense) {
    row0 = kb * 64;
    vlen = min(64, p.Skv - row0);
    return;
  }
  row0 = p.kv_off ? __ldg(p.kv_off + kb) : kb * 64;
  if (p.kv_len) vlen = __ldg(p.kv_len + kb);
  else if (p.kv_off) vlen = min(64, __ldg(p.kv_off + kb + 1) - row0);
  else vlen = 64;
  vlen = min(vlen, max(0, p.Skv - row0));
}

template <bool Q8>
__global__ void __launch_bounds__(ATT_THREADS, 1)
attn_fwd_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                const __grid_constant__ CUtensorMap tmV, const AttnParams p) {
  constexpr int TILE = AttnSmem<Q8>::TILE;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;  // [q block (2)][tile]
  uint8_t* sK = smem + 2 * TILE;
  uint8_t* sV = sK + ATT_STAGES * TILE;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sV + ATT_STAGES * TILE);
  uint64_t* q_full = bars;                    // 1
  uint64_t* k_full = bars + 1;                // STAGES
  uint64_t* v_full = k_full + ATT_STAGES;     // STAGES
  uint64_t* kv_empty = v_full + ATT_STAGES;   // STAGES

  const int pair = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const bool dense = p.sched == nullptr && p.q2k_idx == nullptr;
  // the 8-bit kernel's key blocks are always the quantiser's (kv_off / kv_len, else 64-key blocks): vt8 is laid out by them
  const bool dense_kv = dense && !Q8;

  // this CTA's key walk
  KeyWalk walk;
  walk.i0 = walk.i1 = 0;
  walk.l0 = walk.l1 = nullptr;
  walk.n1 = 0;
  if (dense) {
    walk.mode = 0;
    walk.n0 = Q8 ? p.nkb : (p.Skv + 63) / 64;
  } else if (p.sched != nullptr) {
    walk.mode = 1;
    const int64_t pi = int64_t(b) * p.sched_stride_b + int64_t(h) * p.sched_stride_h + pair;
    walk.l0 = p.sched + pi * p.sched_cap;
    walk.n0 = __ldg(p.sched_cnt + pi);
  } else {
    walk.mode = 2;
    const int64_t r0 = int64_t(b) * p.idx_stride_b + int64_t(h) * p.idx_stride_h + 2 * pair;
    walk.l0 = p.q2k_idx + r0 * p.cap;
    walk.n0 = __ldg(p.q2k_num + r0);
    if (2 * pair + 1 < p.nqb) {
      walk.l1 = walk.l0 + p.cap;
      walk.n1 = __ldg(p.q2k_num + r0 + 1);
    }
  }
  // q rows of the two q blocks
  int q_row0[2], q_rows[2];
#pragma unroll
  for (int s = 0; s < 2; ++s) {
    const int qb = 2 * pair + s;
    if (dense) {
      q_row0[s] = qb * 64;
      q_rows[s] = min(64, max(0, p.Sq - q_row0[s]));
    } else if (qb < p.nqb) {
      q_row0[s] = p.q_off ? __ldg(p.q_off + qb) : qb * 64;
      const int len = p.q_len ? __ldg(p.q_len + qb) : (p.q_off ? __ldg(p.q_off + qb + 1) - q_row0[s] : 64);
      q_rows[s] = min(min(len, 64), max(0, p.Sq - q_row0[s]));
    } else {
      q_row0[s] = p.Sq;
      q_rows[s] = 0;
    }
  }

  if (threadIdx.x == 0) {
    mbar_init(q_full, 1);
    for (int i = 0; i < ATT_STAGES; ++i) {
      mbar_init(&k_full[i], 1);
      mbar_init(&v_full[i], 1);
      mbar_init(&kv_empty[i], 8);  // lane 0 of each consumer warp
    }
    fence_mbar_init();
  }
  __syncthreads();

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp == 8) {
    // ------------------------------ TMA producer ------------------------------
    if (lane == 0) {
      tma_prefetch_desc(&tmK);
      tma_prefetch_desc(&tmV);
      mbar_expect_tx(q_full, 2 * TILE);
#pragma unroll
      for (int s = 0; s < 2; ++s) {
        if constexpr (Q8) {
          tma_load_4d(sQ + s * TILE, &tmQ, q_full, 0, q_row0[s], h, b);
        } else {
#pragma unroll
          for (int hf = 0; hf < 2; ++hf)
            tma_load_4d(sQ + s * TILE + hf * ATT_HALF_BYTES, &tmQ, q_full, hf * 64, q_row0[s], h, b);
        }
      }
      int stage = 0;
      uint32_t phase = 0;
      int kb, flags;
      while (walk.next(kb, flags)) {
        int row0, vlen;
        kv_rows(p, dense_kv, kb, row0, vlen);
        mbar_wait(&kv_empty[stage], phase ^ 1);
        mbar_expect_tx(&k_full[stage], TILE);
        if constexpr (Q8) {
          tma_load_4d(sK + stage * TILE, &tmK, &k_full[stage], 0, row0, h, b);
          mbar_expect_tx(&v_full[stage], TILE);
          tma_load_2d(sV + stage * TILE, &tmV, &v_full[stage], 0, ((b * p.H + h) * p.nkb + kb) * ATT_D);
        } else {
          for (int hf = 0; hf < 2; ++hf)
            tma_load_4d(sK + stage * TILE + hf * ATT_HALF_BYTES, &tmK, &k_full[stage], hf * 64, row0, h, b);
          mbar_expect_tx(&v_full[stage], TILE);
          for (int hf = 0; hf < 2; ++hf)
            tma_load_4d(sV + stage * TILE + hf * ATT_HALF_BYTES, &tmV, &v_full[stage], hf * 64, row0, h, b);
        }
        if (++stage == ATT_STAGES) {
          stage = 0;
          phase ^= 1;
        }
      }
    }
    return;
  }

  // ------------------------------ consumers: warpgroup s = q block 2 pair + s ------------------------------
  const int s = warp >> 2;
  const int wq = warp & 3;
  const int tq = lane & 3;
  const uint32_t qa = smem_u32(sQ + s * TILE);
  const int64_t bh = int64_t(b) * p.H + h;
  float o[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) o[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  float sq[2] = {0.f, 0.f};  // 8-bit: scales of this thread's two q rows
  if constexpr (Q8) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int r = 16 * wq + (lane >> 2) + 8 * i;
      if (r < q_rows[s]) sq[i] = __ldg(p.q_scale + bh * p.Sq + q_row0[s] + r);
    }
  }
  mbar_wait(q_full, 0);
  int stage = 0;
  uint32_t phase = 0;
  int kb, flags;
  while (walk.next(kb, flags)) {
    if (!((flags >> s) & 1)) {  // the other q block's tile: release it without touching it
      mbar_wait(&k_full[stage], phase);
      mbar_wait(&v_full[stage], phase);
      if (lane == 0) mbar_arrive(&kv_empty[stage]);
      if (++stage == ATT_STAGES) {
        stage = 0;
        phase ^= 1;
      }
      continue;
    }
    int row0, vlen;
    kv_rows(p, dense_kv, kb, row0, vlen);
    const uint32_t ka = smem_u32(sK + stage * TILE);
    const uint32_t va = smem_u32(sV + stage * TILE);
    float sc[32];
    int32_t si[32];  // 8-bit: exact integer Q8 K8^T
    float sk[16];    // 8-bit: scales of this thread's keys 8 j + 2 tq + c
    if constexpr (Q8) {
#pragma unroll
      for (int j = 0; j < 8; ++j)
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          const int key = 8 * j + 2 * tq + c;
          sk[2 * j + c] = key < vlen ? __ldg(p.k_scale + bh * p.Skv + row0 + key) : 0.f;
        }
      mbar_wait(&k_full[stage], phase);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < ATT_D / 32; ++k)
        wgmma_ss_s8_n64(si, make_desc_kmajor_sw128(qa) + uint64_t(2 * k), make_desc_kmajor_sw128(ka) + uint64_t(2 * k), k);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(si);
    } else {
#pragma unroll
      for (int i = 0; i < 32; ++i) sc[i] = 0.f;
      mbar_wait(&k_full[stage], phase);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < ATT_D / 16; ++k) {
        const uint32_t off = (k >> 2) * ATT_HALF_BYTES;
        wgmma_ss<64>(sc, make_desc_kmajor_sw128(qa + off) + uint64_t(2 * (k & 3)), make_desc_kmajor_sw128(ka + off) + uint64_t(2 * (k & 3)));
      }
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(sc);
    }

    // online softmax on rows (16 wq + lane / 4 + 8 i), columns 8 j + 2 tq + c
    float alpha[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      float mx = -INFINITY;
#pragma unroll
      for (int j = 0; j < 8; ++j)
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          const int key = 8 * j + 2 * tq + c;
          float x;
          if constexpr (Q8)
            x = key < vlen ? __fmul_rn(__fmul_rn(__fmul_rn(float(si[4 * j + 2 * i + c]), sq[i]), sk[2 * j + c]), p.scale_log2)
                           : -INFINITY;
          else
            x = key < vlen ? sc[4 * j + 2 * i + c] * p.scale_log2 : -INFINITY;
          sc[4 * j + 2 * i + c] = x;
          mx = fmaxf(mx, x);
        }
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float m_new = fmaxf(m_run[i], mx);
      const float m_use = m_new == -INFINITY ? 0.f : m_new;
      alpha[i] = ex2(m_run[i] - m_use);
      m_run[i] = m_new;
      float sum = 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j)
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          const float e = ex2(sc[4 * j + 2 * i + c] - m_use);
          sc[4 * j + 2 * i + c] = e;
          sum += e;
        }
      l_run[i] = l_run[i] * alpha[i] + sum;
    }
    if constexpr (Q8) {
      // P (e4m3 of p * 448) as the register A operand, 32 keys per MMA. Register 2 hf + i of MMA kk holds row i's key slots
      // 16 hf + 4 tq .. +3 of keys 32 kk .. 32 kk + 31, i.e. keys 32 kk + 16 hf + {2 tq, 2 tq + 1, 8 + 2 tq, 9 + 2 tq}: the
      // accumulator columns of j = 4 kk + 2 hf and j + 1. vt8 stores the key of each slot in that order.
      uint32_t pa[2][4];
#pragma unroll
      for (int kk = 0; kk < 2; ++kk)
#pragma unroll
        for (int hf = 0; hf < 2; ++hf)
#pragma unroll
          for (int i = 0; i < 2; ++i) {
            const int j = 4 * kk + 2 * hf;
            const uint32_t lo = __nv_cvt_float2_to_fp8x2(
                make_float2(__fmul_rn(sc[4 * j + 2 * i], 448.f), __fmul_rn(sc[4 * j + 2 * i + 1], 448.f)), __NV_SATFINITE, __NV_E4M3);
            const uint32_t hi = __nv_cvt_float2_to_fp8x2(
                make_float2(__fmul_rn(sc[4 * j + 4 + 2 * i], 448.f), __fmul_rn(sc[4 * j + 4 + 2 * i + 1], 448.f)), __NV_SATFINITE,
                __NV_E4M3);
            pa[kk][2 * hf + i] = lo | (hi << 16);
          }
#pragma unroll
      for (int j = 0; j < 16; ++j)
#pragma unroll
        for (int i = 0; i < 2; ++i)
#pragma unroll
          for (int c = 0; c < 2; ++c) o[4 * j + 2 * i + c] = __fmul_rn(o[4 * j + 2 * i + c], alpha[i]);
      float t[64];  // this tile's P V, overwritten by the first MMA
      mbar_wait(&v_full[stage], phase);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 2; ++kk) wgmma_rs_e4m3_n128(t, pa[kk], make_desc_kmajor_sw64(va) + uint64_t(2 * kk), kk);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(t);
      if (lane == 0) mbar_arrive(&kv_empty[stage]);
#pragma unroll
      for (int i = 0; i < 64; ++i) o[i] = __fadd_rn(o[i], t[i]);
    } else {
#pragma unroll
      for (int j = 0; j < 16; ++j)
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          o[4 * j + 2 * i] *= alpha[i];
          o[4 * j + 2 * i + 1] *= alpha[i];
        }
      // P (bf16) as the register A operand, 16 keys per MMA
      uint32_t pa[4][4];
#pragma unroll
      for (int kk = 0; kk < 4; ++kk)
#pragma unroll
        for (int r = 0; r < 4; ++r) pa[kk][r] = pack_bf16x2(sc[8 * kk + 2 * r], sc[8 * kk + 2 * r + 1]);
      mbar_wait(&v_full[stage], phase);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) wgmma_rs_n128_tb(o, pa[kk], make_desc_mnmajor_sw128(va + kk * 16 * 128, ATT_HALF_BYTES));
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(o);
      if (lane == 0) mbar_arrive(&kv_empty[stage]);
    }
    if (++stage == ATT_STAGES) {
      stage = 0;
      phase ^= 1;
    }
  }

  // ------------------------------ epilogue ------------------------------
  float sv[32];  // 8-bit: v scales of this thread's channels 8 j + 2 tq + c
  if constexpr (Q8) {
#pragma unroll
    for (int j = 0; j < 16; ++j)
#pragma unroll
      for (int c = 0; c < 2; ++c) sv[2 * j + c] = __ldg(p.v_scale + bh * ATT_D + 8 * j + 2 * tq + c);
  }
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    float l = l_run[i];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const int r = 16 * wq + (lane >> 2) + 8 * i;
    if (r >= q_rows[s]) continue;
    const int tok = q_row0[s] + r;
    if constexpr (Q8) {
      const float inv = l > 0.f ? __fdiv_rn(1.f, __fmul_rn(448.f, l)) : 0.f;
      __nv_bfloat16* op = p.o + int64_t(b) * p.o_stride_b + int64_t(tok) * p.o_stride_s + int64_t(h) * p.o_stride_h;
#pragma unroll
      for (int j = 0; j < 16; ++j)
        *reinterpret_cast<uint32_t*>(op + 8 * j + 2 * tq) =
            pack_bf16x2(__fmul_rn(__fmul_rn(o[4 * j + 2 * i], sv[2 * j]), inv), __fmul_rn(__fmul_rn(o[4 * j + 2 * i + 1], sv[2 * j + 1]), inv));
    } else {
      const float inv = l > 0.f ? 1.f / l : 0.f;
      __nv_bfloat16* op = p.o + int64_t(b) * p.o_stride_b + int64_t(tok) * p.o_stride_s + int64_t(h) * p.o_stride_h;
#pragma unroll
      for (int j = 0; j < 16; ++j)
        *reinterpret_cast<uint32_t*>(op + 8 * j + 2 * tq) = pack_bf16x2(o[4 * j + 2 * i] * inv, o[4 * j + 2 * i + 1] * inv);
      if (tq == 0 && p.lse != nullptr)
        p.lse[int64_t(b) * p.lse_stride_b + int64_t(h) * p.lse_stride_h + tok] = l > 0.f ? m_run[i] + log2f(l) : -INFINITY;
    }
  }
}

template <bool Q8>
static int launch_kernel(const CUtensorMap& tmQ, const CUtensorMap& tmK, const CUtensorMap& tmV, const AttnParams& p,
                         int n_pairs, void* stream) {
  constexpr int smem = AttnSmem<Q8>::BYTES;
  static bool configured = false;
  if (!configured) {
    FVB_CHECK_CUDA(cudaFuncSetAttribute(attn_fwd_kernel<Q8>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    configured = true;
  }
  dim3 grid(unsigned(n_pairs), unsigned(p.H), unsigned(p.B));
  attn_fwd_kernel<Q8><<<grid, ATT_THREADS, smem, reinterpret_cast<cudaStream_t>(stream)>>>(tmQ, tmK, tmV, p);
  FVB_CHECK_CUDA(cudaGetLastError());
  return FVB_OK;
}

static int launch_attention(const void* q, const void* k, const void* v, const int64_t* q_strides, const int64_t* k_strides,
                            const int64_t* v_strides, const int64_t* o_strides, AttnParams& p, int n_pairs, void* stream) {
  for (int i = 0; i < 3; ++i)
    FVB_CHECK_ARG(q_strides[i] % 8 == 0 && k_strides[i] % 8 == 0 && v_strides[i] % 8 == 0 && o_strides[i] % 8 == 0,
                  "strides must be multiples of 8 elements");
  FVB_CHECK_ARG(p.H <= 65535 && p.B <= 65535, "too many heads / batches");
  CUtensorMap tmQ, tmK, tmV;
  int r;
  if ((r = make_qkv_tmap(&tmQ, q, p.Sq, p.H, p.B, q_strides[1], q_strides[2], q_strides[0]))) return r;
  if ((r = make_qkv_tmap(&tmK, k, p.Skv, p.H, p.B, k_strides[1], k_strides[2], k_strides[0]))) return r;
  if ((r = make_qkv_tmap(&tmV, v, p.Skv, p.H, p.B, v_strides[1], v_strides[2], v_strides[0]))) return r;
  p.o_stride_b = o_strides[0];
  p.o_stride_s = o_strides[1];
  p.o_stride_h = o_strides[2];
  return launch_kernel<false>(tmQ, tmK, tmV, p, n_pairs, stream);
}

static AttnParams base_params(void* o, float* lse, int64_t lse_stride_b, int64_t lse_stride_h, int B, int H, int Sq, int Skv,
                              float softmax_scale, const int32_t* q_off, const int32_t* q_len, int nqb, const int32_t* kv_off,
                              const int32_t* kv_len, int nkb) {
  AttnParams p = {};
  p.o = reinterpret_cast<__nv_bfloat16*>(o);
  p.lse = lse;
  p.lse_stride_b = lse_stride_b;
  p.lse_stride_h = lse_stride_h;
  p.Sq = Sq;
  p.Skv = Skv;
  p.H = H;
  p.B = B;
  p.scale_log2 = softmax_scale * 1.4426950408889634f;
  p.q_off = q_off;
  p.kv_off = kv_off;
  p.kv_len = kv_len;
  p.q_len = q_len;
  p.nqb = nqb;
  p.nkb = nkb;
  return p;
}

}  // namespace fvb

using namespace fvb;

extern "C" int fvb_attention_fwd(const void* q, const void* k, const void* v, void* o, float* lse,
                                 const int64_t* q_strides /*b,s,h*/, const int64_t* k_strides, const int64_t* v_strides,
                                 const int64_t* o_strides, int64_t lse_stride_b, int64_t lse_stride_h, int B, int H,
                                 int Sq, int Skv, int head_dim, float softmax_scale, const int32_t* sched,
                                 const int32_t* sched_cnt, int64_t sched_stride_b, int64_t sched_stride_h,
                                 int sched_cap, int num_pairs, const int32_t* q_off, const int32_t* q_len, int nqb,
                                 const int32_t* kv_off, const int32_t* kv_len, int nkb, void* stream) {
  FVB_CHECK_ARG(q && k && v && o, "null pointer");
  FVB_CHECK_ARG(head_dim == ATT_D, "head_dim must be 128");
  FVB_CHECK_ARG(B > 0 && H > 0 && Sq > 0 && Skv > 0, "empty problem");
  if (sched != nullptr) FVB_CHECK_ARG(sched_cnt != nullptr && sched_cap > 0 && num_pairs > 0 && nqb > 0 && nkb > 0, "incomplete block schedule");
  AttnParams p = base_params(o, lse, lse_stride_b, lse_stride_h, B, H, Sq, Skv, softmax_scale, q_off, q_len, nqb, kv_off, kv_len, nkb);
  p.sched = sched;
  p.sched_cnt = sched_cnt;
  p.sched_stride_b = sched_stride_b;
  p.sched_stride_h = sched_stride_h;
  p.sched_cap = sched_cap;
  return launch_attention(q, k, v, q_strides, k_strides, v_strides, o_strides, p, sched ? num_pairs : (Sq + 127) / 128, stream);
}

// Kept for ABI compatibility: the block-list path needs no workspace (the two lists of a CTA are merged while they are
// walked), so callers allocate the minimum.
extern "C" int64_t fvb_attention_blocklist_workspace_bytes(int, int, int) { return 256; }

extern "C" int fvb_attention_blocklist_fwd(const void* q, const void* k, const void* v, void* o, float* lse,
                                           const int64_t* q_strides, const int64_t* k_strides, const int64_t* v_strides,
                                           const int64_t* o_strides, int64_t lse_stride_b, int64_t lse_stride_h, int B, int H,
                                           int Sq, int Skv, int head_dim, float softmax_scale, const int32_t* q2k_idx,
                                           const int32_t* q2k_num, int64_t idx_stride_b, int64_t idx_stride_h, int cap,
                                           const int32_t* q_off, const int32_t* q_len, int nqb, const int32_t* kv_off,
                                           const int32_t* kv_len, int nkb, void* workspace, int64_t workspace_bytes,
                                           void* stream) {
  (void)workspace;
  (void)workspace_bytes;
  FVB_CHECK_ARG(q && k && v && o && q2k_idx && q2k_num, "null pointer");
  FVB_CHECK_ARG(head_dim == ATT_D, "head_dim must be 128");
  FVB_CHECK_ARG(B > 0 && H > 0 && Sq > 0 && Skv > 0 && nqb > 0 && nkb > 0 && cap > 0, "empty problem");
  FVB_CHECK_ARG((idx_stride_h == 0 || idx_stride_h == nqb) &&
                    (idx_stride_b == 0 || idx_stride_b == (idx_stride_h ? int64_t(H) * nqb : int64_t(nqb))),
                "index tensors must be contiguous [B or 1, H or 1, nqb, cap]");
  AttnParams p = base_params(o, lse, lse_stride_b, lse_stride_h, B, H, Sq, Skv, softmax_scale, q_off, q_len, nqb, kv_off, kv_len, nkb);
  p.q2k_idx = q2k_idx;
  p.q2k_num = q2k_num;
  p.idx_stride_b = idx_stride_b;
  p.idx_stride_h = idx_stride_h;
  p.cap = cap;
  return launch_attention(q, k, v, q_strides, k_strides, v_strides, o_strides, p, (nqb + 1) / 2, stream);
}

// ------------------------------ 8-bit operands (fvb_attention_8bit_fwd) ------------------------------
extern "C" int fvb_attention_8bit_fwd(const void* q8, const float* q_scale, const void* k8, const float* k_scale,
                                      const void* vt8, const float* v_scale, void* o, float* lse, const int64_t* o_strides,
                                      int B, int H, int Sq, int Skv, int head_dim, float softmax_scale, const int32_t* sched,
                                      const int32_t* q2k_idx, const int32_t* q2k_num, int64_t idx_stride_b,
                                      int64_t idx_stride_h, int cap, const int32_t* q_off, const int32_t* q_len, int nqb,
                                      const int32_t* kv_off, const int32_t* kv_len, int nkb, void* stream) {
  FVB_CHECK_ARG(q8 && q_scale && k8 && k_scale && vt8 && v_scale && o && o_strides, "null pointer");
  if (sched != nullptr) return set_error(FVB_ERR_UNSUPPORTED, "8-bit attention has no pair-schedule (STA) mode%s");
  FVB_CHECK_ARG(lse == nullptr, "8-bit attention writes no LSE: lse must be NULL");
  FVB_CHECK_ARG(head_dim == ATT_D, "head_dim must be 128");
  FVB_CHECK_ARG(B > 0 && H > 0 && Sq > 0 && Skv > 0 && nkb > 0, "empty problem");
  FVB_CHECK_ARG(H <= 65535 && B <= 65535, "too many heads / batches");
  FVB_CHECK_ARG(int64_t(B) * H * nkb * ATT_D < (int64_t(1) << 31), "too many key blocks");
  if (kv_off == nullptr) FVB_CHECK_ARG(nkb == (Skv + 63) / 64, "without kv_off, nkb must be ceil(Skv / 64)");
  if (q2k_idx != nullptr) {
    FVB_CHECK_ARG(q2k_num != nullptr && nqb > 0 && cap > 0, "incomplete block lists");
    FVB_CHECK_ARG((idx_stride_h == 0 || idx_stride_h == nqb) &&
                      (idx_stride_b == 0 || idx_stride_b == (idx_stride_h ? int64_t(H) * nqb : int64_t(nqb))),
                  "index tensors must be contiguous [B or 1, H or 1, nqb, cap]");
  } else {
    FVB_CHECK_ARG(q2k_num == nullptr, "q2k_num without q2k_idx");
  }
  for (int i = 0; i < 3; ++i) FVB_CHECK_ARG(o_strides[i] % 8 == 0, "o strides must be multiples of 8 elements");
  AttnParams p = base_params(o, nullptr, 0, 0, B, H, Sq, Skv, softmax_scale, q_off, q_len, nqb, kv_off, kv_len, nkb);
  p.q2k_idx = q2k_idx;
  p.q2k_num = q2k_num;
  p.idx_stride_b = idx_stride_b;
  p.idx_stride_h = idx_stride_h;
  p.cap = cap;
  p.q_scale = q_scale;
  p.k_scale = k_scale;
  p.v_scale = v_scale;
  p.o_stride_b = o_strides[0];
  p.o_stride_s = o_strides[1];
  p.o_stride_h = o_strides[2];
  // q8 / k8: int8 [B, H, S, 128]; vt8: e4m3 [B * H * nkb * 128 channel rows][64 key slots]
  CUtensorMap tmQ, tmK, tmV;
  int r;
  {
    uint64_t dims[4] = {(uint64_t)ATT_D, (uint64_t)Sq, (uint64_t)H, (uint64_t)B};
    uint64_t str[4] = {1, (uint64_t)ATT_D, (uint64_t)Sq * ATT_D, (uint64_t)H * Sq * ATT_D};
    uint32_t box[4] = {ATT_D, 64, 1, 1};
    if ((r = make_tmap_u8(&tmQ, q8, 4, dims, str, box))) return r;
  }
  {
    uint64_t dims[4] = {(uint64_t)ATT_D, (uint64_t)Skv, (uint64_t)H, (uint64_t)B};
    uint64_t str[4] = {1, (uint64_t)ATT_D, (uint64_t)Skv * ATT_D, (uint64_t)H * Skv * ATT_D};
    uint32_t box[4] = {ATT_D, 64, 1, 1};
    if ((r = make_tmap_u8(&tmK, k8, 4, dims, str, box))) return r;
  }
  {
    uint64_t dims[2] = {64, (uint64_t)B * H * nkb * ATT_D};
    uint64_t str[2] = {1, 64};
    uint32_t box[2] = {64, ATT_D};
    if ((r = make_tmap_u8(&tmV, vt8, 2, dims, str, box, CU_TENSOR_MAP_SWIZZLE_64B))) return r;
  }
  const int n_pairs = q2k_idx ? (nqb + 1) / 2 : (Sq + 127) / 128;
  return launch_kernel<true>(tmQ, tmK, tmV, p, n_pairs, stream);
}
