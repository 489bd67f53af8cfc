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
#include "fvb_host.cuh"
#include "fvb_ptx.cuh"

namespace fvb {

constexpr int ATT_D = 128;
constexpr int ATT_THREADS = 288;
constexpr int ATT_STAGES = 4;
constexpr int ATT_TILE_BYTES = 64 * ATT_D * 2;  // 16 KB: [d half (2)][64 rows][128 B]
constexpr int ATT_HALF_BYTES = 64 * 128;        // 8 KB
constexpr int ATT_SMEM_BYTES = ATT_TILE_BYTES * (2 + 2 * ATT_STAGES) + 1024 + 256;

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
};

// The CTA's walk over key blocks: next() yields (kv block, flags) in ascending order, flags bit s = q block s attends.
// Every thread runs its own copy over the same global lists, so producer and consumers agree without communication.
struct KeyWalk {
  const int32_t* l0;
  const int32_t* l1;
  int n0, n1, i0, i1;
  int mode;  // 0 dense, 1 pair list, 2 two q-block lists

  FVB_DEVICE bool next(int& kb, int& flags) {
    if (mode == 2) {
      const int a = i0 < n0 ? __ldg(l0 + i0) : 0x7fffffff;
      const int b = i1 < n1 ? __ldg(l1 + i1) : 0x7fffffff;
      if (a == 0x7fffffff && b == 0x7fffffff) return false;
      kb = min(a, b);
      flags = (a == kb ? 1 : 0) | (b == kb ? 2 : 0);
      i0 += a == kb;
      i1 += b == kb;
      return true;
    }
    if (i0 >= n0) return false;
    if (mode == 0) {
      kb = i0++;
      flags = 3;
      return true;
    }
    const int ent = __ldg(l0 + i0++);
    kb = ent & 0xFFFFFF;
    flags = (ent >> 24) & 3;
    return true;
  }
};

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

__global__ void __launch_bounds__(ATT_THREADS, 1)
attn_fwd_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                const __grid_constant__ CUtensorMap tmV, const AttnParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;  // [q block (2)][tile]
  uint8_t* sK = smem + 2 * ATT_TILE_BYTES;
  uint8_t* sV = sK + ATT_STAGES * ATT_TILE_BYTES;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sV + ATT_STAGES * ATT_TILE_BYTES);
  uint64_t* q_full = bars;                    // 1
  uint64_t* k_full = bars + 1;                // STAGES
  uint64_t* v_full = k_full + ATT_STAGES;     // STAGES
  uint64_t* kv_empty = v_full + ATT_STAGES;   // STAGES

  const int pair = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const bool dense = p.sched == nullptr && p.q2k_idx == nullptr;

  // this CTA's key walk
  KeyWalk walk;
  walk.i0 = walk.i1 = 0;
  walk.l0 = walk.l1 = nullptr;
  walk.n1 = 0;
  if (dense) {
    walk.mode = 0;
    walk.n0 = (p.Skv + 63) / 64;
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
      mbar_expect_tx(q_full, 2 * ATT_TILE_BYTES);
#pragma unroll
      for (int s = 0; s < 2; ++s)
#pragma unroll
        for (int hf = 0; hf < 2; ++hf)
          tma_load_4d(sQ + s * ATT_TILE_BYTES + hf * ATT_HALF_BYTES, &tmQ, q_full, hf * 64, q_row0[s], h, b);
      int stage = 0;
      uint32_t phase = 0;
      int kb, flags;
      while (walk.next(kb, flags)) {
        int row0, vlen;
        kv_rows(p, dense, kb, row0, vlen);
        mbar_wait(&kv_empty[stage], phase ^ 1);
        mbar_expect_tx(&k_full[stage], ATT_TILE_BYTES);
        for (int hf = 0; hf < 2; ++hf)
          tma_load_4d(sK + stage * ATT_TILE_BYTES + hf * ATT_HALF_BYTES, &tmK, &k_full[stage], hf * 64, row0, h, b);
        mbar_expect_tx(&v_full[stage], ATT_TILE_BYTES);
        for (int hf = 0; hf < 2; ++hf)
          tma_load_4d(sV + stage * ATT_TILE_BYTES + hf * ATT_HALF_BYTES, &tmV, &v_full[stage], hf * 64, row0, h, b);
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
  const uint32_t qa = smem_u32(sQ + s * ATT_TILE_BYTES);
  float o[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) o[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
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
    kv_rows(p, dense, kb, row0, vlen);
    const uint32_t ka = smem_u32(sK + stage * ATT_TILE_BYTES);
    const uint32_t va = smem_u32(sV + stage * ATT_TILE_BYTES);
    float sc[32];
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
          const float x = key < vlen ? sc[4 * j + 2 * i + c] * p.scale_log2 : -INFINITY;
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
    if (++stage == ATT_STAGES) {
      stage = 0;
      phase ^= 1;
    }
  }

  // ------------------------------ epilogue ------------------------------
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    float l = l_run[i];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const int r = 16 * wq + (lane >> 2) + 8 * i;
    if (r >= q_rows[s]) continue;
    const int tok = q_row0[s] + r;
    const float inv = l > 0.f ? 1.f / l : 0.f;
    __nv_bfloat16* op = p.o + int64_t(b) * p.o_stride_b + int64_t(tok) * p.o_stride_s + int64_t(h) * p.o_stride_h;
#pragma unroll
    for (int j = 0; j < 16; ++j)
      *reinterpret_cast<uint32_t*>(op + 8 * j + 2 * tq) = pack_bf16x2(o[4 * j + 2 * i] * inv, o[4 * j + 2 * i + 1] * inv);
    if (tq == 0 && p.lse != nullptr)
      p.lse[int64_t(b) * p.lse_stride_b + int64_t(h) * p.lse_stride_h + tok] = l > 0.f ? m_run[i] + log2f(l) : -INFINITY;
  }
}

static int make_qkv_tmap(CUtensorMap* tm, const void* base, int64_t S, int64_t H, int64_t B, int64_t stride_s,
                         int64_t stride_h, int64_t stride_b) {
  uint64_t dims[4] = {(uint64_t)ATT_D, (uint64_t)S, (uint64_t)H, (uint64_t)B};
  uint64_t str[4] = {2, (uint64_t)stride_s * 2, (uint64_t)stride_h * 2, (uint64_t)stride_b * 2};
  uint32_t box[4] = {64, 64, 1, 1};
  return make_tmap_bf16(tm, base, 4, dims, str, box);
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
  static bool configured = false;
  if (!configured) {
    FVB_CHECK_CUDA(cudaFuncSetAttribute(attn_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, ATT_SMEM_BYTES));
    configured = true;
  }
  dim3 grid(unsigned(n_pairs), unsigned(p.H), unsigned(p.B));
  attn_fwd_kernel<<<grid, ATT_THREADS, ATT_SMEM_BYTES, reinterpret_cast<cudaStream_t>(stream)>>>(tmQ, tmK, tmV, p);
  FVB_CHECK_CUDA(cudaGetLastError());
  return FVB_OK;
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
