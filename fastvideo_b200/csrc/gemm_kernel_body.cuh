// gemm_kernel_body.cuh -- the body of the sm_90a GEMM kernel (gemm_sm90.cu), included by gemm_kernel and gemm_aux_kernel.
// In scope: the template parameters BN, EPI, FP8, W8, I8, TA, TB, the kernel parameters tmA, tmB, p, and AUX (p.aux / p.ldaux
// receive the bf16 y = bf16(acc + bias) of every element before the epilogue consumes it).
  static_assert(!((TA || TB) && (FP8 || W8 || I8)), "transposed operands are bf16 only: e4m3 / s8 wgmma has no transpose bits");
  static_assert(TB || !TA, "the transposed producer loads B MN-major: TA comes with TB (wgrad)");
  using Cfg = GemmCfg<BN>;
  constexpr int BK = FP8 || I8 ? GEMM_BK_FP8 : GEMM_BK;
  using Acc = std::conditional_t<I8, int32_t, float>;
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
    if constexpr (W8)
      for (int i = 0; i < Cfg::STAGES; ++i) mbar_init(&bars[2 * Cfg::STAGES + i], 1);  // `landed` below
    fence_mbar_init();
  }
  __syncthreads();

  if (wg == 0) {
    // ------------------------------ TMA producer ------------------------------
    reg_dealloc<40>();
    if constexpr (W8) {
      // thread 0 issues the TMA loads onto `landed`; warps 1-3 widen each landed weight tile, then release the stage to
      // the consumers on `full`
      uint64_t* landed = bars + 2 * Cfg::STAGES;
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        int m_blk, n_blk;
        const int bt = tile / tiles_per_batch;
        tile_coords(tile - bt * tiles_per_batch, p.num_m, p.num_n, p.stripe_n, m_blk, n_blk);
        for (int kb = 0; kb < p.num_k; ++kb) {
          uint8_t* sa = smem + stage * Cfg::STAGE_BYTES;
          uint8_t* sb = sa + Cfg::A_BYTES;
          if (threadIdx.x == 0) {
            mbar_wait(&empty[stage], phase ^ 1);
            mbar_expect_tx(&landed[stage], Cfg::A_BYTES + BN * GEMM_BK);
            const int k0 = kb * GEMM_BK;
            const int seg = k0 / p.a_seg_len;
            tma_load_4d(sa, &tmA, &landed[stage], k0 - seg * p.a_seg_len, m_blk * GEMM_BM, seg, bt);
            tma_load_3d(sb + W8_STAGING_OFFSET<BN>, &tmB, &landed[stage], k0, n_blk * BN, bt);
          } else if (threadIdx.x >= 32) {
            mbar_wait(&landed[stage], phase);
            w8_widen_tile<BN>(smem_u32(sb), threadIdx.x - 32);
            fence_proxy_async();  // the generic-proxy stores are read by wgmma (async proxy)
            named_bar_sync(1, W8_CONVERT_THREADS);
            if (threadIdx.x == 32) mbar_arrive(&full[stage]);
          }
          if (++stage == Cfg::STAGES) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
      return;
    }
    if constexpr (TA || TB) {
      // MN-major operands: one 2-D TMA per 64-wide chunk ([K][MN] maps; MN and K tails zero-filled), chunk-major in the stage.
      // A K-major A (TB only) is the forward's 4-D load.
      if (threadIdx.x == 0) {
        int stage = 0;
        uint32_t phase = 0;
        for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
          int m_blk, n_blk;
          tile_coords(tile, p.num_m, p.num_n, p.stripe_n, m_blk, n_blk);
          for (int kb = 0; kb < p.num_k; ++kb) {
            mbar_wait(&empty[stage], phase ^ 1);
            uint8_t* sa = smem + stage * Cfg::STAGE_BYTES;
            uint8_t* sb = sa + Cfg::A_BYTES;
            mbar_expect_tx(&full[stage], Cfg::STAGE_BYTES);
            if constexpr (TA) {
#pragma unroll
              for (int c = 0; c < GEMM_BM / GEMM_MN_CHUNK; ++c)
                tma_load_2d(sa + c * GEMM_MN_CHUNK_BYTES, &tmA, &full[stage], m_blk * GEMM_BM + c * GEMM_MN_CHUNK, kb * BK);
            } else {
              tma_load_4d(sa, &tmA, &full[stage], kb * BK, m_blk * GEMM_BM, 0, 0);
            }
#pragma unroll
            for (int c = 0; c < BN / GEMM_MN_CHUNK; ++c)
              tma_load_2d(sb + c * GEMM_MN_CHUNK_BYTES, &tmB, &full[stage], n_blk * BN + c * GEMM_MN_CHUNK, kb * BK);
            if (++stage == Cfg::STAGES) {
              stage = 0;
              phase ^= 1;
            }
          }
        }
      }
      return;
    }
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
            const int k0 = kb * BK;
            const int seg = k0 / p.a_seg_len;
            tma_load_4d(sa, &tmA, &full[stage], k0 - seg * p.a_seg_len, m_blk * GEMM_BM, seg, bt);
          }
          tma_load_3d(sb, &tmB, &full[stage], kb * BK, n_blk * BN, bt);
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
    Acc acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = Acc(0);
    int prev = -1;
    if constexpr (FP8) {
      // per k-block partial sums in `part` (the first MMA overwrites it), promoted into the fp32 accumulators after the
      // k-block's MMAs complete; the other consumer warpgroup keeps the tensor cores busy meanwhile
      float part[BN / 2];
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) part[i] = 0.f;
      for (int kb = 0; kb < p.num_k; ++kb) {
        mbar_wait(&full[stage], phase);
        const uint32_t sa = smem_u32(smem + stage * Cfg::STAGE_BYTES) + half * (64 * 128);
        const uint32_t sb = smem_u32(smem + stage * Cfg::STAGE_BYTES + Cfg::A_BYTES);
        const uint64_t da = make_desc_kmajor_sw128(sa);
        const uint64_t db = make_desc_kmajor_sw128(sb);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < GEMM_BK_FP8 / 32; ++k) wgmma_ss_e4m3<BN>(part, da + uint64_t(2 * k), db + uint64_t(2 * k), k);
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(part);
        if (lane == 0) mbar_arrive(&empty[stage]);
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[i] = __fadd_rn(acc[i], part[i]);
        if (++stage == Cfg::STAGES) {
          stage = 0;
          phase ^= 1;
        }
      }
    } else {
    for (int kb = 0; kb < p.num_k; ++kb) {
      mbar_wait(&full[stage], phase);
      const uint32_t sa = smem_u32(smem + stage * Cfg::STAGE_BYTES) + half * (64 * 128);
      const uint32_t sb = smem_u32(smem + stage * Cfg::STAGE_BYTES + Cfg::A_BYTES);
      const uint64_t da = make_desc_kmajor_sw128(sa);
      const uint64_t db = make_desc_kmajor_sw128(sb);
      wgmma_fence();
      if constexpr (I8) {
#pragma unroll
        for (int k = 0; k < GEMM_BK_FP8 / 32; ++k) wgmma_ss_s8<BN>(acc, da + uint64_t(2 * k), db + uint64_t(2 * k), 1);
      } else if constexpr (TA || TB) {
        // MN-major: this warpgroup's 64 A rows are chunk `half` (the same +8 KB as the K-major half); chunks are 8 KB apart
        // (LBO), 8-row k groups 1024 B (SBO); a k16 step is 16 rows of 128 B (+128 on the descriptor)
        const uint64_t ta = TA ? make_desc_mnmajor_sw128(sa, GEMM_MN_CHUNK_BYTES) : da;
        const uint64_t tb = TB ? make_desc_mnmajor_sw128(sb, GEMM_MN_CHUNK_BYTES) : db;
#pragma unroll
        for (int k = 0; k < GEMM_BK / 16; ++k)
          wgmma_ss_trans<BN, TA, TB>(acc, ta + uint64_t(k * (TA ? 128 : 2)), tb + uint64_t(k * (TB ? 128 : 2)));
      } else {
#pragma unroll
        for (int k = 0; k < GEMM_BK / 16; ++k) wgmma_ss<BN>(acc, da + uint64_t(2 * k), db + uint64_t(2 * k));
      }
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
    }

    // ------------------------------ epilogue ------------------------------
    const int row0 = m_blk * GEMM_BM + half * 64 + warp * 16 + (lane >> 2);
    const float* gate_rows_p[2] = {p.gate, p.gate};
    if constexpr (EPI != FVB_EPI_RESID_BF16)
      if (p.gate_rows > 0)
        for (int i = 0; i < 2; ++i) gate_rows_p[i] += int64_t((row0 + 8 * i) / p.gate_rows) * p.gate_stride;
    float sx[2] = {1.f, 1.f};
    if constexpr (FP8 || I8)
      for (int i = 0; i < 2; ++i) sx[i] = row0 + 8 * i < p.M ? __ldg(p.a_scale + row0 + 8 * i) : 0.f;
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      const int col = n_blk * BN + 8 * j + 2 * (lane & 3);
      if (col >= p.N) continue;  // N is a multiple of 8: the pair (col, col + 1) is inside or outside together
      const int64_t out_col = p.out_col_offsets ? __ldg(p.out_col_offsets + (col >> 7)) + (col & 127) : int64_t(col);
      float2 bf = make_float2(0.f, 0.f);
      if (p.bias != nullptr) bf = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(p.bias + col));
      float2 sw = make_float2(1.f, 1.f);
      if constexpr (FP8 || W8 || I8) {
        sw.x = col < p.N_valid ? __ldg(p.b_scale + col) : 0.f;
        sw.y = col + 1 < p.N_valid ? __ldg(p.b_scale + col + 1) : 0.f;
      }
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int row = row0 + 8 * i;
        if (row >= p.M) continue;
        // I8: float(acc) rounds to nearest (exact up to 2^24)
        float f0 = acc_f32(acc[4 * j + 2 * i]), f1 = acc_f32(acc[4 * j + 2 * i + 1]);
        if constexpr (FP8 || I8) {  // (acc * s_x[m]) * s_w[n], fp32 round-to-nearest, before the bias
          f0 = __fmul_rn(__fmul_rn(f0, sx[i]), sw.x);
          f1 = __fmul_rn(__fmul_rn(f1, sx[i]), sw.y);
        } else if constexpr (W8) {  // acc * s_w[n], fp32 round-to-nearest, before the bias
          f0 = __fmul_rn(f0, sw.x);
          f1 = __fmul_rn(f1, sw.y);
        }
        if (p.bias != nullptr) {
          f0 = __fadd_rn(f0, bf.x);
          f1 = __fadd_rn(f1, bf.y);
        }
        // y = bf16(acc + bias) in every mode (the reference's F.linear output dtype)
        if constexpr (AUX) *reinterpret_cast<uint32_t*>(p.aux + int64_t(row) * p.ldaux + col) = pack_bf16x2(f0, f1);
        if constexpr (EPI == FVB_EPI_BIAS_GELU_TANH) {
          f0 = gelu_tanh_f(bf16_round(f0));
          f1 = gelu_tanh_f(bf16_round(f1));
        } else if constexpr (EPI == FVB_EPI_DIV) {
          f0 = __fdiv_rn(bf16_round(f0), p.div);
          f1 = __fdiv_rn(bf16_round(f1), p.div);
        } else if constexpr (EPI == EPI_DGELU_TANH) {
          const float2 h = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(p.resid + int64_t(row) * p.ldr + col));
          f0 = __fmul_rn(bf16_round(f0), gelu_tanh_grad_f(h.x));
          f1 = __fmul_rn(bf16_round(f1), gelu_tanh_grad_f(h.y));
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
