// pxa_gemm_bf16: out = epilogue(A[M,K] . W[N,K]^T + bias) on wgmma tensor cores (sm_90a).
//
// Structure (one persistent CTA per SM, 384 threads = 3 warpgroups):
//   warp 0       TMA producer: A tile 128x64 and W tile BNx64 (bf16, 128B-swizzled) into a kStages-deep smem ring, and the
//                tile's epilogue operand (fp32 / bf16 residual, bf16 pre-activation) into the output tile in smem
//                (the rest of its warpgroup gives its registers away with setmaxnreg and idles)
//   warps 4-11   two consumer warpgroups.  Warpgroup g owns the 128 x BN/2 half [g BN/2, (g+1) BN/2) of the tile: per K-block
//                it issues 2 (64-row halves) x 4 (K steps) wgmma.mma_async m64 x BN/2 x 16 with both operands read from the
//                ring through shared-memory descriptors, fp32 accumulators in registers (BN/2 per thread).
//                Epilogue: bias / GELU / gate * x + residual / LayerNorm-modulate are applied to the accumulator fragments,
//                the results are written into the warpgroup's half of the swizzled output tile (over the operand) and one
//                thread issues TMA stores of its 128 x 32 slabs; the warpgroup goes on to the next tile's MMAs while the stores
//                drain.  Before the output tile is written again, the storing thread waits for the stores' smem reads
//                (cp.async.bulk.wait_group.read), part way into the next main loop, and then lets the producer load the
//                next operand into it.
// Tiles are visited n-fastest so the CTAs running concurrently share the same few A row-blocks through L2 and the
// whole weight matrix stays L2-resident.
//
// K-tail (kTail, pxa_gemm_lora_bf16): after the tile's last K-block of A W^T the producer loads ceil(tail_k / 64) more
// K-blocks from the tail operands (tail_a [M, tail_k], tail_w [N, tail_k]) into the same ring, and the consumers run the same
// wgmma loop over them: the epilogue sees A W^T + tail_a tail_w^T.  TMA zero-fills the columns past tail_k.
//
// Column scale (kScale, pxa_gemm_dora_bf16): the epilogue multiplies accumulator column n by col_scale[n] before anything
// else (bias, GELU, gate, residual, aux copies), the DoRA magnitude-over-norm factor of an adapted projection.
//
// Algorithmic work: 2*M*N*K FLOP; bytes: M*K*2 (A) + N*K*2 (W) + M*N*out bytes (+ residual read).
#include "gemm_common.cuh"

namespace pxa {

// Tensor maps of the K-tail operands; empty in the instantiations without a tail.
template <bool kTail> struct TailMaps {
  CUtensorMap a, w;
  int num_kb;
};
template <> struct TailMaps<false> {};

// K-block of a tile (counted from the tile's first) after which the consumers release the output tile of the previous tile:
// late enough for its stores to have drained, early enough for the next operand to arrive before the tile's epilogue.
PXA_DEVICE int release_kb(int nk) {
  const int q = nk / 4 > 1 ? nk / 4 : 1;
  return q < nk - 1 ? q : nk - 1;
}

// ------------------------------------------------------------------------------------------------- kernel
// kMn: both operands are given MN-major -- A as [K, M] (M contiguous), W as [K, N] (N contiguous) -- the layout of the
// weight-gradient product dW[N, K] = dY[M, N]^T X[M, K], whose contraction runs over the token dimension.  Each K-block
// is staged as 64-wide swizzle atoms of 64 k-rows (two for the 128 rows of A, BN / 64 for W) and consumed through
// MN-major descriptors (atoms LBO apart, 16 k-rows = 2048 B per K-step).  With p.k_splits > 1 the K range is split
// across tiles (split-K); legal only with the reduce-add form of the fp32 residual epilogue: the output tile is added into
// `out` by TMA reductions, so that the partial sums add up in L2.
//
// tmap_out / tmap_res: `out` and the epilogue operand as 3-D tensors (column, x, line) with 32 x 128 x 1 boxes.  x runs over
// the GEMM rows (one line), except for a convolution over a virtual width, where it runs over the W real pixels of an image
// line: the stores drop the columns x >= W and the rows >= M.
template <int BN, int EPI, typename OutT, bool kConv = false, bool kMn = false, bool kTail = false, bool kScale = false>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_bf16_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_w,
                 const __grid_constant__ CUtensorMap tmap_out, const __grid_constant__ CUtensorMap tmap_res, const GemmParams p,
                 const __grid_constant__ TailMaps<kTail> tail) {
  constexpr bool kF32Res = (EPI == PXA_EPI_BIAS_RESIDUAL) && sizeof(OutT) == 4;
  constexpr bool kRes = EPI == PXA_EPI_BIAS_RESIDUAL;
  constexpr bool kLn = (EPI == PXA_EPI_LN_BIAS || EPI == PXA_EPI_LN_BIAS_GELU);
  using Cfg = GemmCfg<BN, OutT>;
  constexpr int kStages = Cfg::kStages;
  constexpr int NW = BN / 2;                       // columns per consumer warpgroup
  constexpr int kSlabs = NW / 32;                  // output slabs per consumer warpgroup
  static_assert(!kMn || NW % 64 == 0, "MN-major W is staged in 64-column atoms");
  static_assert(!kTail || (!kConv && !kMn && !kLn), "the K-tail belongs to the K-major, non-LayerNorm forms");
  static_assert(!kScale || (!kConv && !kMn && !kLn && EPI != PXA_EPI_MUL_DGELU), "the column scale belongs to the forward forms");
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* otile = smem + kStages * Cfg::kStage;                                  // output tile: slab cs at cs * kSlabBytes
  EpiConst<BN>* consts = reinterpret_cast<EpiConst<BN>*>(otile + Cfg::kEpiTile);
  float2* rowbuf = reinterpret_cast<float2*>(otile + Cfg::kEpiTile + Cfg::kConstBytes);
  uint64_t* bars = reinterpret_cast<uint64_t*>(otile + Cfg::kEpiSmem);
  uint64_t* full_bar = bars;                    // [kStages]  TMA -> consumers
  uint64_t* empty_bar = bars + kStages;         // [kStages]  consumers -> TMA (one arrival per consumer warp)
  uint64_t* opnd_full = bars + 2 * kStages;     // the tile's epilogue operand has landed in the output tile
  uint64_t* opnd_empty = opnd_full + 1;         // the previous tile's stores have read the output tile (one arrival per warpgroup)

  const int warp = warp_idx_sync();
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    prefetch_tmap(&tmap_a);
    prefetch_tmap(&tmap_w);
    prefetch_tmap(&tmap_out);
    if constexpr (kTail) {
      prefetch_tmap(&tail.a);
      prefetch_tmap(&tail.w);
    }
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], kNumEpiThreads / 32);
    }
    mbar_init(opnd_full, 1);
    mbar_init(opnd_empty, 2);
    fence_mbar_init();
  }
  __syncthreads();

  const int mn_tiles = p.num_m_tiles * p.num_n_tiles;
  const int num_tiles = mn_tiles * p.k_splits;
  const int num_kb = (p.K + kBK - 1) / kBK;
  int tail_kb = 0;                              // K-blocks of the tail, after the last K-block of every tile (k_splits == 1)
  if constexpr (kTail) tail_kb = tail.num_kb;
  // tile -> (k split, m tile, n tile), n fastest; K-blocks [kb_lo, kb_hi) of split ks
  auto eff = [&](int tile) { return p.reverse_tiles ? num_tiles - 1 - tile : tile; };
  auto kb_lo = [&](int tile) { return (int)((long long)(tile / mn_tiles) * num_kb / p.k_splits); };
  auto kb_hi = [&](int tile) { return (int)((long long)(tile / mn_tiles + 1) * num_kb / p.k_splits); };
  auto tile_m0 = [&](int tile) { return ((tile % mn_tiles) / p.num_n_tiles) * kBM; };
  auto tile_n0 = [&](int tile) { return ((tile % mn_tiles) % p.num_n_tiles) * BN; };
  // (x, line) of the tile's first output row in tmap_out / tmap_res
  auto out_xy = [&](int m0) {
    if (kConv && p.conv_Wp != p.conv_W) return make_int2(m0 % p.conv_Wp, m0 / p.conv_Wp);
    return make_int2(m0, 0);
  };
  // in-place split-K accumulation: partial sums are added into `out` (no residual read)
  const bool reduce = kF32Res && p.k_splits > 1;
  // the epilogue reads a [M, N] operand laid out like `out`: the residual, or the pre-activation of EPI_MUL_DGELU
  const bool has_opnd = (kRes && !reduce) || EPI == PXA_EPI_MUL_DGELU;

  if (warp < kEpiWarp0) {
    // ================================================================ TMA producer
    reg_dealloc<40>();
    if (warp == 0 && elect_one()) {
      if (has_opnd) prefetch_tmap(&tmap_res);
      int stage = 0;
      uint32_t phase = 0;
      int titer = 0;
      for (int t = blockIdx.x; t < num_tiles; t += gridDim.x, ++titer) {
        const int tile = eff(t);
        const int m0 = tile_m0(tile);
        const int n0 = tile_n0(tile);
        const int kb0 = kb_lo(tile), kb1 = kb_hi(tile) + tail_kb;
        const int rel = release_kb(kb1 - kb0);
        for (int kb = kb0; kb < kb1; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = smem + stage * Cfg::kStage;
          uint8_t* sb = sa + Cfg::kStageA;
          mbar_arrive_expect_tx(&full_bar[stage], Cfg::kStage);
          if constexpr (kMn) {
#pragma unroll
            for (int i = 0; i < kBM / 64; ++i) tma_load_2d(sa + i * 8192, &tmap_a, &full_bar[stage], m0 + 64 * i, kb * kBK, kEvictNormal);
#pragma unroll
            for (int j = 0; j < BN / 64; ++j) tma_load_2d(sb + j * 8192, &tmap_w, &full_bar[stage], n0 + 64 * j, kb * kBK, kEvictNormal);
          } else {
            const CUtensorMap* ma = &tmap_a;
            const CUtensorMap* mw = &tmap_w;
            int kc = kb;                                              // K-block within its operand pair
            if constexpr (kTail) {
              if (kb >= num_kb) { ma = &tail.a; mw = &tail.w; kc = kb - num_kb; }
            }
            if constexpr (kConv) {
              // implicit GEMM: K-block kb = (tap, 64-channel slice); the A tile is the tile's pixel block shifted by the
              // tap offset -- zero padding comes for free from TMA out-of-bounds fill on the W / H dimensions
              const int tap = kb / p.conv_cin_blocks;
              const int c0 = (kb - tap * p.conv_cin_blocks) * kBK;
              const int pix = m0;                                     // first pixel of the tile in (b, y, x) order of the virtual image
              const int x0 = pix % p.conv_Wp;
              const int y0 = (pix / p.conv_Wp) % p.conv_H;
              const int b0 = pix / (p.conv_Wp * p.conv_H);
              tma_load_4d(sa, &tmap_a, &full_bar[stage], c0, x0 + tap % 3 - 1, y0 + tap / 3 - 1, b0, kEvictNormal);
            } else {
              tma_load_2d(sa, ma, &full_bar[stage], kc * kBK, m0, kEvictNormal);
            }
            tma_load_2d(sb, mw, &full_bar[stage], kc * kBK, n0, kEvictLast);
          }
          if (++stage == kStages) { stage = 0; phase ^= 1; }
          if (has_opnd && kb - kb0 == rel) {
            // the consumers release the output tile at this K-block of the tile (see release_kb)
            mbar_wait(opnd_empty, titer & 1);
            const int slabs = (p.N - n0 + 31) / 32 < BN / 32 ? (p.N - n0 + 31) / 32 : BN / 32;
            mbar_arrive_expect_tx(opnd_full, slabs * Cfg::kSlabBytes);
            const int2 xy = out_xy(m0);
            for (int cs = 0; cs < slabs; ++cs)
              tma_load_3d(otile + cs * Cfg::kSlabBytes, &tmap_res, opnd_full, n0 + 32 * cs, xy.x, xy.y, kEvictNormal);
          }
        }
      }
    }
  } else {
    // ================================================================ consumers: wgmma main loop + epilogue
    reg_alloc<232>();
    const int g = (warp - kEpiWarp0) >> 2;          // consumer warpgroup = column half of the tile
    const int q = warp & 3;                         // this warp's 16-row slice of each 64-row half of the tile
    const int tid = threadIdx.x - kEpiWarp0 * 32;   // 0..255
    const bool storer = (tid & 127) == 0;           // issues and waits for this warpgroup's TMA stores
    int stage = 0;
    uint32_t phase = 0;
    int titer = 0;
    EpiRegs<BN> er;                                                // constants / LN statistics of a tile, loaded one tile ahead
    [[maybe_unused]] LnStatRegs sr;
    if ((int)blockIdx.x < num_tiles) {
      const int ft = eff(blockIdx.x);
      load_epi_consts<BN, kLn, kScale>(er, p, tid, tile_m0(ft), tile_n0(ft));
      if constexpr (kLn) if (g == 0) load_ln_stats(sr, p, tile_m0(ft) + tid);
    }
    float acc[2][NW / 2];
    for (int t = blockIdx.x; t < num_tiles; t += gridDim.x, ++titer) {
      const int tile = eff(t);
      const int m0 = tile_m0(tile);
      const int n0 = tile_n0(tile);
      // ---- main loop
      // One wgmma group stays in flight: the group of K-block kb is committed before the group of kb - 1 is waited for, and a
      // stage goes back to the producer once the group that read it has completed.
      const int kb0 = kb_lo(tile), kb1 = kb_hi(tile) + tail_kb;
      const int rel = release_kb(kb1 - kb0);
      int prev_stage = -1;
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t sa = smem_u32(smem + stage * Cfg::kStage);
        const uint32_t sb = sa + Cfg::kStageA + (kMn ? (g * NW / 64) * 8192 : g * NW * 128);
        // K-major: 8-row groups 1024 B apart; MN-major: 64-wide atoms 8192 B apart (LBO), 8 k-rows = 1024 B (SBO)
        const uint64_t adesc0 = make_smem_desc(sa, kMn ? 8192 : 16, 1024, kLayoutSW128);
        const uint64_t adesc1 = make_smem_desc(sa + 8192, kMn ? 8192 : 16, 1024, kLayoutSW128);   // rows 64..127 of the tile
        const uint64_t bdesc = make_smem_desc(sb, kMn ? 8192 : 16, 1024, kLayoutSW128);
        // one K-step = 16 elements along K: 32 B inside the swizzle atom (K-major) / 16 rows of 128 B (MN-major)
        constexpr int kStep = kMn ? (2048 >> 4) : 2;
        wgmma_fence_regs(acc[0]);
        wgmma_fence_regs(acc[1]);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kBK / 16; ++k) {
          const uint32_t accum = ((kb - kb0) | k) != 0 ? 1u : 0u;
          wgmma_ss<NW, kMn ? 1 : 0, kMn ? 1 : 0>(acc[0], adesc0 + kStep * k, bdesc + kStep * k, accum);
          wgmma_ss<NW, kMn ? 1 : 0, kMn ? 1 : 0>(acc[1], adesc1 + kStep * k, bdesc + kStep * k, accum);
        }
        wgmma_commit();
        wgmma_wait<1>();
        if (prev_stage >= 0 && lane == 0) mbar_arrive(&empty_bar[prev_stage]);   // this warp has finished reading that stage
        prev_stage = stage;
        if (++stage == kStages) { stage = 0; phase ^= 1; }
        if (kb - kb0 == rel && storer) {            // the previous tile's stores have read this warpgroup's slabs
          tma_store_wait_read<0>();
          if (has_opnd) mbar_arrive(opnd_empty);
        }
      }
      wgmma_wait<0>();
      wgmma_fence_regs(acc[0]);
      wgmma_fence_regs(acc[1]);
      if (prev_stage >= 0 && lane == 0) mbar_arrive(&empty_bar[prev_stage]);
      // ---- epilogue
      EpiConst<BN>* cb = consts + (titer & 1);
      float2* lnc = rowbuf + (titer & 1) * kBM;                    // LN consumer: (rstd, -rstd * mean) of each tile row
      store_epi_consts<BN>(cb, er, tid);
      if constexpr (kLn) if (g == 0) lnc[tid] = ln_row_coeffs(p, sr);
      named_bar_sync(2, kNumEpiThreads);
      if (has_opnd) mbar_wait(opnd_full, titer & 1);
      const int row_split = cb->row_split;
      // samples shorter than a tile (rows_per_batch < 128, tiny images): a tile may span more than two samples, so the gate row
      // is looked up per row in global memory instead of the two staged rows
      const bool per_row_gate = kRes && p.gate != nullptr && p.rows_per_batch < kBM;
      __nv_bfloat16* aux = p.out_aux;
      [[maybe_unused]] float2 st[2][2] = {};                        // (sum, sum of squares) of each of this thread's rows
      // fragment (i, j, h) of this thread: tile row 64 i + 16 q + lane / 4 + 8 h, warpgroup columns 8 j + 2 (lane % 4) + {0, 1}
#pragma unroll
      for (int s = 0; s < kSlabs; ++s) {
        const int cs = g * kSlabs + s;                              // slab of the tile (warpgroup-uniform)
        if (n0 + 32 * cs >= p.N) continue;
        uint8_t* slab = otile + cs * Cfg::kSlabBytes;
#pragma unroll
        for (int i = 0; i < 2; ++i)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int row = 64 * i + 16 * q + (lane >> 2) + 8 * h;
            const int grow = m0 + row;
            const bool second = row >= row_split;
            [[maybe_unused]] float2 ln = make_float2(1.f, 0.f);
            if constexpr (kLn) ln = lnc[row];
#pragma unroll
            for (int jj = 0; jj < 4; ++jj) {
              const int c = 8 * jj + 2 * (lane & 3);                // column in the slab
              const int tc = 32 * cs + c;                           // column in the tile
              const int gcol = n0 + tc;
              float a0 = acc[i][4 * (4 * s + jj) + 2 * h], a1 = acc[i][4 * (4 * s + jj) + 2 * h + 1];
              if constexpr (kScale) {
                const float2 cs = *reinterpret_cast<const float2*>(cb->ex1 + tc);
                a0 *= cs.x;
                a1 *= cs.y;
              }
              uint8_t* e = slab + slab_offset<OutT>(row, c);
              const bool aux_ok = aux != nullptr && grow < p.M && gcol < p.N;
              const size_t off = (size_t)grow * p.ldo + gcol;
              if constexpr (kRes) {
                // out = residual + gate * (acc + bias); aux = bf16 of out or of the branch output acc + bias (aux_branch),
                // times aux_scale of the row's sample when given
                const float2 b = *reinterpret_cast<const float2*>(cb->bias + tc);
                float2 gt = *reinterpret_cast<const float2*>((second ? cb->gate1 : cb->gate0) + tc);
                if (per_row_gate)
                  gt = (grow < p.M && gcol < p.N)
                           ? __ldg(reinterpret_cast<const float2*>(p.gate + (size_t)(grow / p.rows_per_batch) *
                                                                                 p.gate_batch_stride + gcol))
                           : make_float2(1.f, 1.f);
                float2 r = make_float2(0.f, 0.f);
                if constexpr (sizeof(OutT) == 4) {
                  if (!reduce) r = *reinterpret_cast<const float2*>(e);
                } else {
                  const uint32_t u = *reinterpret_cast<const uint32_t*>(e);
                  r = make_float2(bf16_lo(u), bf16_hi(u));
                }
                const float2 yb = make_float2(a0 + b.x, a1 + b.y);   // the branch output
                const float2 o = make_float2(fmaf(gt.x, yb.x, r.x), fmaf(gt.y, yb.y, r.y));
                if constexpr (sizeof(OutT) == 4) {
                  *reinterpret_cast<float2*>(e) = o;
                  if (gcol < p.N) {
                    st[i][h].x += o.x + o.y;
                    st[i][h].y = fmaf(o.x, o.x, fmaf(o.y, o.y, st[i][h].y));
                  }
                } else {
                  *reinterpret_cast<uint32_t*>(e) = pack_bf16x2(o.x, o.y);
                }
                if (aux_ok) {
                  float2 ax = p.aux_branch ? yb : o;
                  if (kF32Res && p.aux_scale != nullptr) {
                    const float2 sc = *reinterpret_cast<const float2*>((second ? cb->ex1 : cb->ex0) + tc);
                    ax = make_float2(ax.x * sc.x, ax.y * sc.y);
                  }
                  *reinterpret_cast<uint32_t*>(aux + off) = pack_bf16x2(ax.x, ax.y);
                }
              } else {
                float x0, x1;
                if constexpr (kLn) {   // out = [gelu](rstd * (acc - mu * u) + v), u / v of the row's sample
                  const float2 v = *reinterpret_cast<const float2*>((second ? cb->gate0 : cb->bias) + tc);
                  const float2 u = *reinterpret_cast<const float2*>((second ? cb->ex1 : cb->ex0) + tc);
                  x0 = fmaf(ln.x, a0, fmaf(ln.y, u.x, v.x));
                  x1 = fmaf(ln.x, a1, fmaf(ln.y, u.y, v.y));
                } else {
                  const float2 b = *reinterpret_cast<const float2*>(cb->bias + tc);
                  x0 = a0 + b.x;
                  x1 = a1 + b.y;
                }
                if constexpr (EPI == PXA_EPI_BIAS_GELU_AUX) {       // aux = the pre-activation the GELU backward needs
                  if (aux_ok) *reinterpret_cast<uint32_t*>(aux + off) = pack_bf16x2(x0, x1);
                }
                if constexpr (EPI == PXA_EPI_BIAS_GELU || EPI == PXA_EPI_BIAS_GELU_AUX || EPI == PXA_EPI_LN_BIAS_GELU) {
                  x0 = gelu_tanh(x0);
                  x1 = gelu_tanh(x1);
                }
                if constexpr (EPI == PXA_EPI_MUL_DGELU) {           // out = acc * gelu'(pre), pre over which out is written
                  const uint32_t w = *reinterpret_cast<const uint32_t*>(e);
                  x0 *= gelu_tanh_grad(bf16_lo(w));
                  x1 *= gelu_tanh_grad(bf16_hi(w));
                }
                *reinterpret_cast<uint32_t*>(e) = pack_bf16x2(x0, x1);
              }
            }
          }
      }
      if (t + (int)gridDim.x < num_tiles) {                          // next tile's loads: in flight during the next main loop
        const int nt_ = eff(t + gridDim.x);
        load_epi_consts<BN, kLn, kScale>(er, p, tid, tile_m0(nt_), tile_n0(nt_));
        if constexpr (kLn) if (g == 0) load_ln_stats(sr, p, tile_m0(nt_) + tid);
      }
      // the warpgroup's slabs are written: one thread hands them to the TMA engine
      fence_proxy_async_smem();
      named_bar_sync(4 + g, 128);
      if (storer) {
        const int2 xy = out_xy(m0);
#pragma unroll
        for (int s = 0; s < kSlabs; ++s) {
          const int cs = g * kSlabs + s;
          if (n0 + 32 * cs >= p.N) continue;
          if (kF32Res && reduce) tma_reduce_add_3d(&tmap_out, otile + cs * Cfg::kSlabBytes, n0 + 32 * cs, xy.x, xy.y);
          else tma_store_3d(&tmap_out, otile + cs * Cfg::kSlabBytes, n0 + 32 * cs, xy.x, xy.y);
        }
        tma_store_commit();
      }
      if constexpr (kF32Res) {
        if (p.row_stats_out != nullptr) {       // partial LayerNorm statistics of this row: part = n tile (both warpgroups' halves)
          float2* wg_stats = rowbuf;
#pragma unroll
          for (int i = 0; i < 2; ++i)
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
              for (int d = 1; d < 4; d <<= 1) {
                st[i][h].x += __shfl_xor_sync(0xffffffffu, st[i][h].x, d);
                st[i][h].y += __shfl_xor_sync(0xffffffffu, st[i][h].y, d);
              }
          const bool quad_lead = (lane & 3) == 0;
          if (g == 1 && quad_lead)
#pragma unroll
            for (int i = 0; i < 2; ++i)
#pragma unroll
              for (int h = 0; h < 2; ++h) wg_stats[64 * i + 16 * q + (lane >> 2) + 8 * h] = st[i][h];
          named_bar_sync(3, kNumEpiThreads);
          if (g == 0 && quad_lead) {
            const int nt = (tile % mn_tiles) % p.num_n_tiles;
#pragma unroll
            for (int i = 0; i < 2; ++i)
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                const int row = 64 * i + 16 * q + (lane >> 2) + 8 * h;
                if (m0 + row >= p.M) continue;
                const float2 o = wg_stats[row];
                float2* sp = reinterpret_cast<float2*>(p.row_stats_out) + (size_t)(m0 + row) * PXA_LN_STAT_PARTS;
                sp[nt] = make_float2(st[i][h].x + o.x, st[i][h].y + o.y);
                if (nt == p.num_n_tiles - 1)
                  for (int k = p.num_n_tiles; k < PXA_LN_STAT_PARTS; ++k) sp[k] = make_float2(0.f, 0.f);
              }
          }
          named_bar_sync(3, kNumEpiThreads);
        }
      }
    }
    if (storer) tma_store_wait_all<0>();
  }
}


// ------------------------------------------------------------------------------------------------- host
struct ConvGeom {
  int B, H, W, Cin, tile_w, tile_h;
  int Wp;          // virtual width of the M index (= W when W tiles; else W rounded up to 128, see GemmParams::conv_Wp)
};

template <int BN, int EPI, typename OutT, bool kConv = false, bool kMn = false, bool kTail = false, bool kScale = false>
static int launch_gemm(const PxaGemmArgs& a, cudaStream_t stream, const ConvGeom* cg = nullptr, int k_splits = 1,
                       const PxaGemmTail* tl = nullptr, const float* col_scale = nullptr) {
  CUtensorMap ta, tw;
  if constexpr (kMn) {
    // A stored [K, M] (row stride lda), W stored [K, N] (row stride ldw): 64 x 64 boxes, M / N the contiguous dimension
    uint64_t dims_a[2] = {(uint64_t)a.M, (uint64_t)a.K}, dims_w[2] = {(uint64_t)a.N, (uint64_t)a.K};
    uint64_t str_a[1] = {(uint64_t)a.lda * 2}, str_w[1] = {(uint64_t)a.ldw * 2};
    uint32_t box[2] = {64, kBK};
    int rc = make_tmap_bf16(&ta, a.a, 2, dims_a, str_a, box, CU_TENSOR_MAP_SWIZZLE_128B);
    if (rc) return rc;
    rc = make_tmap_bf16(&tw, a.w, 2, dims_w, str_w, box, CU_TENSOR_MAP_SWIZZLE_128B);
    if (rc) return rc;
  } else if constexpr (kConv) {
    // NHWC image as a 4-D tensor (c, x, y, b); one A tile = tile_h rows x tile_w pixels x 64 channels
    uint64_t dims[4] = {(uint64_t)cg->Cin, (uint64_t)cg->W, (uint64_t)cg->H, (uint64_t)cg->B};
    uint64_t str[3] = {(uint64_t)cg->Cin * 2, (uint64_t)cg->W * cg->Cin * 2, (uint64_t)cg->H * cg->W * cg->Cin * 2};
    uint32_t box[4] = {kBK, (uint32_t)cg->tile_w, (uint32_t)cg->tile_h, 1};
    int rc = make_tmap_bf16(&ta, a.a, 4, dims, str, box, CU_TENSOR_MAP_SWIZZLE_128B);
    if (rc) return rc;
  } else {
    uint64_t dims[2] = {(uint64_t)a.K, (uint64_t)a.M};
    uint64_t str[1] = {(uint64_t)a.lda * 2};
    uint32_t box[2] = {kBK, kBM};
    int rc = make_tmap_bf16(&ta, a.a, 2, dims, str, box, CU_TENSOR_MAP_SWIZZLE_128B);
    if (rc) return rc;
  }
  if constexpr (!kMn) {
    uint64_t dims[2] = {(uint64_t)a.K, (uint64_t)a.N};
    uint64_t str[1] = {(uint64_t)a.ldw * 2};
    uint32_t box[2] = {kBK, (uint32_t)BN};
    int rc = make_tmap_bf16(&tw, a.w, 2, dims, str, box, CU_TENSOR_MAP_SWIZZLE_128B);
    if (rc) return rc;
  }
  // out and the epilogue operand (same layout) as (column, x, line): x over the GEMM rows, or over the W pixels of an image line
  // for a convolution over a virtual width (its columns x >= W are then clipped by the stores)
  CUtensorMap to, tr;
  {
    constexpr uint64_t es = sizeof(OutT);
    const bool lines = kConv && cg->Wp != cg->W;
    const uint64_t X = lines ? (uint64_t)cg->W : (uint64_t)a.M;
    uint64_t dims[3] = {(uint64_t)a.N, X, lines ? (uint64_t)cg->B * cg->H : 1ull};
    uint64_t str[2] = {(uint64_t)a.ldo * es, X * a.ldo * es};
    uint32_t box[3] = {32, kBM, 1};
    const CUtensorMapDataType dt = es == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
    const CUtensorMapSwizzle swz = es == 4 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B;
    int rc = make_tmap(&to, dt, a.out, 3, dims, str, box, swz);
    if (rc) return rc;
    tr = to;
    if (a.residual != nullptr) {
      rc = make_tmap(&tr, dt, a.residual, 3, dims, str, box, swz);
      if (rc) return rc;
    }
  }
  TailMaps<kTail> tm;
  if constexpr (kTail) {
    uint64_t dims_a[2] = {(uint64_t)tl->tail_k, (uint64_t)a.M}, dims_w[2] = {(uint64_t)tl->tail_k, (uint64_t)a.N};
    uint64_t str_a[1] = {(uint64_t)tl->lda_tail * 2}, str_w[1] = {(uint64_t)tl->ldw_tail * 2};
    uint32_t box_a[2] = {kBK, kBM}, box_w[2] = {kBK, (uint32_t)BN};
    int rc = make_tmap_bf16(&tm.a, tl->tail_a, 2, dims_a, str_a, box_a, CU_TENSOR_MAP_SWIZZLE_128B);
    if (rc) return rc;
    rc = make_tmap_bf16(&tm.w, tl->tail_w, 2, dims_w, str_w, box_w, CU_TENSOR_MAP_SWIZZLE_128B);
    if (rc) return rc;
    tm.num_kb = (tl->tail_k + kBK - 1) / kBK;
  }
  using Cfg = GemmCfg<BN, OutT>;
  GemmParams p = {};
  p.bias = reinterpret_cast<const __nv_bfloat16*>(a.bias);
  p.out = a.out;
  p.out_aux = reinterpret_cast<__nv_bfloat16*>(a.out_aux_bf16);
  p.residual = a.residual;
  p.gate = a.gate;
  p.gate_batch_stride = a.gate_batch_stride;
  p.rows_per_batch = a.rows_per_batch > 0 ? a.rows_per_batch : a.M;
  p.M = a.M; p.N = a.N; p.K = a.K; p.ldo = a.ldo;
  p.num_m_tiles = (a.M + kBM - 1) / kBM;
  p.num_n_tiles = (a.N + BN - 1) / BN;
  p.k_splits = k_splits;
  p.aux_branch = a.aux_is_branch;
  fill_ln_params(p, a);
  p.conv_H = p.conv_W = p.conv_tile_w = p.conv_tile_h = p.conv_cin_blocks = 0;
  if constexpr (kConv) {
    p.conv_H = cg->H; p.conv_W = cg->W; p.conv_tile_w = cg->tile_w; p.conv_tile_h = cg->tile_h;
    p.conv_cin_blocks = cg->Cin / kBK;
  }
  p.conv_Wp = kConv ? cg->Wp : 0;
  p.col_scale = col_scale;
  auto kern = gemm_bf16_kernel<BN, EPI, OutT, kConv, kMn, kTail, kScale>;
  PXA_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmem));
  int grid = device_info().sms;
  if (a.max_ctas > 0 && a.max_ctas < grid) grid = a.max_ctas;
  const int tiles = p.num_m_tiles * p.num_n_tiles * p.k_splits;
  if (tiles < grid) grid = tiles;
  kern<<<grid, kGemmThreads, Cfg::kSmem, stream>>>(ta, tw, to, tr, p, tm);
  launch_counter()++;
  PXA_CHECK_CUDA(cudaGetLastError());
  return PXA_OK;
}

template <int BN, bool kTail = false, bool kScale = false>
static int dispatch_epi(const PxaGemmArgs& a, cudaStream_t s, const PxaGemmTail* tl = nullptr, const float* cs = nullptr) {
  switch (a.epilogue) {
    case PXA_EPI_BIAS:
      if (a.out_dtype != PXA_DTYPE_BF16) return fail(PXA_ERR_ARG, "EPI_BIAS writes bf16 only");
      return launch_gemm<BN, PXA_EPI_BIAS, __nv_bfloat16, false, false, kTail, kScale>(a, s, nullptr, 1, tl, cs);
    case PXA_EPI_BIAS_GELU:
      if (a.out_dtype != PXA_DTYPE_BF16) return fail(PXA_ERR_ARG, "EPI_BIAS_GELU writes bf16 only");
      return launch_gemm<BN, PXA_EPI_BIAS_GELU, __nv_bfloat16, false, false, kTail, kScale>(a, s, nullptr, 1, tl, cs);
    case PXA_EPI_BIAS_GELU_AUX:
      return launch_gemm<BN, PXA_EPI_BIAS_GELU_AUX, __nv_bfloat16, false, false, kTail, kScale>(a, s, nullptr, 1, tl, cs);
    case PXA_EPI_MUL_DGELU:
      if constexpr (kScale) return fail(PXA_ERR_ARG, "the column scale does not take EPI_MUL_DGELU");
      else return launch_gemm<BN, PXA_EPI_MUL_DGELU, __nv_bfloat16, false, false, kTail>(a, s, nullptr, 1, tl);
    case PXA_EPI_LN_BIAS:
    case PXA_EPI_LN_BIAS_GELU:
      if constexpr (kScale) {
        return fail(PXA_ERR_ARG, "the column scale does not take the fused LayerNorm epilogues");
      } else if constexpr (kTail) {
        return fail(PXA_ERR_ARG, "the K-tail does not take the fused LayerNorm epilogues");
      } else {
        if (a.epilogue == PXA_EPI_LN_BIAS) return launch_gemm<BN, PXA_EPI_LN_BIAS, __nv_bfloat16>(a, s);
        return launch_gemm<BN, PXA_EPI_LN_BIAS_GELU, __nv_bfloat16>(a, s);
      }
    case PXA_EPI_BIAS_RESIDUAL:
      if (a.residual == nullptr) return fail(PXA_ERR_ARG, "EPI_BIAS_RESIDUAL needs residual");
      if (a.out_dtype == PXA_DTYPE_F32)
        return launch_gemm<(BN == 256 || kTail || kScale) ? 128 : BN, PXA_EPI_BIAS_RESIDUAL, float, false, false, kTail, kScale>(
            a, s, nullptr, 1, tl, cs);
      return launch_gemm<kScale ? 128 : BN, PXA_EPI_BIAS_RESIDUAL, __nv_bfloat16, false, false, kTail, kScale>(a, s, nullptr, 1, tl, cs);
    default:
      return fail(PXA_ERR_ARG, "unknown epilogue %d", a.epilogue);
  }
}


// Weight-gradient form: out[M, N] += A^T W with A [K, M], W [K, N] (both MN-major), fp32 out accumulated in place through
// the reduce-add epilogue, K split over tiles so that the persistent grid is evenly loaded (the layer shapes give
// only 54 .. 216 output tiles against 132 SMs; each tile's K loop is thousands of blocks long).
template <int BN>
static int launch_wgrad(const PxaGemmArgs& a, cudaStream_t s) {
  const int tiles = ((a.M + kBM - 1) / kBM) * ((a.N + BN - 1) / BN);
  const int num_kb = (a.K + kBK - 1) / kBK;
  int sms = device_info().sms;
  if (a.max_ctas > 0 && a.max_ctas < sms) sms = a.max_ctas;
  int best = 1;
  double best_eff = 0.0;
  for (int ks = 1; ks <= 16 && num_kb / ks >= 8; ++ks) {
    const int t = tiles * ks;
    const double eff = (double)t / (double)(((t + sms - 1) / sms) * sms);
    if (eff > best_eff + 1e-9) { best_eff = eff; best = ks; }
  }
  if (a.k_splits > 0) best = a.k_splits;
  if (best > num_kb) best = num_kb;
  return launch_gemm<BN, PXA_EPI_BIAS_RESIDUAL, float, false, true>(a, s, nullptr, best);
}

template <int BN>
static int dispatch_conv(const PxaGemmArgs& a, cudaStream_t s, const ConvGeom& cg) {
  if (a.epilogue == PXA_EPI_BIAS_RESIDUAL) return launch_gemm<BN, PXA_EPI_BIAS_RESIDUAL, __nv_bfloat16, true>(a, s, &cg);
  return launch_gemm<BN, PXA_EPI_BIAS, __nv_bfloat16, true>(a, s, &cg);
}

}  // namespace pxa

extern "C" int pxa_conv3x3_nhwc_bf16(const PxaConv3x3Args* args, void* stream) {
  using namespace pxa;
  if (!args) return fail(PXA_ERR_ARG, "null args");
  const PxaConv3x3Args& c = *args;
  if (!c.x || !c.w || !c.out) return fail(PXA_ERR_ARG, "null x / w / out");
  if (c.B <= 0 || c.H <= 0 || c.W <= 0 || c.Cin <= 0 || c.Cout <= 0) return fail(PXA_ERR_ARG, "bad shape");
  if (c.Cin % 64) return fail(PXA_ERR_ARG, "Cin must be a multiple of 64 (got %d)", c.Cin);
  if (c.Cout % 8) return fail(PXA_ERR_ARG, "Cout must be a multiple of 8 (got %d)", c.Cout);
  ConvGeom cg;
  cg.B = c.B; cg.H = c.H; cg.W = c.W; cg.Cin = c.Cin;
  // M tile = 128 consecutive pixels = ONE TMA box: tile_h full lines when W is a power of two <= 128 (and H a multiple of tile_h),
  // 128 pixels of one line when W is a multiple of 128.  Every other geometry (e.g. the 1024-MS aspect buckets: latent 104 x 152 ->
  // 832 x 1216) runs over a virtual width Wp = W rounded up to 128, one line segment per tile: columns >= W are zero fill going in
  // (the right-hand padding of the convolution, exactly) and are dropped going out; the tail tile of a line is partly idle (W / Wp of
  // the MMA work is useful: 0.81 at W = 104, 0.95 at W = 1216).
  cg.tile_w = c.W < 128 ? c.W : 128;
  cg.tile_h = (128 % cg.tile_w) ? 1 : 128 / cg.tile_w;
  cg.Wp = c.W;
  if ((128 % cg.tile_w) || c.W % cg.tile_w || c.H % cg.tile_h) {
    cg.tile_w = 128; cg.tile_h = 1;
    cg.Wp = (c.W + 127) / 128 * 128;
  }
  if ((reinterpret_cast<uintptr_t>(c.x) | reinterpret_cast<uintptr_t>(c.w) | reinterpret_cast<uintptr_t>(c.out) |
       reinterpret_cast<uintptr_t>(c.bias) | reinterpret_cast<uintptr_t>(c.residual)) & 15)
    return fail(PXA_ERR_ALIGN, "pointers must be 16-byte aligned");
  PXA_REQUIRE_SM90();
  PxaGemmArgs a = {};
  a.a = c.x; a.w = c.w; a.bias = c.bias; a.out = c.out; a.residual = c.residual;
  if ((long long)c.B * c.H * cg.Wp >= (1ll << 31)) return fail(PXA_ERR_ARG, "B x H x W too large");
  a.M = c.B * c.H * cg.Wp; a.N = c.Cout; a.K = 9 * c.Cin;
  a.lda = c.Cin; a.ldw = 9 * c.Cin; a.ldo = c.Cout;
  a.rows_per_batch = a.M;
  a.epilogue = c.residual ? PXA_EPI_BIAS_RESIDUAL : PXA_EPI_BIAS;
  a.out_dtype = PXA_DTYPE_BF16;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  if (c.Cout % 256 == 0) return dispatch_conv<256>(a, s, cg);
  if (c.Cout % 192 == 0) return dispatch_conv<192>(a, s, cg);
  return dispatch_conv<128>(a, s, cg);
}

namespace pxa {
static int gemm_impl(const PxaGemmArgs* args, const PxaGemmTail* tl, const float* col_scale, void* stream) {
  if (!args) return fail(PXA_ERR_ARG, "null args");
  const PxaGemmArgs& a = *args;
  if (!a.a || !a.w || !a.out) return fail(PXA_ERR_ARG, "null a / w / out");
  if (a.M <= 0 || a.N <= 0 || a.K <= 0) return fail(PXA_ERR_ARG, "bad shape M=%d N=%d K=%d", a.M, a.N, a.K);
  if ((a.N & 7) || (!a.operands_mn_major && (a.K & 7)) || (a.operands_mn_major && (a.M & 7)) || (a.lda & 7) ||
      (a.ldw & 7) || (a.ldo & 7))
    return fail(PXA_ERR_ALIGN, "N, the contiguous operand dimension (K; M for operands_mn_major), lda, ldw, ldo must be "
                               "multiples of 8 (M=%d N=%d K=%d lda=%d ldw=%d ldo=%d)", a.M, a.N, a.K, a.lda, a.ldw, a.ldo);
  if (a.k_splits < 0 || (a.k_splits > 1 && !a.operands_mn_major)) return fail(PXA_ERR_ARG, "k_splits needs operands_mn_major");
  if ((reinterpret_cast<uintptr_t>(a.out) | reinterpret_cast<uintptr_t>(a.bias) |
       reinterpret_cast<uintptr_t>(a.residual) | reinterpret_cast<uintptr_t>(a.gate) |
       reinterpret_cast<uintptr_t>(a.out_aux_bf16)) & 15)
    return fail(PXA_ERR_ALIGN, "out / bias / residual / gate / aux must be 16-byte aligned");
  if (a.gate && (a.gate_batch_stride & 3)) return fail(PXA_ERR_ALIGN, "gate_batch_stride must be a multiple of 4");
  if (tl) {
    if (!tl->tail_a || !tl->tail_w) return fail(PXA_ERR_ARG, "null tail_a / tail_w");
    if (tl->tail_k <= 0 || (tl->tail_k & 7)) return fail(PXA_ERR_ARG, "tail_k must be a positive multiple of 8 (got %d)", tl->tail_k);
    if (a.operands_mn_major) return fail(PXA_ERR_ARG, "the K-tail does not take operands_mn_major");
    if (a.epilogue == PXA_EPI_LN_BIAS || a.epilogue == PXA_EPI_LN_BIAS_GELU)
      return fail(PXA_ERR_ARG, "the K-tail does not take the fused LayerNorm epilogues");
    if ((reinterpret_cast<uintptr_t>(tl->tail_a) | reinterpret_cast<uintptr_t>(tl->tail_w)) & 15)
      return fail(PXA_ERR_ALIGN, "tail_a / tail_w must be 16-byte aligned");
    if ((tl->lda_tail & 7) || (tl->ldw_tail & 7))
      return fail(PXA_ERR_ALIGN, "lda_tail / ldw_tail must be multiples of 8 (got %d, %d)", tl->lda_tail, tl->ldw_tail);
    if (tl->lda_tail < tl->tail_k || tl->ldw_tail < tl->tail_k) return fail(PXA_ERR_ARG, "lda_tail / ldw_tail < tail_k");
  }
  if (col_scale) {
    if (a.operands_mn_major) return fail(PXA_ERR_ARG, "the column scale does not take operands_mn_major");
    if (a.epilogue != PXA_EPI_BIAS && a.epilogue != PXA_EPI_BIAS_GELU && a.epilogue != PXA_EPI_BIAS_GELU_AUX &&
        a.epilogue != PXA_EPI_BIAS_RESIDUAL)
      return fail(PXA_ERR_ARG, "the column scale takes EPI_BIAS, EPI_BIAS_GELU, EPI_BIAS_GELU_AUX and EPI_BIAS_RESIDUAL only");
    if (a.aux_scale || a.row_stats_out) return fail(PXA_ERR_ARG, "the column scale does not take aux_scale / row_stats_out");
    if (reinterpret_cast<uintptr_t>(col_scale) & 3) return fail(PXA_ERR_ALIGN, "col_scale must be 4-byte aligned");
  }
  PXA_REQUIRE_SM90();
  int bn = a.block_n;
  if (bn == 0) bn = (a.N % 192 == 0) ? 192 : ((a.N % 256 == 0) ? 256 : (a.N >= 192 ? 192 : 128));
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  if (a.operands_mn_major) {
    if (a.epilogue != PXA_EPI_BIAS_RESIDUAL || a.out_dtype != PXA_DTYPE_F32 || a.residual != a.out || a.bias || a.gate ||
        a.out_aux_bf16)
      return fail(PXA_ERR_ARG, "operands_mn_major is the weight-gradient form: EPI_BIAS_RESIDUAL, fp32 out, residual == out, "
                               "no bias / gate / aux");
    switch (bn) {
      case 128: return launch_wgrad<128>(a, s);
      case 192: return launch_wgrad<128>(a, s);      // MN-major W is staged in 64-column atoms per warpgroup: 96 does not tile
      case 256: return launch_wgrad<128>(a, s);      // fp32 output tiles run at 128 columns (GemmCfg)
      default: return fail(PXA_ERR_ARG, "block_n must be 0, 128, 192 or 256 (got %d)", bn);
    }
  }
  if (a.epilogue == PXA_EPI_BIAS_RESIDUAL && a.residual == nullptr) return fail(PXA_ERR_ARG, "EPI_BIAS_RESIDUAL needs residual");
  if (a.epilogue != PXA_EPI_BIAS_RESIDUAL && a.out_dtype != PXA_DTYPE_BF16)
    return fail(PXA_ERR_ARG, "EPI_BIAS / EPI_BIAS_GELU write bf16 only");
  if (a.epilogue == PXA_EPI_BIAS_GELU_AUX && a.out_aux_bf16 == nullptr) return fail(PXA_ERR_ARG, "EPI_BIAS_GELU_AUX needs out_aux_bf16");
  if (a.epilogue == PXA_EPI_MUL_DGELU && (a.residual == nullptr || a.bias != nullptr))
    return fail(PXA_ERR_ARG, "EPI_MUL_DGELU needs the pre-activation in `residual` and no bias");
  // fused LayerNorm-modulate: consumer epilogues and the producer by-products of the fp32 residual epilogue
  const bool ln_epi = a.epilogue == PXA_EPI_LN_BIAS || a.epilogue == PXA_EPI_LN_BIAS_GELU;
  const int rpb = a.rows_per_batch > 0 ? a.rows_per_batch : a.M;
  if (ln_epi) {
    if (!a.ln_stats || !a.ln_u || !a.ln_v || a.ln_dim <= 0 || a.bias)
      return fail(PXA_ERR_ARG, "EPI_LN_*: ln_stats / ln_u / ln_v / ln_dim required and bias must be NULL (it is part of ln_v)");
    if ((reinterpret_cast<uintptr_t>(a.ln_stats) | reinterpret_cast<uintptr_t>(a.ln_u) | reinterpret_cast<uintptr_t>(a.ln_v)) & 15)
      return fail(PXA_ERR_ALIGN, "ln_stats / ln_u / ln_v must be 16-byte aligned");
  }
  if (a.aux_scale || a.row_stats_out) {
    if (a.epilogue != PXA_EPI_BIAS_RESIDUAL || a.out_dtype != PXA_DTYPE_F32)
      return fail(PXA_ERR_ARG, "aux_scale / row_stats_out belong to the fp32 residual epilogue");
    if (a.aux_scale && !a.out_aux_bf16) return fail(PXA_ERR_ARG, "aux_scale needs out_aux_bf16");
    if ((reinterpret_cast<uintptr_t>(a.aux_scale) | reinterpret_cast<uintptr_t>(a.row_stats_out)) & 15)
      return fail(PXA_ERR_ALIGN, "aux_scale / row_stats_out must be 16-byte aligned");
  }
  if ((ln_epi || a.aux_scale) && rpb < kBM && a.M > rpb)
    return fail(PXA_ERR_ARG, "the fused LayerNorm-modulate needs rows_per_batch >= %d (a tile may span two samples at most)", kBM);
  if (bn == 256 && a.out_dtype == PXA_DTYPE_F32) bn = 128;   // fp32 output tiles run at 128 columns (GemmCfg)
  // the tail instantiations spill at BN 256 and, with fp32 output, at BN 192: they run at 192 and 128 instead
  if (tl && bn == 256) bn = 192;
  if (tl && bn == 192 && a.out_dtype == PXA_DTYPE_F32) bn = 128;
  // the column-scaled instantiations spill at BN 256 and, with the residual epilogue, at BN 192: they run at 192 and 128
  if (col_scale && bn == 256) bn = 192;
  if (col_scale && a.epilogue == PXA_EPI_BIAS_RESIDUAL) bn = 128;
  if (a.row_stats_out && (a.N + bn - 1) / bn > PXA_LN_STAT_PARTS)
    return fail(PXA_ERR_ARG, "row_stats_out: N / block_n = %d column tiles exceed PXA_LN_STAT_PARTS", (a.N + bn - 1) / bn);
  if (tl && col_scale) {
    switch (bn) {
      case 128: return dispatch_epi<128, true, true>(a, s, tl, col_scale);
      case 192: return dispatch_epi<192, true, true>(a, s, tl, col_scale);
      default: return fail(PXA_ERR_ARG, "block_n must be 0, 128, 192 or 256 (got %d)", bn);
    }
  }
  if (tl) {
    switch (bn) {
      case 128: return dispatch_epi<128, true>(a, s, tl);
      case 192: return dispatch_epi<192, true>(a, s, tl);
      default: return fail(PXA_ERR_ARG, "block_n must be 0, 128, 192 or 256 (got %d)", bn);
    }
  }
  if (col_scale) {
    switch (bn) {
      case 128: return dispatch_epi<128, false, true>(a, s, nullptr, col_scale);
      case 192: return dispatch_epi<192, false, true>(a, s, nullptr, col_scale);
      default: return fail(PXA_ERR_ARG, "block_n must be 0, 128, 192 or 256 (got %d)", bn);
    }
  }
  switch (bn) {
    case 128: return dispatch_epi<128>(a, s);
    case 192: return dispatch_epi<192>(a, s);
    case 256: return dispatch_epi<256>(a, s);
    default: return fail(PXA_ERR_ARG, "block_n must be 0, 128, 192 or 256 (got %d)", bn);
  }
}
}  // namespace pxa

extern "C" int pxa_gemm_bf16(const PxaGemmArgs* args, void* stream) { return pxa::gemm_impl(args, nullptr, nullptr, stream); }

extern "C" int pxa_gemm_lora_bf16(const PxaGemmArgs* args, const PxaGemmTail* tail, void* stream) {
  if (!tail) return pxa::fail(PXA_ERR_ARG, "null tail");
  return pxa::gemm_impl(args, tail, nullptr, stream);
}

extern "C" int pxa_gemm_dora_bf16(const PxaGemmArgs* args, const PxaGemmTail* tail, const float* col_scale, void* stream) {
  if (!col_scale) return pxa::fail(PXA_ERR_ARG, "null col_scale");
  return pxa::gemm_impl(args, tail, col_scale, stream);
}
