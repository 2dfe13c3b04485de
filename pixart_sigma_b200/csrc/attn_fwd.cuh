// Flash-attention forward kernels on wgmma tensor cores (sm_90a): flash_fwd_d72_kernel behind pxa_flash_attn_d72_bf16
// (head_dim 72, var-len keys), and what it shares with t5_attn_fwd_kernel (t5_attn_sm90.cu): parameters and tensor maps.
//
// flash_fwd_d72_kernel.  One CTA = 128 query rows of one (sample, head), 384 threads, one CTA per SM:
//   - warpgroup 0 is the producer.  It gives up most of its registers (setmaxnreg) and one thread issues every TMA load: Q once,
//     then K and V blocks of 128 keys into rings of kFaStages stages each.  K and V have their own full barriers, so Q K^T of a
//     block can start before its V has landed, and the consumers hand stages back through per-stage empty barriers.  The main
//     loop has no CTA-wide barrier.
//   - warpgroups 1 and 2 are the consumers, 64 query rows each (240 registers per thread).  Per 128-key block: S = Q K^T by
//     wgmma with both operands in shared memory (a 64 x 128 fp32 tile in registers), online softmax on the accumulator
//     fragments (a row lives in the four lanes of a quad), P packed to bf16 in registers -- the accumulator layout of S is the
//     A-fragment layout of the next wgmma -- and O += P V with V consumed MN-major from its natural [key, d] layout.
//   - Within a warpgroup the two products of neighbouring blocks overlap: iteration n issues S(n) = Q K(n)^T, rescales O,
//     issues O += P(n-1) V(n-1), waits for S(n) only and runs its softmax while P V is still on the tensor cores, then waits
//     for P V and packs P(n).  All P fragments are packed before the first wgmma of a P V chain, so ptxas never has to
//     serialise the chain on register writes.
//   - Between the warpgroups, two named barriers make their wgmma issue slots alternate, so that one warpgroup's products run
//     while the other computes its softmax.
//   - Each logit becomes one FFMA (s * scale_log2 - m * scale_log2) and one ex2; the key < kv_len mask is applied in the last,
//     partial block only.
//
// head_dim 72 is not a multiple of the 64-element swizzle atom nor of the MMA K = 16: each Q / K / V tile is staged as a "main"
// part (d 0..63, 128B swizzle, 128 B rows) plus a "tail" part (d 64..79, 32B swizzle, 32 B rows) whose d 72..79 are zero-filled
// by TMA out-of-bounds handling (the tensor maps' innermost extent is 72).  Q K^T = 4 main K-steps + 1 tail K-step of
// m64n128k16; P V = m64n64k16 on the main part + m64n16k16 on the tail part per 16 keys.  The tail is kept narrow on purpose:
// staged as a 64-column 128B-swizzled part instead (8 real columns and 56 zero-filled ones per 128 B row), the K / V loads
// bounded this kernel at about 335 TFLOP/s on c3 self-attention (H100 80GB HBM3, 700 W), with the softmax, the P V product
// and the warpgroup ping-pong each making no measurable difference.
#pragma once
#include <math.h>

#include <type_traits>

#include "host_common.cuh"
#include "ptx.cuh"

namespace pxa {

struct FaParams {
  __nv_bfloat16* out;
  float* lse;           // optional [B, H, Nq]: log2-domain log-sum-exp of the scaled scores (training: consumed by the backward)
  const int* kv_len;
  const int* kv_off;
  const float* bias;      // T5: dense [H, Nq, Nk] or NULL
  const float* rel_bias;  // T5: Toeplitz [H, 2 Nk - 1] or NULL
  const float* key_bias;  // T5: [B, Nk] or NULL
  int B, H, Nq, Nk, ldo;
  float scale_log2;       // >= 0 for the head_dim-72 kernel
  int reverse_batch;    // CTAs take the samples from the last to the first (L2 reuse of the freshly written qkv rows)
};

// ================================================================================================ head_dim 72
constexpr int kFaThreads = 384;                 // producer warpgroup + two consumer warpgroups
constexpr int kFaTileQ = 128;
constexpr int kFaBlk = 128;                     // keys per block
constexpr int kFaStages = 3;                    // K and V ring depth
constexpr int kFaPart = 128 * 128;              // the main part of a 128-row Q tile or K / V block: d 0..63, 128 rows x 128 B
constexpr int kFaTail = 128 * 32;               // its tail part: d 64..79, 128 rows x 32 B
constexpr int kFaTile = kFaPart + kFaTail;
constexpr int kFaOffQ = 0;
constexpr int kFaOffK = kFaOffQ + kFaTile;
constexpr int kFaOffV = kFaOffK + kFaStages * kFaTile;
constexpr int kFaOffBars = kFaOffV + kFaStages * kFaTile;
constexpr int kFaSmem = kFaOffBars + (1 + 4 * kFaStages) * 8 + 1024;   // + alignment slack
constexpr int kFaConsumerWarps = 8;
constexpr uint32_t kFaBarWg0 = 1;               // named barriers 1 / 2: "consumer warpgroup 0 / 1 may issue its products"

// Tensor maps of the main ([0]: d 0..63, 128B swizzle) and tail ([1]: d 64..79, 32B swizzle) parts of Q, K and V
struct FaMaps {
  CUtensorMap q[2], k[2], v[2];
};

template <bool kSplitP>
__global__ void __launch_bounds__(kFaThreads, 1)
flash_fwd_d72_kernel(const __grid_constant__ FaMaps tm, const FaParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* q_full = reinterpret_cast<uint64_t*>(smem + kFaOffBars);
  uint64_t* k_full = q_full + 1;                // [kFaStages] each: TMA -> consumers
  uint64_t* v_full = k_full + kFaStages;
  uint64_t* k_empty = v_full + kFaStages;       // consumers -> TMA, one arrival per consumer warp
  uint64_t* v_empty = k_empty + kFaStages;

  const int warp = warp_idx_sync();
  const int lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * kFaTileQ;
  const int h = blockIdx.y;
  const int b = p.reverse_batch ? p.B - 1 - (int)blockIdx.z : (int)blockIdx.z;
  int kv_len = p.kv_len ? p.kv_len[b] : p.Nk;
  if (kv_len > p.Nk) kv_len = p.Nk;
  const long long kv0 = p.kv_off ? p.kv_off[b] : (long long)b * p.Nk;
  const int nblk = kv_len > 0 ? (kv_len + kFaBlk - 1) / kFaBlk : 0;

  if (threadIdx.x == 0) {
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      prefetch_tmap(&tm.q[c]);
      prefetch_tmap(&tm.k[c]);
      prefetch_tmap(&tm.v[c]);
    }
    mbar_init(q_full, 1);
    for (int s = 0; s < kFaStages; ++s) {
      mbar_init(&k_full[s], 1);
      mbar_init(&v_full[s], 1);
      mbar_init(&k_empty[s], kFaConsumerWarps);
      mbar_init(&v_empty[s], kFaConsumerWarps);
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp < 4) {
    // ================================================================ TMA producer
    reg_dealloc<24>();
    if (warp == 0 && elect_one() && nblk > 0) {
      mbar_arrive_expect_tx(q_full, kFaTile);
#pragma unroll
      for (int c = 0; c < 2; ++c) tma_load_3d(smem + kFaOffQ + c * kFaPart, &tm.q[c], q_full, 64 * c, h, b * p.Nq + q0, kEvictFirst);
      auto load = [&](const CUtensorMap* map, uint64_t* full, uint64_t* empty, int off, int n) {
        const int s = n % kFaStages;
        mbar_wait(&empty[s], ((n / kFaStages) & 1) ^ 1);
        uint8_t* dst = smem + off + s * kFaTile;
        const int krow = (int)(kv0 + (long long)n * kFaBlk);
        mbar_arrive_expect_tx(&full[s], kFaTile);
#pragma unroll
        for (int c = 0; c < 2; ++c) tma_load_3d(dst + c * kFaPart, &map[c], &full[s], 64 * c, h, krow, kEvictLast);
      };
      // the consumers take K(n + 1) before V(n)
      load(tm.k, k_full, k_empty, kFaOffK, 0);
      for (int n = 0; n < nblk; ++n) {
        if (n + 1 < nblk) load(tm.k, k_full, k_empty, kFaOffK, n + 1);
        load(tm.v, v_full, v_empty, kFaOffV, n);
      }
    }
    return;
  }

  // ================================================================ consumers
  reg_alloc<240>();
  const int wg = (warp >> 2) - 1;
  // accumulator fragment rows of this thread: row_h = 64 wg + 16 (warp % 4) + lane / 4 + 8 h
  const int row_in_tile = 64 * wg + 16 * (warp & 3) + (lane >> 2);
  const int cq = 2 * (lane & 3);
  float o[32], ot[8];                                               // O columns 0..63 and 64..79
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) ot[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};

  if (nblk > 0) {
    const uint32_t sbase = smem_u32(smem);
    const float sl2 = p.scale_log2;
    const bool partial = (kv_len % kFaBlk) != 0;
    const uint32_t bar_mine = kFaBarWg0 + wg, bar_other = kFaBarWg0 + (wg ^ 1);
    float s[64];
    float corr[2];
    uint32_t phi[8][4];                                             // P (bf16) as the A fragments of the 8 K-steps of P V
    [[maybe_unused]] uint32_t plo[kSplitP ? 8 : 1][4];              // kSplitP: the rounding remainder P - bf16(P), also bf16

    auto issue_qk = [&](int n) {
      const uint32_t kst = sbase + kFaOffK + (n % kFaStages) * kFaTile;
      wgmma_fence();
      const uint64_t qd = make_smem_desc(sbase + kFaOffQ + wg * 8192, 16, 1024, kLayoutSW128);
      const uint64_t kd = make_smem_desc(kst, 16, 1024, kLayoutSW128);
#pragma unroll
      for (int k = 0; k < 4; ++k) wgmma_ss<kFaBlk, 0, 0>(s, qd + 2 * k, kd + 2 * k, k != 0 ? 1u : 0u);
      // tail K-step: 32 B rows, 8-row groups 256 B apart
      wgmma_ss<kFaBlk, 0, 0>(s, make_smem_desc(sbase + kFaOffQ + kFaPart + wg * 2048, 16, 256, kLayoutSW32),
                             make_smem_desc(kst + kFaPart, 16, 256, kLayoutSW32), 1u);
      wgmma_commit();
    };
    // O += P V with V MN-major: N = 64 from the main part (16 keys = 2048 B per K-step) and N = 16 from the tail part
    // (16 keys = 512 B per K-step)
    auto issue_pv = [&](int n) {
      const uint32_t vst = sbase + kFaOffV + (n % kFaStages) * kFaTile;
      const uint64_t vd = make_smem_desc(vst, kFaPart, 1024, kLayoutSW128);
      const uint64_t vdt = make_smem_desc(vst + kFaPart, kFaTail, 256, kLayoutSW32);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < kFaBlk / 16; ++kk) {
        wgmma_rs<64, 1>(o, phi[kk], vd + (uint64_t)(kk * (2048 >> 4)), 1u);
        wgmma_rs<16, 1>(ot, phi[kk], vdt + (uint64_t)(kk * (512 >> 4)), 1u);
        if constexpr (kSplitP) {
          wgmma_rs<64, 1>(o, plo[kk], vd + (uint64_t)(kk * (2048 >> 4)), 1u);
          wgmma_rs<16, 1>(ot, plo[kk], vdt + (uint64_t)(kk * (512 >> 4)), 1u);
        }
      }
      wgmma_commit();
    };
    // online softmax of block n in the log2 domain: S -> unnormalised P (fp32, in place), corr = rescale factor of O and l
    auto softmax = [&](auto masked, int n) {
      constexpr bool kMasked = decltype(masked)::value;
      const int rem = kv_len - n * kFaBlk;                          // valid keys in this block; >= 1
      float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
      for (int j = 0; j < kFaBlk / 8; ++j)
#pragma unroll
        for (int hh = 0; hh < 2; ++hh)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            float& x = s[4 * j + 2 * hh + e];
            if constexpr (kMasked) x = 8 * j + cq + e < rem ? x : -INFINITY;
            mx[hh] = fmaxf(mx[hh], x);
          }
      float neg_m[2];
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 1));
        mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 2));
        // every block has a valid key in every row, so the running max is finite from block 0 on; scale_log2 >= 0 makes
        // max(s) * scale_log2 the max of the scaled logits
        const float m_new = fmaxf(m_run[hh], mx[hh] * sl2);
        corr[hh] = fast_exp2(m_run[hh] - m_new);                    // block 0: exp2(-inf) = 0
        m_run[hh] = m_new;
        neg_m[hh] = -m_new;
      }
      float sum[2] = {0.f, 0.f};
#pragma unroll
      for (int j = 0; j < kFaBlk / 8; ++j)
#pragma unroll
        for (int hh = 0; hh < 2; ++hh)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            float& x = s[4 * j + 2 * hh + e];
            float pe = fast_exp2(fmaf(x, sl2, neg_m[hh]));
            if constexpr (kMasked) pe = 8 * j + cq + e < rem ? pe : 0.f;
            x = pe;
            sum[hh] += pe;
          }
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) l_run[hh] = fmaf(l_run[hh], corr[hh], sum[hh]);
    };
    auto softmax_block = [&](int n) {
      if (partial && n == nblk - 1) softmax(std::true_type{}, n);
      else softmax(std::false_type{}, n);
    };
    auto pack_p = [&]() {
#pragma unroll
      for (int kk = 0; kk < kFaBlk / 16; ++kk)
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          phi[kk][i] = pack_bf16x2(s[8 * kk + 2 * i], s[8 * kk + 2 * i + 1]);
          if constexpr (kSplitP)
            plo[kk][i] = pack_bf16x2(s[8 * kk + 2 * i] - bf16_lo(phi[kk][i]), s[8 * kk + 2 * i + 1] - bf16_hi(phi[kk][i]));
        }
    };
    auto rescale_o = [&]() {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        o[4 * j] *= corr[0]; o[4 * j + 1] *= corr[0];
        o[4 * j + 2] *= corr[1]; o[4 * j + 3] *= corr[1];
      }
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        ot[4 * j] *= corr[0]; ot[4 * j + 1] *= corr[0];
        ot[4 * j + 2] *= corr[1]; ot[4 * j + 3] *= corr[1];
      }
    };

    // Issue slots alternate between the warpgroups: warpgroup 0 goes first, and each slot ends by opening the other's
    // barrier.  Both warpgroups have nblk + 1 slots; the last slot of warpgroup 1 opens nothing, which balances the arrival
    // that starts warpgroup 0.
    if (wg == 1) named_bar_arrive(kFaBarWg0, 256);
    mbar_wait(q_full, 0);
    mbar_wait(&k_full[0], 0);
    named_bar_sync(bar_mine, 256);
    issue_qk(0);
    named_bar_arrive(bar_other, 256);
    wgmma_wait<0>();
    wgmma_fence_regs(s);
    if (lane == 0) mbar_arrive(&k_empty[0]);
    softmax_block(0);
    pack_p();
    for (int n = 1; n < nblk; ++n) {
      const int st = n % kFaStages, pst = (n - 1) % kFaStages;
      mbar_wait(&k_full[st], (n / kFaStages) & 1);
      named_bar_sync(bar_mine, 256);
      issue_qk(n);
      rescale_o();
      mbar_wait(&v_full[pst], ((n - 1) / kFaStages) & 1);
      issue_pv(n - 1);
      named_bar_arrive(bar_other, 256);
      wgmma_wait<1>();                                              // S(n) is done; P(n-1) V(n-1) may still run
      wgmma_fence_regs(s);
      if (lane == 0) mbar_arrive(&k_empty[st]);
      softmax_block(n);
      wgmma_wait<0>();
      wgmma_fence_regs(o);
      wgmma_fence_regs(ot);
      if (lane == 0) mbar_arrive(&v_empty[pst]);
      pack_p();
    }
    rescale_o();
    mbar_wait(&v_full[(nblk - 1) % kFaStages], ((nblk - 1) / kFaStages) & 1);
    named_bar_sync(bar_mine, 256);
    issue_pv(nblk - 1);
    if (wg == 0) named_bar_arrive(bar_other, 256);
    wgmma_wait<0>();
    wgmma_fence_regs(o);
    wgmma_fence_regs(ot);
  }

  // ---- epilogue: O / row_sum -> bf16 -> out[(b*Nq + qrow), h*72 ..]; rows without keys produce zeros and lse 0
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    float l = l_run[hh];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const int qrow = q0 + row_in_tile + 8 * hh;
    if (qrow >= p.Nq) continue;
    const float inv = l > 0.f ? 1.0f / l : 0.f;
    if (p.lse != nullptr && (lane & 3) == 0)                        // P = exp2(S * scale_log2 - lse) in the backward
      p.lse[((size_t)b * p.H + h) * p.Nq + qrow] = l > 0.f ? m_run[hh] + log2f(l) : 0.f;
    __nv_bfloat16* dst = p.out + (size_t)(b * p.Nq + qrow) * p.ldo + h * 72 + cq;
#pragma unroll
    for (int j = 0; j < 8; ++j)
      *reinterpret_cast<uint32_t*>(dst + 8 * j) = pack_bf16x2(o[4 * j + 2 * hh] * inv, o[4 * j + 2 * hh + 1] * inv);
    *reinterpret_cast<uint32_t*>(dst + 64) = pack_bf16x2(ot[2 * hh] * inv, ot[2 * hh + 1] * inv);
  }
}

// Tensor map over q / k / v rows as (d, head, row): boxes of `box_cols` columns x `box_rows` rows; columns >= dh read as zero.
inline int make_fa_map(CUtensorMap* map, const void* base, int dh, int H, long long rows, long long s_row, long long s_head, int box_cols,
                       int box_rows, CUtensorMapSwizzle swz) {
  uint64_t dims[3] = {(uint64_t)dh, (uint64_t)H, (uint64_t)rows};
  uint64_t str[2] = {(uint64_t)s_head * 2, (uint64_t)s_row * 2};
  uint32_t box[3] = {(uint32_t)box_cols, 1, (uint32_t)box_rows};
  return make_tmap_bf16(map, base, 3, dims, str, box, swz);
}

}  // namespace pxa
