// pxa_t5_attn_d64_bf16: self-attention of the T5 caption encoder (head_dim 64, additive relative-position bias and key padding
// bias) on wgmma tensor cores (sm_90a).  The bias of a (query, key) pair is read where the logit is
// produced: the Toeplitz form (2 L - 1 floats per head) and the key bias stay cache-resident.
#include "attn_fwd.cuh"

namespace pxa {

// 128 query rows per CTA, two warpgroups, two CTAs per SM; 64-key blocks through a two-stage TMA ring fed by thread 0, with a
// __syncthreads per block handing the consumed stage back.  Per block and warpgroup: S = Q K^T by wgmma from shared memory,
// online softmax with the bias added where each logit is produced, P packed to bf16 A fragments, O += P V with V MN-major.
constexpr int kT5Threads = 256;
constexpr int kT5TileQ = 128;
constexpr int kT5Blk = 64;                      // keys per block
constexpr int kT5QBytes = kT5TileQ * 128;       // the 128 x 64 Q tile
constexpr int kT5KvBytes = kT5Blk * 128;        // a 64 x 64 K or V block
constexpr int kT5StageBytes = 2 * kT5KvBytes;   // stage s: K, then V
constexpr int kT5OffKV = kT5QBytes;
constexpr int kT5OffBars = kT5OffKV + 2 * kT5StageBytes;
constexpr int kT5Smem = kT5OffBars + 64 + 1024;  // + alignment slack

__global__ void __launch_bounds__(kT5Threads, 2)
t5_attn_fwd_kernel(const __grid_constant__ CUtensorMap tm_q, const __grid_constant__ CUtensorMap tm_k,
                   const __grid_constant__ CUtensorMap tm_v, const FaParams p) {
  constexpr float kLog2e = 1.4426950408889634f;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* q_full = reinterpret_cast<uint64_t*>(smem + kT5OffBars);
  uint64_t* kv_full = q_full + 1;           // [2]

  const int warp = warp_idx_sync();
  const int lane = threadIdx.x & 31;
  const int wg = warp >> 2;
  const int q0 = blockIdx.x * kT5TileQ;
  const int h = blockIdx.y;
  const int b = blockIdx.z;
  const int kv_len = p.Nk;
  const long long kv0 = (long long)b * p.Nk;
  const int nblk = (kv_len + kT5Blk - 1) / kT5Blk;

  if (threadIdx.x == 0) {
    prefetch_tmap(&tm_q);
    prefetch_tmap(&tm_k);
    prefetch_tmap(&tm_v);
    mbar_init(q_full, 1);
    mbar_init(&kv_full[0], 1);
    mbar_init(&kv_full[1], 1);
    fence_mbar_init();
  }
  __syncthreads();

  auto load_kv = [&](int n) {
    const int s = n & 1;
    uint8_t* st = smem + kT5OffKV + s * kT5StageBytes;
    const int krow = (int)(kv0 + (long long)n * kT5Blk);
    mbar_arrive_expect_tx(&kv_full[s], kT5StageBytes);
    tma_load_3d(st, &tm_k, &kv_full[s], 0, h, krow, kEvictLast);
    tma_load_3d(st + kT5KvBytes, &tm_v, &kv_full[s], 0, h, krow, kEvictLast);
  };
  if (threadIdx.x == 0 && nblk > 0) {
    mbar_arrive_expect_tx(q_full, kT5QBytes);
    tma_load_3d(smem, &tm_q, q_full, 0, h, b * p.Nq + q0, kEvictFirst);
    load_kv(0);
  }

  // accumulator fragment rows of this thread: row_h = 64 wg + 16 (warp % 4) + lane / 4 + 8 h
  const int row_in_tile = 64 * wg + 16 * (warp & 3) + (lane >> 2);
  const int cq = 2 * (lane & 3);
  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};

  const float* brow[2];
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int qi = min(q0 + row_in_tile + 8 * hh, p.Nq - 1);       // rows >= Nq are computed on a clamped bias row, never stored
    brow[hh] = p.rel_bias ? p.rel_bias + (size_t)h * (2 * p.Nk - 1) + (p.Nk - 1 - qi) : p.bias + ((size_t)h * p.Nq + qi) * p.Nk;
  }
  const float* kbias = p.key_bias ? p.key_bias + (size_t)b * p.Nk : nullptr;

  const uint32_t sbase = smem_u32(smem);
  if (nblk > 0) mbar_wait(q_full, 0);
  for (int n = 0; n < nblk; ++n) {
    if (threadIdx.x == 0 && n + 1 < nblk) load_kv(n + 1);           // its stage was handed back by the barrier that ended block n - 1
    mbar_wait(&kv_full[n & 1], (n >> 1) & 1);
    const uint32_t st = sbase + kT5OffKV + (n & 1) * kT5StageBytes;
    // ---- S = Q K^T (this warpgroup's 64 rows x 64 keys)
    float s[kT5Blk / 2];
    wgmma_fence();
    const uint64_t qd = make_smem_desc(sbase + wg * 8192, 16, 1024, kLayoutSW128);
    const uint64_t kd = make_smem_desc(st, 16, 1024, kLayoutSW128);
#pragma unroll
    for (int k = 0; k < 4; ++k) wgmma_ss<kT5Blk, 0, 0>(s, qd + 2 * k, kd + 2 * k, k != 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(s);
    // ---- online softmax in the log2 domain
    const int jbase = n * kT5Blk + cq;
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int j = 0; j < kT5Blk / 8; ++j)
#pragma unroll
      for (int hh = 0; hh < 2; ++hh)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int key = jbase + 8 * j + e;
          float t = -INFINITY;
          if (key < kv_len) {
            t = s[4 * j + 2 * hh + e] * p.scale_log2;
            t = fmaf((__ldg(brow[hh] + key) + (kbias ? __ldg(kbias + key) : 0.f)), kLog2e, t);
          }
          s[4 * j + 2 * hh + e] = t;
          mx[hh] = fmaxf(mx[hh], t);
        }
    float corr[2], m_use[2];
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 1));
      mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 2));
      const float m_new = fmaxf(m_run[hh], mx[hh]);
      m_use[hh] = m_new == -INFINITY ? 0.f : m_new;                  // every key so far masked to -inf: P = 0 (no NaN)
      corr[hh] = fast_exp2((m_run[hh] == -INFINITY ? (m_new == -INFINITY ? 0.f : -INFINITY) : m_run[hh]) - m_use[hh]);
      m_run[hh] = m_new;
      l_run[hh] *= corr[hh];
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      o[4 * j] *= corr[0]; o[4 * j + 1] *= corr[0];
      o[4 * j + 2] *= corr[1]; o[4 * j + 3] *= corr[1];
    }
#pragma unroll
    for (int j = 0; j < kT5Blk / 8; ++j)
#pragma unroll
      for (int hh = 0; hh < 2; ++hh)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float pe = fast_exp2(s[4 * j + 2 * hh + e] - m_use[hh]);
          s[4 * j + 2 * hh + e] = pe;
          l_run[hh] += pe;
        }
    // ---- O += P V: P as bf16 A fragments straight from the S accumulators, all packed before the first wgmma
    uint32_t a[kT5Blk / 16][4];
#pragma unroll
    for (int kk = 0; kk < kT5Blk / 16; ++kk)
#pragma unroll
      for (int i = 0; i < 4; ++i) a[kk][i] = pack_bf16x2(s[8 * kk + 2 * i], s[8 * kk + 2 * i + 1]);
    const uint64_t vd = make_smem_desc(st + kT5KvBytes, kT5KvBytes, 1024, kLayoutSW128);
    wgmma_fence_regs(o);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < kT5Blk / 16; ++kk) wgmma_rs<64, 1>(o, a[kk], vd + (uint64_t)(kk * (2048 >> 4)), 1u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(o);
    __syncthreads();                                                // both warpgroups are done with this stage
  }

  // ---- epilogue: O / row_sum -> bf16 -> out[(b*Nq + qrow), h*64 ..]
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    float l = l_run[hh];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const int qrow = q0 + row_in_tile + 8 * hh;
    if (qrow >= p.Nq) continue;
    const float inv = l > 0.f ? 1.0f / l : 0.f;
    __nv_bfloat16* dst = p.out + (size_t)(b * p.Nq + qrow) * p.ldo + h * 64 + cq;
#pragma unroll
    for (int j = 0; j < 8; ++j)
      *reinterpret_cast<uint32_t*>(dst + 8 * j) = pack_bf16x2(o[4 * j + 2 * hh] * inv, o[4 * j + 2 * hh + 1] * inv);
  }
}

}  // namespace pxa

extern "C" int pxa_t5_attn_d64_bf16(const PxaT5AttnArgs* args, void* stream) {
  using namespace pxa;
  constexpr int kT5D = 64;
  constexpr int kT5MaxL = 384;
  if (!args) return fail(PXA_ERR_ARG, "null args");
  const PxaT5AttnArgs& a = *args;
  if (!a.q || !a.k || !a.v || !a.out) return fail(PXA_ERR_ARG, "null q / k / v / out");
  if (!a.bias && !a.rel_bias) return fail(PXA_ERR_ARG, "one of bias [H, L, L] / rel_bias [H, 2L-1] is required");
  if (a.B <= 0 || a.H <= 0 || a.L <= 0) return fail(PXA_ERR_ARG, "bad B / H / L");
  if (a.L > kT5MaxL) return fail(PXA_ERR_ARG, "L = %d: at most %d keys", a.L, kT5MaxL);
  if ((a.q_sn & 7) || (a.q_sh & 7) || (a.k_sn & 7) || (a.k_sh & 7) || (a.v_sn & 7) || (a.v_sh & 7) || (a.ldo & 7))
    return fail(PXA_ERR_ALIGN, "strides must be multiples of 8 elements");
  if ((reinterpret_cast<uintptr_t>(a.out) & 15) || (reinterpret_cast<uintptr_t>(a.bias) & 3) || (reinterpret_cast<uintptr_t>(a.key_bias) & 3) ||
      (reinterpret_cast<uintptr_t>(a.rel_bias) & 3))
    return fail(PXA_ERR_ALIGN, "out must be 16-byte aligned, bias / key_bias 4-byte aligned");
  if ((long long)a.H * kT5D > a.ldo) return fail(PXA_ERR_ARG, "ldo smaller than H * 64");
  PXA_REQUIRE_SM90();
  FaParams p = {};
  p.out = reinterpret_cast<__nv_bfloat16*>(a.out);
  p.bias = a.rel_bias ? nullptr : a.bias;
  p.rel_bias = a.rel_bias;
  p.key_bias = a.key_bias;
  p.B = a.B; p.H = a.H; p.Nq = a.L; p.Nk = a.L; p.ldo = (int)a.ldo;
  p.scale_log2 = a.scale * 1.4426950408889634f;
  const long long rows = (long long)a.B * a.L;
  CUtensorMap qm, km, vm;
  int rc;
  if ((rc = make_fa_map(&qm, a.q, kT5D, a.H, rows, a.q_sn, a.q_sh, 64, kT5TileQ, CU_TENSOR_MAP_SWIZZLE_128B))) return rc;
  if ((rc = make_fa_map(&km, a.k, kT5D, a.H, rows, a.k_sn, a.k_sh, 64, kT5Blk, CU_TENSOR_MAP_SWIZZLE_128B))) return rc;
  if ((rc = make_fa_map(&vm, a.v, kT5D, a.H, rows, a.v_sn, a.v_sh, 64, kT5Blk, CU_TENSOR_MAP_SWIZZLE_128B))) return rc;
  PXA_CHECK_CUDA(cudaFuncSetAttribute(t5_attn_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kT5Smem));
  dim3 grid((a.L + kT5TileQ - 1) / kT5TileQ, a.H, a.B);
  t5_attn_fwd_kernel<<<grid, kT5Threads, kT5Smem, reinterpret_cast<cudaStream_t>(stream)>>>(qm, km, vm, p);
  launch_counter()++;
  PXA_CHECK_CUDA(cudaGetLastError());
  return PXA_OK;
}
