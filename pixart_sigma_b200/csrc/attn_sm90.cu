// pxa_flash_attn_d72_bf16: softmax(Q K^T * scale) V for head_dim 72 on wgmma tensor cores (sm_90a); kernel in attn_fwd.cuh.
//
// Algorithmic work: 4 * Nq * Nk * 72 FLOP per (sample, head).
#include "attn_fwd.cuh"

extern "C" int pxa_flash_attn_d72_bf16(const PxaAttnArgs* args, void* stream) {
  using namespace pxa;
  constexpr int kD = 72;
  if (!args) return fail(PXA_ERR_ARG, "null args");
  const PxaAttnArgs& a = *args;
  if (!a.q || !a.k || !a.v || !a.out) return fail(PXA_ERR_ARG, "null q / k / v / out");
  if (a.B <= 0 || a.H <= 0 || a.Nq <= 0 || a.Nk < 0) return fail(PXA_ERR_ARG, "bad B/H/Nq/Nk");
  if (a.kv_rows <= 0) return fail(PXA_ERR_ARG, "kv_rows must be > 0");
  if ((a.q_sn & 7) || (a.q_sh & 7) || (a.k_sn & 7) || (a.k_sh & 7) || (a.v_sn & 7) || (a.v_sh & 7) || (a.ldo & 7))
    return fail(PXA_ERR_ALIGN, "strides must be multiples of 8 elements");
  if (reinterpret_cast<uintptr_t>(a.out) & 15) return fail(PXA_ERR_ALIGN, "out must be 16-byte aligned");
  if (a.H * kD > a.ldo) return fail(PXA_ERR_ARG, "ldo smaller than H*72");
  PXA_REQUIRE_SM90();
  if (a.p_precision != 0 && a.p_precision != 1) return fail(PXA_ERR_ARG, "p_precision must be 0 (bf16 P) or 1 (bf16 hi + lo P)");
  if (!(a.scale >= 0.f)) return fail(PXA_ERR_ARG, "scale must be >= 0");   // the kernel takes the row max on unscaled logits
  FaParams p = {};
  p.out = reinterpret_cast<__nv_bfloat16*>(a.out);
  p.lse = a.lse;
  p.kv_len = a.kv_len;
  p.kv_off = a.kv_off;
  p.B = a.B; p.H = a.H; p.Nq = a.Nq; p.Nk = a.Nk; p.ldo = a.ldo;
  p.scale_log2 = a.scale * 1.4426950408889634f;
  p.reverse_batch = a.reverse_batch ? 1 : 0;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const long long q_rows = (long long)a.B * a.Nq;
  FaMaps maps;
  const void* base[3] = {a.q, a.k, a.v};
  const long long rows[3] = {q_rows, a.kv_rows, a.kv_rows}, sn[3] = {a.q_sn, a.k_sn, a.v_sn}, sh[3] = {a.q_sh, a.k_sh, a.v_sh};
  CUtensorMap* m[3] = {maps.q, maps.k, maps.v};
  for (int t = 0; t < 3; ++t) {
    const int box_rows = t == 0 ? kFaTileQ : kFaBlk;
    int rc = make_fa_map(&m[t][0], base[t], kD, a.H, rows[t], sn[t], sh[t], 64, box_rows, CU_TENSOR_MAP_SWIZZLE_128B);
    if (!rc) rc = make_fa_map(&m[t][1], base[t], kD, a.H, rows[t], sn[t], sh[t], 16, box_rows, CU_TENSOR_MAP_SWIZZLE_32B);
    if (rc) return rc;
  }
  auto kernel = a.p_precision ? flash_fwd_d72_kernel<true> : flash_fwd_d72_kernel<false>;
  PXA_CHECK_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kFaSmem));
  dim3 grid((a.Nq + kFaTileQ - 1) / kFaTileQ, a.H, a.B);
  kernel<<<grid, kFaThreads, kFaSmem, s>>>(maps, p);
  launch_counter()++;
  PXA_CHECK_CUDA(cudaGetLastError());
  return PXA_OK;
}
