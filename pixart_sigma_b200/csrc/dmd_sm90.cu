// DMD distribution-matching loss (pxa_dmd_loss): the glue between the one-step generator's x0, the real model's CFG batch and
// the fake model's output, with the gradient with respect to the generator's output.  Elementwise and HBM-bound.  Products,
// sums and divisions that restate a reference fp32 tensor operation use the _rn intrinsics, which the compiler never
// contracts into an FMA, so each is rounded once, as the reference's separate torch operations are.  The per-sample mean and
// the loss are summed from fixed fp64 per-CTA partials in a fixed order, never with floating-point atomics.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <math.h>

#include "host_common.cuh"

namespace pxa {

constexpr int kDmdThreads = 256;

__device__ __forceinline__ void dmd_load4(const float* __restrict__ p, float (&v)[4]) {
  const float4 t = *reinterpret_cast<const float4*>(p);
  v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
}
__device__ __forceinline__ void dmd_load4(const __nv_bfloat16* __restrict__ p, float (&v)[4]) {
  const uint2 t = *reinterpret_cast<const uint2*>(p);
  const __nv_bfloat162 a = *reinterpret_cast<const __nv_bfloat162*>(&t.x), b = *reinterpret_cast<const __nv_bfloat162*>(&t.y);
  const float2 fa = __bfloat1622float2(a), fb = __bfloat1622float2(b);
  v[0] = fa.x; v[1] = fa.y; v[2] = fb.x; v[3] = fb.y;
}
__device__ __forceinline__ void dmd_store4(float* __restrict__ p, const float (&v)[4]) {
  *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
}

// Deterministic fp64 block sum (fixed shuffle tree, then warp partials in warp order); thread 0 receives the result.
__device__ __forceinline__ double dmd_block_sum(double v) {
  __shared__ double red[kDmdThreads / 32];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  double s = 0.0;
  if (threadIdx.x == 0) {
#pragma unroll
    for (int k = 0; k < kDmdThreads / 32; ++k) s += red[k];
  }
  return s;
}

// sqrt(a), sqrt(1 - a) of sample img (`alpha_prod_t ** 0.5`, `(1.0 - alpha_prod_t) ** 0.5`); NaN for a timestep out of range
__device__ __forceinline__ void dmd_alpha(const PxaDmdLossArgs& a, int img, float& sa, float& sb) {
  const long long t = a.timesteps[img];
  const float ac = (t >= 0 && t < a.n_timesteps) ? a.alphas_cumprod[t] : __int_as_float(0x7fc00000);
  sa = __fsqrt_rn(ac);
  sb = __fsqrt_rn(__fsub_rn(1.f, ac));
}

// score_real = su + cfg (sc - su) with su = -eps_u, sc = -eps_c (train_pixart_dmd.py:538-539)
template <typename RT>
__device__ __forceinline__ void dmd_score_real(const PxaDmdLossArgs& a, int img, int e, float (&sr)[4]) {
  const RT* real = reinterpret_cast<const RT*>(a.real_out);
  float eu[4], ec[4];
  dmd_load4(real + (size_t)img * a.real_batch_stride + e, eu);
  dmd_load4(real + (size_t)(img + a.b) * a.real_batch_stride + e, ec);
#pragma unroll
  for (int k = 0; k < 4; ++k) sr[k] = __fadd_rn(-eu[k], __fmul_rn(a.cfg, __fsub_rn(-ec[k], -eu[k])));
}

// Launch 1, grid (PXA_DMD_PARTS, b): partials[img * PARTS + cta] = fp64 sum of |latents - pred| over the CTA's elements.
template <typename RT>
__global__ void __launch_bounds__(kDmdThreads) dmd_abs_kernel(PxaDmdLossArgs a) {
  const int img = blockIdx.y;
  float sa, sb;
  dmd_alpha(a, img, sa, sb);
  double acc = 0.0;
  for (int i = blockIdx.x * kDmdThreads + threadIdx.x; i < a.hw; i += PXA_DMD_PARTS * kDmdThreads) {
    const int e = i * 4;
    const size_t off = (size_t)img * 4 * a.hw + e;
    float sr[4], lat[4], nz[4];
    dmd_score_real<RT>(a, img, e, sr);
    dmd_load4(a.latents + off, lat);
    dmd_load4(a.noisy + off, nz);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float pred = __fdiv_rn(__fadd_rn(nz[k], __fmul_rn(sb, sr[k])), sa);
      acc += (double)fabsf(__fsub_rn(lat[k], pred));
    }
  }
  const double s = dmd_block_sum(acc);
  if (threadIdx.x == 0) a.partials[(size_t)img * PXA_DMD_PARTS + blockIdx.x] = s;
}

// Launch 2, grid (PXA_DMD_PARTS, b): weight, gradient and loss partials (written after the abs partials).
template <typename RT, typename FT>
__global__ void __launch_bounds__(kDmdThreads) dmd_grad_kernel(PxaDmdLossArgs a, float two_over_n) {
  __shared__ float w_s;
  const int img = blockIdx.y;
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int k = 0; k < PXA_DMD_PARTS; ++k) s += a.partials[(size_t)img * PXA_DMD_PARTS + k];
    const float mean = (float)(s / (4.0 * (double)a.hw));
    w_s = __fdiv_rn(1.f, __fadd_rn(mean, 1e-5f));
    if (blockIdx.x == 0) a.weight[img] = w_s;
  }
  __syncthreads();
  const float w = w_s;
  float sa, sb;
  dmd_alpha(a, img, sa, sb);
  const FT* fake = reinterpret_cast<const FT*>(a.fake_out);
  double acc = 0.0;
  for (int i = blockIdx.x * kDmdThreads + threadIdx.x; i < a.hw; i += PXA_DMD_PARTS * kDmdThreads) {
    const int e = i * 4;
    float* dout = a.d_gen_out + (size_t)img * a.out_channels * a.hw + e;
    if (a.out_channels == 8) dmd_store4(dout + 4 * (size_t)a.hw, {0.f, 0.f, 0.f, 0.f});
    float sr[4], ef[4], lat[4], g[4];
    dmd_score_real<RT>(a, img, e, sr);
    dmd_load4(fake + (size_t)img * a.fake_batch_stride + e, ef);
    dmd_load4(a.latents + (size_t)img * 4 * a.hw + e, lat);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float coeff = __fdiv_rn(__fmul_rn(__fsub_rn(-ef[k], sr[k]), sb), sa);
      const float target = __fsub_rn(lat[k], __fmul_rn(w, coeff));
      const float d = __fsub_rn(lat[k], target);
      acc += (double)__fmul_rn(d, d);
      g[k] = -__fmul_rn(__fdiv_rn(__fmul_rn(d, two_over_n), a.gen_sqrt_alpha), a.gen_sqrt_beta);
    }
    dmd_store4(dout, g);
  }
  const double s = dmd_block_sum(acc);
  if (threadIdx.x == 0) a.partials[(size_t)(a.b + img) * PXA_DMD_PARTS + blockIdx.x] = s;
}

// Launch 3, one CTA: loss = (sum of the loss partials in index order) / count.
__global__ void __launch_bounds__(kDmdThreads) dmd_loss_finalize_kernel(const double* __restrict__ partials, int n,
                                                                        float* __restrict__ loss, double count) {
  double acc = 0.0;
  for (int i = threadIdx.x; i < n; i += kDmdThreads) acc += partials[i];
  const double s = dmd_block_sum(acc);
  if (threadIdx.x == 0) *loss = (float)(s / count);
}

inline bool dmd_misaligned(const void* p, uintptr_t bytes) { return reinterpret_cast<uintptr_t>(p) & (bytes - 1); }

inline int dmd_check_out(const void* p, int dtype, int64_t batch_stride, int hw, const char* what) {
  if (!p) return fail(PXA_ERR_ARG, "%s: null pointer", what);
  if (dtype != PXA_DTYPE_F32 && dtype != PXA_DTYPE_BF16) return fail(PXA_ERR_ARG, "%s: dtype must be PXA_DTYPE_F32 or _BF16", what);
  if (batch_stride < 4LL * hw) return fail(PXA_ERR_ARG, "%s: batch stride smaller than 4*hw", what);
  const int esz = dtype == PXA_DTYPE_F32 ? 4 : 2;
  if (dmd_misaligned(p, 4 * esz) || ((batch_stride * esz) & (4 * esz - 1)))
    return fail(PXA_ERR_ALIGN, "%s: base and batch stride must be aligned to 4 elements", what);
  return PXA_OK;
}

template <typename RT, typename FT>
void dmd_launch(const PxaDmdLossArgs& a, cudaStream_t s, float two_over_n) {
  const dim3 grid(PXA_DMD_PARTS, (unsigned)a.b);
  dmd_abs_kernel<RT><<<grid, kDmdThreads, 0, s>>>(a);
  launch_counter()++;
  dmd_grad_kernel<RT, FT><<<grid, kDmdThreads, 0, s>>>(a, two_over_n);
  launch_counter()++;
}

}  // namespace pxa

extern "C" int pxa_dmd_loss(const PxaDmdLossArgs* args, void* stream) {
  using namespace pxa;
  if (!args) return fail(PXA_ERR_ARG, "null args");
  const PxaDmdLossArgs& a = *args;
  if (!a.latents || !a.noisy || !a.timesteps || !a.alphas_cumprod || !a.d_gen_out || !a.loss || !a.weight || !a.partials)
    return fail(PXA_ERR_ARG, "null pointer");
  if (a.b <= 0 || a.b > 65535 || a.hw <= 0 || (a.hw & 3))
    return fail(PXA_ERR_ARG, "b in 1..65535 and hw a positive multiple of 4 required (b=%d hw=%d)", a.b, a.hw);
  if (a.n_timesteps <= 0) return fail(PXA_ERR_ARG, "n_timesteps must be positive");
  if (a.out_channels != 4 && a.out_channels != 8) return fail(PXA_ERR_ARG, "out_channels must be 4 or 8");
  if (int rc = dmd_check_out(a.real_out, a.real_dtype, a.real_batch_stride, a.hw, "real_out")) return rc;
  if (int rc = dmd_check_out(a.fake_out, a.fake_dtype, a.fake_batch_stride, a.hw, "fake_out")) return rc;
  if (dmd_misaligned(a.latents, 16) || dmd_misaligned(a.noisy, 16) || dmd_misaligned(a.d_gen_out, 16) ||
      dmd_misaligned(a.partials, 8) || dmd_misaligned(a.timesteps, 8) || dmd_misaligned(a.alphas_cumprod, 4) ||
      dmd_misaligned(a.weight, 4) || dmd_misaligned(a.loss, 4))
    return fail(PXA_ERR_ALIGN, "latents / noisy / d_gen_out must be 16-byte aligned, partials / timesteps 8-byte");
  PXA_REQUIRE_SM90();
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const double count = 4.0 * (double)a.b * (double)a.hw;
  const float two_over_n = (float)(2.0 / count);
  const bool rf = a.real_dtype == PXA_DTYPE_F32, ff = a.fake_dtype == PXA_DTYPE_F32;
  if (rf && ff) dmd_launch<float, float>(a, s, two_over_n);
  else if (rf) dmd_launch<float, __nv_bfloat16>(a, s, two_over_n);
  else if (ff) dmd_launch<__nv_bfloat16, float>(a, s, two_over_n);
  else dmd_launch<__nv_bfloat16, __nv_bfloat16>(a, s, two_over_n);
  PXA_CHECK_CUDA(cudaGetLastError());
  dmd_loss_finalize_kernel<<<1, kDmdThreads, 0, s>>>(a.partials + (size_t)a.b * PXA_DMD_PARTS, a.b * PXA_DMD_PARTS, a.loss, count);
  launch_counter()++;
  PXA_CHECK_CUDA(cudaGetLastError());
  return PXA_OK;
}
