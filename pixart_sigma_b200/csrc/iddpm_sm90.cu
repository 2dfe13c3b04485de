// IDDPM ancestral sampling step (pxa_iddpm_step): forward_with_cfg's three-channel CFG mix, the learned-range variance, the
// x0 prediction, the posterior mean and the noise term of one p_sample in one elementwise pass (include/pixart_sm100.h).
// One thread per pixel of one image: it reads the 8 output channels of its row (guided: of both rows of the CFG pair), so the
// mix needs no exchange between threads and any hw works.  Consecutive threads take consecutive pixels, so every load and
// store of a warp is one contiguous run per channel.  Elementwise and HBM-bound; a few microseconds per step at 1024px.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <math.h>

#include "host_common.cuh"

namespace pxa {

constexpr int kIddpmThreads = 256;

__device__ __forceinline__ float iddpm_ld(const float* p) { return __ldg(p); }
__device__ __forceinline__ float iddpm_ld(const __nv_bfloat16* p) { return __bfloat162float(*p); }
__device__ __forceinline__ float iddpm_ld(const __half* p) { return __half2float(*p); }

struct IddpmScalars {
  float cfg, sra, srm1, c1, c2, log_beta, post_logvar;
};

// p_mean_variance + p_sample for one element: x the row's current sample, eps its (mixed) noise prediction, v its variance
// channel, z its noise draw (unused without noise).
template <bool kClip, bool kNoise>
__device__ __forceinline__ float iddpm_update(const IddpmScalars& s, float x, float eps, float v, float z) {
  const float frac = (v + 1.f) * 0.5f;
  const float logvar = frac * s.log_beta + (1.f - frac) * s.post_logvar;
  float x0 = s.sra * x - s.srm1 * eps;
  if constexpr (kClip) x0 = fminf(fmaxf(x0, -1.f), 1.f);
  const float mean = s.c1 * x0 + s.c2 * x;
  if constexpr (kNoise) return mean + expf(0.5f * logvar) * z;
  return mean;
}

template <typename OT, bool kGuided, bool kClip, bool kNoise>
__global__ void __launch_bounds__(kIddpmThreads) iddpm_step_kernel(const OT* __restrict__ mo, float* __restrict__ img,
                                                                   const float* __restrict__ noise,
                                                                   float* __restrict__ next_in, long long obs, int n, int hw,
                                                                   IddpmScalars s) {
  const long long total = (long long)n * hw;                 // guided: one thread per (pair, pixel); else per (row, pixel)
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int r = (int)(i / hw);
    const int p = (int)(i - (long long)r * hw);
    const OT* oc = mo + (size_t)r * obs + p;                 // this row (guided: the conditional row)
    const size_t xc = (size_t)r * 4 * hw + p;
    if constexpr (kGuided) {
      const OT* ou = mo + (size_t)(r + n) * obs + p;         // its unconditional partner
      const size_t xu = (size_t)(r + n) * 4 * hw + p;
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const size_t off = (size_t)c * hw;
        float ec = iddpm_ld(oc + off), eu = iddpm_ld(ou + off);
        if (c < 3) {                                         // forward_with_cfg mixes channels 0..2 only
          ec = eu + s.cfg * (ec - eu);
          eu = ec;
        }
        const float zc = kNoise ? __ldg(noise + xc + off) : 0.f, zu = kNoise ? __ldg(noise + xu + off) : 0.f;
        const float nc = iddpm_update<kClip, kNoise>(s, img[xc + off], ec, iddpm_ld(oc + 4 * (size_t)hw + off), zc);
        const float nu = iddpm_update<kClip, kNoise>(s, img[xu + off], eu, iddpm_ld(ou + 4 * (size_t)hw + off), zu);
        img[xc + off] = nc;
        img[xu + off] = nu;
        next_in[xc + off] = nc;                              // the next model input [img[:n] ; img[:n]]
        next_in[xu + off] = nc;
      }
    } else {
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const size_t off = (size_t)c * hw;
        const float z = kNoise ? __ldg(noise + xc + off) : 0.f;
        img[xc + off] = iddpm_update<kClip, kNoise>(s, img[xc + off], iddpm_ld(oc + off), iddpm_ld(oc + 4 * (size_t)hw + off), z);
      }
    }
  }
}

template <typename OT>
void iddpm_launch(const PxaIddpmStepArgs& a, const IddpmScalars& s, int grid, cudaStream_t st) {
  const OT* mo = reinterpret_cast<const OT*>(a.model_out);
#define PXA_IDDPM_LAUNCH(G, C, Z) \
  iddpm_step_kernel<OT, G, C, Z><<<grid, kIddpmThreads, 0, st>>>(mo, a.img, a.noise, a.next_in, a.out_batch_stride, a.n, a.hw, s)
#define PXA_IDDPM_NOISE(G, C) \
  if (a.noise) PXA_IDDPM_LAUNCH(G, C, true); else PXA_IDDPM_LAUNCH(G, C, false)
#define PXA_IDDPM_CLIP(G) \
  if (a.clip) { PXA_IDDPM_NOISE(G, true); } else { PXA_IDDPM_NOISE(G, false); }
  if (a.guided) { PXA_IDDPM_CLIP(true); } else { PXA_IDDPM_CLIP(false); }
#undef PXA_IDDPM_CLIP
#undef PXA_IDDPM_NOISE
#undef PXA_IDDPM_LAUNCH
}

}  // namespace pxa

extern "C" int pxa_iddpm_step(const PxaIddpmStepArgs* args, void* stream) {
  using namespace pxa;
  if (!args) return fail(PXA_ERR_ARG, "null args");
  const PxaIddpmStepArgs& a = *args;
  if (!a.model_out || !a.img) return fail(PXA_ERR_ARG, "null pointer");
  if (a.guided != 0 && a.guided != 1) return fail(PXA_ERR_ARG, "guided must be 0 or 1");
  if (a.clip != 0 && a.clip != 1) return fail(PXA_ERR_ARG, "clip must be 0 or 1");
  if (a.guided && !a.next_in) return fail(PXA_ERR_ARG, "next_in required in guided mode");
  if (a.n <= 0 || a.hw <= 0) return fail(PXA_ERR_ARG, "n > 0 and hw > 0 required (n=%d hw=%d)", a.n, a.hw);
  if (a.out_batch_stride < 8LL * a.hw) return fail(PXA_ERR_ARG, "out_batch_stride smaller than 8*hw");
  if (a.out_dtype != PXA_DTYPE_F32 && a.out_dtype != PXA_DTYPE_BF16 && a.out_dtype != PXA_DTYPE_F16)
    return fail(PXA_ERR_ARG, "out_dtype must be PXA_DTYPE_F32, PXA_DTYPE_BF16 or PXA_DTYPE_F16");
  const uintptr_t esz = a.out_dtype == PXA_DTYPE_F32 ? 4 : 2;
  if ((reinterpret_cast<uintptr_t>(a.model_out) & (esz - 1)) ||
      ((reinterpret_cast<uintptr_t>(a.img) | reinterpret_cast<uintptr_t>(a.noise) | reinterpret_cast<uintptr_t>(a.next_in)) & 3))
    return fail(PXA_ERR_ALIGN, "model_out / img / noise / next_in must be aligned to their element size");
  PXA_REQUIRE_SM90();
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const IddpmScalars s{a.cfg_scale, a.sqrt_recip_ac, a.sqrt_recipm1_ac, a.post_c1, a.post_c2, a.log_beta, a.post_logvar};
  const long long total = (long long)a.n * a.hw;
  int grid = (int)((total + kIddpmThreads - 1) / kIddpmThreads);
  const int cap = device_info().sms * 8;
  if (grid > cap) grid = cap;
  if (a.out_dtype == PXA_DTYPE_F32)
    iddpm_launch<float>(a, s, grid, st);
  else if (a.out_dtype == PXA_DTYPE_BF16)
    iddpm_launch<__nv_bfloat16>(a, s, grid, st);
  else
    iddpm_launch<__half>(a, s, grid, st);
  launch_counter()++;
  PXA_CHECK_CUDA(cudaGetLastError());
  return PXA_OK;
}
