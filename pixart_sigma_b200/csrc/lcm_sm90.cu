// LCM kernels: the few-step sampler step (pxa_lcm_step), the consistency-distillation glue (pxa_lcm_teacher_target,
// pxa_lcm_consistency_loss) and the flat EMA update (pxa_ema_flat).  All are elementwise and HBM-bound.  Products, sums and
// divisions that restate a reference fp32 tensor operation use the _rn intrinsics, which the compiler never contracts into
// an FMA, so each is rounded once, as the reference's separate torch operations are.  The loss sum uses fixed per-CTA
// partials reduced in a fixed order, never floating-point atomics.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <math.h>

#include "host_common.cuh"

namespace pxa {

constexpr int kLcmThreads = 256;

__device__ __forceinline__ void lcm_load4(const float* __restrict__ p, float (&v)[4]) {
  const float4 t = *reinterpret_cast<const float4*>(p);
  v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
}
__device__ __forceinline__ void lcm_load4(const __nv_bfloat16* __restrict__ p, float (&v)[4]) {
  const uint2 t = *reinterpret_cast<const uint2*>(p);
  const __nv_bfloat162 a = *reinterpret_cast<const __nv_bfloat162*>(&t.x), b = *reinterpret_cast<const __nv_bfloat162*>(&t.y);
  const float2 fa = __bfloat1622float2(a), fb = __bfloat1622float2(b);
  v[0] = fa.x; v[1] = fa.y; v[2] = fb.x; v[3] = fb.y;
}
__device__ __forceinline__ void lcm_store4(float* __restrict__ p, const float (&v)[4]) {
  *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
}

// ------------------------------------------------------------------------------------------------- sampler step
// One thread per 4 consecutive latent elements of one image (hw % 4 == 0).
template <typename OT>
__global__ void __launch_bounds__(kLcmThreads) lcm_step_kernel(const OT* __restrict__ mo, const float* x,
                                                                const float* __restrict__ noise, float* __restrict__ denoised,
                                                                float* x_next, long long obs, int n, int hw, float sqrt_alpha,
                                                                float sqrt_beta, float c_skip, float c_out, float c_prev,
                                                                float c_noise) {
  const long long total = (long long)n * hw;  // 4 channels x hw elements / 4 per thread
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int img = (int)(i / hw);
    const int e = (int)(i - (long long)img * hw) * 4;
    const size_t off = (size_t)img * 4 * hw + e;
    float eps[4], xs[4], nz[4] = {0.f, 0.f, 0.f, 0.f}, den[4], nx[4];
    lcm_load4(mo + (size_t)img * obs + e, eps);
    lcm_load4(x + off, xs);
    if (c_noise != 0.f) lcm_load4(noise + off, nz);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float x0 = __fdiv_rn(__fsub_rn(xs[k], __fmul_rn(sqrt_beta, eps[k])), sqrt_alpha);
      den[k] = __fadd_rn(__fmul_rn(c_out, x0), __fmul_rn(c_skip, xs[k]));
      nx[k] = c_noise != 0.f ? __fadd_rn(__fmul_rn(c_prev, den[k]), __fmul_rn(c_noise, nz[k])) : __fmul_rn(c_prev, den[k]);
    }
    lcm_store4(denoised + off, den);
    lcm_store4(x_next + off, nx);
  }
}

// ------------------------------------------------------------------------------------------------- distillation
__device__ __forceinline__ bool lcm_row(const PxaLcmRow* __restrict__ table, const int64_t* __restrict__ index, int img,
                                        int n_rows, PxaLcmRow& r) {
  const long long k = index[img];
  if (k < 0 || k >= n_rows) return false;
  r = table[k];
  return true;
}

template <typename OT>
__global__ void __launch_bounds__(kLcmThreads) lcm_teacher_kernel(const OT* __restrict__ to, const float* __restrict__ x_t,
                                                                   const int64_t* __restrict__ index,
                                                                   const PxaLcmRow* __restrict__ table,
                                                                   float* __restrict__ x_prev, long long obs, int b, int hw,
                                                                   int n_rows, float w) {
  const long long total = (long long)b * hw;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int img = (int)(i / hw);
    const int e = (int)(i - (long long)img * hw) * 4;
    const size_t off = (size_t)img * 4 * hw + e;
    PxaLcmRow r;
    float out[4];
    if (!lcm_row(table, index, img, n_rows, r)) {
#pragma unroll
      for (int k = 0; k < 4; ++k) out[k] = __int_as_float(0x7fc00000);
      lcm_store4(x_prev + off, out);
      continue;
    }
    float ec[4], eu[4], xs[4];
    lcm_load4(to + (size_t)img * obs + e, ec);
    lcm_load4(to + (size_t)(img + b) * obs + e, eu);
    lcm_load4(x_t + off, xs);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float sx = __fmul_rn(r.sra_s, xs[k]);
      const float x0c = __fsub_rn(sx, __fmul_rn(r.srm1_s, ec[k]));
      const float x0u = __fsub_rn(sx, __fmul_rn(r.srm1_s, eu[k]));
      const float x0 = __fadd_rn(x0c, __fmul_rn(w, __fsub_rn(x0c, x0u)));
      const float ep = __fadd_rn(ec[k], __fmul_rn(w, __fsub_rn(ec[k], eu[k])));
      out[k] = __double2float_rn(__dadd_rn(__dmul_rn(r.sqrt_acp, (double)x0), __dmul_rn(r.sqrt_1macp, (double)ep)));
    }
    lcm_store4(x_prev + off, out);
  }
}

// Deterministic fp64 block sum (fixed shuffle tree, then warp partials in warp order); thread 0 receives the result.
__device__ __forceinline__ double lcm_block_sum(double v) {
  __shared__ double red[kLcmThreads / 32];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  double s = 0.0;
  if (threadIdx.x == 0) {
#pragma unroll
    for (int k = 0; k < kLcmThreads / 32; ++k) s += red[k];
  }
  return s;
}

template <typename ET, bool kHuber>
__global__ void __launch_bounds__(kLcmThreads) lcm_loss_kernel(PxaLcmLossArgs a, float inv_count) {
  const ET* __restrict__ ema = reinterpret_cast<const ET*>(a.ema_out);
  const long long total = (long long)a.b * a.hw;
  const float c = a.huber_c, c2 = __fmul_rn(a.huber_c, a.huber_c);
  double acc = 0.0;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int img = (int)(i / a.hw);
    const int e = (int)(i - (long long)img * a.hw) * 4;
    const size_t off = (size_t)img * 4 * a.hw + e;
    float* dout = a.d_student_out + (size_t)img * a.out_channels * a.hw + e;
    if (a.out_channels == 8) lcm_store4(dout + 4 * (size_t)a.hw, {0.f, 0.f, 0.f, 0.f});
    PxaLcmRow r;
    float g[4];
    if (!lcm_row(a.table, a.index, img, a.n_rows, r)) {
#pragma unroll
      for (int k = 0; k < 4; ++k) g[k] = __int_as_float(0x7fc00000);
      lcm_store4(dout, g);
      acc += (double)g[0];
      continue;
    }
    float es[4], ee[4], xs[4], xp[4];
    lcm_load4(a.student_out + (size_t)img * a.student_batch_stride + e, es);
    lcm_load4(ema + (size_t)img * a.ema_batch_stride + e, ee);
    lcm_load4(a.x_t + off, xs);
    lcm_load4(a.x_prev + off, xp);
    const float coef = __fmul_rn(-__fmul_rn(r.cout_s, r.srm1_s), inv_count);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float x0s = __fsub_rn(__fmul_rn(r.sra_s, xs[k]), __fmul_rn(r.srm1_s, es[k]));
      const float pred = __fadd_rn(__fmul_rn(r.cskip_s, xs[k]), __fmul_rn(r.cout_s, x0s));
      const float x0e = __fsub_rn(__fmul_rn(r.sra_t, xp[k]), __fmul_rn(r.srm1_t, ee[k]));
      const float tgt = __double2float_rn(__dadd_rn(__dmul_rn((double)r.cskip_t, (double)xp[k]),
                                                    (double)__fmul_rn(r.cout_t, x0e)));
      const float d = __fsub_rn(pred, tgt);
      const float d2 = __fmul_rn(d, d);
      float l, dl;
      if (kHuber) {
        const float rt = sqrtf(__fadd_rn(d2, c2));
        l = __fdiv_rn(d2, __fadd_rn(rt, c));
        dl = __fdiv_rn(d, rt);
      } else {
        l = d2;
        dl = __fmul_rn(2.f, d);
      }
      acc += (double)l;
      g[k] = __fmul_rn(dl, coef);
    }
    lcm_store4(dout, g);
  }
  const double s = lcm_block_sum(acc);
  if (threadIdx.x == 0) a.partials[blockIdx.x] = s;
}

__global__ void __launch_bounds__(kLcmThreads) lcm_loss_finalize_kernel(const double* __restrict__ partials,
                                                                        float* __restrict__ loss, double count) {
  double acc = 0.0;
  for (int i = threadIdx.x; i < PXA_LCM_LOSS_PARTS; i += kLcmThreads) acc += partials[i];
  const double s = lcm_block_sum(acc);
  if (threadIdx.x == 0) *loss = (float)(s / count);
}

// ------------------------------------------------------------------------------------------------- EMA
__global__ void __launch_bounds__(kLcmThreads) ema_flat_kernel(const PxaEmaBucket* __restrict__ table, float rate, float omr) {
  const PxaEmaBucket e = table[blockIdx.y];
  const long long n4 = e.n >> 2;
  const long long stride = (long long)gridDim.x * kLcmThreads;
  const long long first = (long long)blockIdx.x * kLcmThreads + threadIdx.x;
  float4* m4 = reinterpret_cast<float4*>(e.master);
  const float4* s4 = reinterpret_cast<const float4*>(e.src);
  uint2* h4 = reinterpret_cast<uint2*>(e.shadow);
  for (long long i = first; i < n4; i += stride) {
    float4 m = m4[i];
    const float4 s = s4[i];
    m.x = __fadd_rn(__fmul_rn(m.x, rate), __fmul_rn(s.x, omr));
    m.y = __fadd_rn(__fmul_rn(m.y, rate), __fmul_rn(s.y, omr));
    m.z = __fadd_rn(__fmul_rn(m.z, rate), __fmul_rn(s.z, omr));
    m.w = __fadd_rn(__fmul_rn(m.w, rate), __fmul_rn(s.w, omr));
    m4[i] = m;
    if (h4) {
      const __nv_bfloat162 lo = __floats2bfloat162_rn(m.x, m.y), hi = __floats2bfloat162_rn(m.z, m.w);
      uint2 v;
      v.x = *reinterpret_cast<const uint32_t*>(&lo);
      v.y = *reinterpret_cast<const uint32_t*>(&hi);
      h4[i] = v;
    }
  }
  const long long tail = (n4 << 2) + first;
  if (tail < e.n) {
    const float m = __fadd_rn(__fmul_rn(e.master[tail], rate), __fmul_rn(e.src[tail], omr));
    e.master[tail] = m;
    if (e.shadow) reinterpret_cast<__nv_bfloat16*>(e.shadow)[tail] = __float2bfloat16_rn(m);
  }
}

inline bool lcm_misaligned(const void* p, uintptr_t bytes) { return reinterpret_cast<uintptr_t>(p) & (bytes - 1); }

inline int lcm_grid(long long items) {
  long long grid = (items + kLcmThreads - 1) / kLcmThreads;
  const long long cap = (long long)device_info().sms * 8;
  if (grid > cap) grid = cap;
  return (int)(grid < 1 ? 1 : grid);
}

// the model output of an elementwise LCM kernel: fp32 or bf16, 4-element aligned base and batch stride
inline int lcm_check_out(const void* p, int dtype, int64_t batch_stride, int hw, const char* what) {
  if (!p) return fail(PXA_ERR_ARG, "%s: null pointer", what);
  if (dtype != PXA_DTYPE_F32 && dtype != PXA_DTYPE_BF16) return fail(PXA_ERR_ARG, "%s: dtype must be PXA_DTYPE_F32 or _BF16", what);
  if (batch_stride < 4LL * hw) return fail(PXA_ERR_ARG, "%s: batch stride smaller than 4*hw", what);
  const int esz = dtype == PXA_DTYPE_F32 ? 4 : 2;
  if (lcm_misaligned(p, 4 * esz) || ((batch_stride * esz) & (4 * esz - 1)))
    return fail(PXA_ERR_ALIGN, "%s: base and batch stride must be aligned to 4 elements", what);
  return PXA_OK;
}

}  // namespace pxa

extern "C" int pxa_lcm_step(const PxaLcmStepArgs* args, void* stream) {
  using namespace pxa;
  if (!args) return fail(PXA_ERR_ARG, "null args");
  const PxaLcmStepArgs& a = *args;
  if (!a.x || !a.denoised || !a.x_next) return fail(PXA_ERR_ARG, "null pointer");
  if (a.c_noise != 0.f && !a.noise) return fail(PXA_ERR_ARG, "noise required when c_noise is non-zero");
  if (a.n <= 0 || a.hw <= 0 || (a.hw & 3)) return fail(PXA_ERR_ARG, "n > 0 and hw a positive multiple of 4 required (n=%d hw=%d)", a.n, a.hw);
  if (int rc = lcm_check_out(a.model_out, a.out_dtype, a.out_batch_stride, a.hw, "model_out")) return rc;
  if (lcm_misaligned(a.x, 16) || lcm_misaligned(a.noise, 16) || lcm_misaligned(a.denoised, 16) || lcm_misaligned(a.x_next, 16))
    return fail(PXA_ERR_ALIGN, "x / noise / denoised / x_next must be 16-byte aligned");
  PXA_REQUIRE_SM90();
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const int grid = lcm_grid((long long)a.n * a.hw);
  if (a.out_dtype == PXA_DTYPE_F32)
    lcm_step_kernel<float><<<grid, kLcmThreads, 0, s>>>(reinterpret_cast<const float*>(a.model_out), a.x, a.noise, a.denoised,
                                                        a.x_next, a.out_batch_stride, a.n, a.hw, a.sqrt_alpha, a.sqrt_beta,
                                                        a.c_skip, a.c_out, a.c_prev, a.c_noise);
  else
    lcm_step_kernel<__nv_bfloat16><<<grid, kLcmThreads, 0, s>>>(reinterpret_cast<const __nv_bfloat16*>(a.model_out), a.x, a.noise,
                                                                a.denoised, a.x_next, a.out_batch_stride, a.n, a.hw, a.sqrt_alpha,
                                                                a.sqrt_beta, a.c_skip, a.c_out, a.c_prev, a.c_noise);
  launch_counter()++;
  PXA_CHECK_CUDA(cudaGetLastError());
  return PXA_OK;
}

extern "C" int pxa_lcm_teacher_target(const PxaLcmTeacherArgs* args, void* stream) {
  using namespace pxa;
  if (!args) return fail(PXA_ERR_ARG, "null args");
  const PxaLcmTeacherArgs& a = *args;
  if (!a.x_t || !a.index || !a.table || !a.x_prev) return fail(PXA_ERR_ARG, "null pointer");
  if (a.b <= 0 || a.hw <= 0 || (a.hw & 3)) return fail(PXA_ERR_ARG, "b > 0 and hw a positive multiple of 4 required (b=%d hw=%d)", a.b, a.hw);
  if (a.n_rows <= 0 || a.n_rows > PXA_LCM_MAX_ROWS) return fail(PXA_ERR_ARG, "n_rows must be in 1..%d", PXA_LCM_MAX_ROWS);
  if (int rc = lcm_check_out(a.teacher_out, a.out_dtype, a.out_batch_stride, a.hw, "teacher_out")) return rc;
  if (lcm_misaligned(a.x_t, 16) || lcm_misaligned(a.x_prev, 16) || lcm_misaligned(a.table, 16) || lcm_misaligned(a.index, 8))
    return fail(PXA_ERR_ALIGN, "x_t / x_prev / table must be 16-byte aligned, index 8-byte");
  PXA_REQUIRE_SM90();
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const int grid = lcm_grid((long long)a.b * a.hw);
  if (a.out_dtype == PXA_DTYPE_F32)
    lcm_teacher_kernel<float><<<grid, kLcmThreads, 0, s>>>(reinterpret_cast<const float*>(a.teacher_out), a.x_t, a.index, a.table,
                                                           a.x_prev, a.out_batch_stride, a.b, a.hw, a.n_rows, a.w);
  else
    lcm_teacher_kernel<__nv_bfloat16><<<grid, kLcmThreads, 0, s>>>(reinterpret_cast<const __nv_bfloat16*>(a.teacher_out), a.x_t,
                                                                   a.index, a.table, a.x_prev, a.out_batch_stride, a.b, a.hw,
                                                                   a.n_rows, a.w);
  launch_counter()++;
  PXA_CHECK_CUDA(cudaGetLastError());
  return PXA_OK;
}

extern "C" int pxa_lcm_consistency_loss(const PxaLcmLossArgs* args, void* stream) {
  using namespace pxa;
  if (!args) return fail(PXA_ERR_ARG, "null args");
  const PxaLcmLossArgs& a = *args;
  if (!a.x_t || !a.x_prev || !a.index || !a.table || !a.d_student_out || !a.loss || !a.partials)
    return fail(PXA_ERR_ARG, "null pointer");
  if (a.b <= 0 || a.hw <= 0 || (a.hw & 3)) return fail(PXA_ERR_ARG, "b > 0 and hw a positive multiple of 4 required (b=%d hw=%d)", a.b, a.hw);
  if (a.n_rows <= 0 || a.n_rows > PXA_LCM_MAX_ROWS) return fail(PXA_ERR_ARG, "n_rows must be in 1..%d", PXA_LCM_MAX_ROWS);
  if (a.out_channels != 4 && a.out_channels != 8) return fail(PXA_ERR_ARG, "out_channels must be 4 or 8");
  if (a.loss_type != PXA_LCM_HUBER && a.loss_type != PXA_LCM_L2) return fail(PXA_ERR_ARG, "loss_type must be PXA_LCM_HUBER or PXA_LCM_L2");
  if (a.loss_type == PXA_LCM_HUBER && !(a.huber_c > 0.f)) return fail(PXA_ERR_ARG, "huber_c must be positive");
  if (int rc = lcm_check_out(a.student_out, PXA_DTYPE_F32, a.student_batch_stride, a.hw, "student_out")) return rc;
  if (int rc = lcm_check_out(a.ema_out, a.ema_dtype, a.ema_batch_stride, a.hw, "ema_out")) return rc;
  if (lcm_misaligned(a.x_t, 16) || lcm_misaligned(a.x_prev, 16) || lcm_misaligned(a.table, 16) || lcm_misaligned(a.index, 8) ||
      lcm_misaligned(a.d_student_out, 16) || lcm_misaligned(a.partials, 16) || lcm_misaligned(a.loss, 4))
    return fail(PXA_ERR_ALIGN, "x_t / x_prev / table / d_student_out / partials must be 16-byte aligned, index 8-byte, loss 4-byte");
  PXA_REQUIRE_SM90();
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const long long count = 4LL * a.b * a.hw;
  const float inv_count = (float)(1.0 / (double)count);
  const bool huber = a.loss_type == PXA_LCM_HUBER;
#define PXA_LCM_LOSS(ET, H) lcm_loss_kernel<ET, H><<<PXA_LCM_LOSS_PARTS, kLcmThreads, 0, s>>>(a, inv_count)
  if (a.ema_dtype == PXA_DTYPE_F32) {
    if (huber) PXA_LCM_LOSS(float, true); else PXA_LCM_LOSS(float, false);
  } else {
    if (huber) PXA_LCM_LOSS(__nv_bfloat16, true); else PXA_LCM_LOSS(__nv_bfloat16, false);
  }
#undef PXA_LCM_LOSS
  launch_counter()++;
  PXA_CHECK_CUDA(cudaGetLastError());
  lcm_loss_finalize_kernel<<<1, kLcmThreads, 0, s>>>(a.partials, a.loss, (double)count);
  launch_counter()++;
  PXA_CHECK_CUDA(cudaGetLastError());
  return PXA_OK;
}

extern "C" int pxa_ema_flat(const PxaEmaArgs* args, void* stream) {
  using namespace pxa;
  if (!args) return fail(PXA_ERR_ARG, "null args");
  const PxaEmaArgs& a = *args;
  if (!a.table) return fail(PXA_ERR_ARG, "null table");
  if (a.n_buckets <= 0 || a.n_buckets > 65535) return fail(PXA_ERR_ARG, "n_buckets must be in 1..65535 (got %d)", a.n_buckets);
  if (a.max_n <= 0) return fail(PXA_ERR_ARG, "max_n must be positive");
  if (!(a.rate >= 0.0 && a.rate <= 1.0)) return fail(PXA_ERR_ARG, "rate must be in [0, 1]");
  if (lcm_misaligned(a.table, 16)) return fail(PXA_ERR_ALIGN, "table must be 16-byte aligned");
  PXA_REQUIRE_SM90();
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  long long per = (a.max_n / 4 + kLcmThreads - 1) / kLcmThreads;
  const long long cap = ((long long)device_info().sms * 8 + a.n_buckets - 1) / a.n_buckets;
  if (per > cap) per = cap;
  if (per < 1) per = 1;
  const dim3 grid((unsigned)per, (unsigned)a.n_buckets);
  ema_flat_kernel<<<grid, kLcmThreads, 0, s>>>(a.table, (float)a.rate, (float)(1.0 - a.rate));
  launch_counter()++;
  PXA_CHECK_CUDA(cudaGetLastError());
  return PXA_OK;
}
