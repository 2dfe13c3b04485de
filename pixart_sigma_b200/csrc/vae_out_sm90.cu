// VAE output head (pxa_vae_out_u8): the decoder's conv_out (Cin -> 3 channels, 3x3, zero padding 1) on the NHWC bf16 output
// of conv_norm_out + SiLU, followed by torchvision's save_image arithmetic to uint8 pixels, in one pass (include/pixart_sm100.h).
// A CTA owns a 8 x 32 tile of output pixels, one thread per pixel.  The input tile with its one-pixel halo (10 x 34 pixels)
// is staged in shared memory 32 channels at a time, zero outside the image, together with the matching fp32 weight slice;
// each thread then does 9 taps x 32 channels x 3 outputs of FMAs (CUDA cores: N = 3 leaves a tensor-core tile mostly empty).
// The staged pixel stride is 40 channels (80 bytes), so the 16-byte reads of 8 neighbouring pixels hit 8 distinct bank
// groups.  Accumulation is fp32; the u8 conversion is done op by op in fp32 with round-to-nearest intrinsics.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "host_common.cuh"

namespace pxa {

constexpr int kVoTh = 8, kVoTw = 32;                            // output tile (rows x columns), one thread per pixel
constexpr int kVoThreads = kVoTh * kVoTw;
constexpr int kVoHh = kVoTh + 2, kVoHw = kVoTw + 2;             // tile + halo
constexpr int kVoChunk = 32;                                    // channels staged per pass
constexpr int kVoPitch = kVoChunk + 8;                          // staged pixel stride in channels (80 B: conflict-free 16 B reads)

// torchvision.utils.save_image(normalize=True, value_range=(-1, 1)): clamp to the range, (y + 1) / 2, * 255 + 0.5, clamp to
// [0, 255], truncate to uint8.  Each op rounded on its own, as the tensor ops do.
__device__ __forceinline__ uint8_t vae_out_u8(float y) {
  float v = fminf(fmaxf(y, -1.f), 1.f);
  v = __fdiv_rn(__fadd_rn(v, 1.f), 2.f);
  v = __fadd_rn(__fmul_rn(v, 255.f), 0.5f);
  v = fminf(fmaxf(v, 0.f), 255.f);
  return (uint8_t)(int)v;
}

__global__ void __launch_bounds__(kVoThreads) vae_out_u8_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ w,
                                                                const float* __restrict__ bias, uint8_t* __restrict__ out_u8,
                                                                float* __restrict__ out_f32, long long sb, long long sh, long long sw,
                                                                int H, int W, int Cin) {
  __shared__ __align__(16) __nv_bfloat16 tile[kVoHh * kVoHw * kVoPitch];
  __shared__ float wsm[3 * 9 * kVoChunk];                       // [o][tap][c] of the current channel chunk
  const int b = blockIdx.z;
  const int y0 = blockIdx.y * kVoTh, x0 = blockIdx.x * kVoTw;
  const int ty = threadIdx.x / kVoTw, tx = threadIdx.x % kVoTw;
  const __nv_bfloat16* xb = x + (size_t)b * sb;
  float acc[3] = {0.f, 0.f, 0.f};
  for (int c0 = 0; c0 < Cin; c0 += kVoChunk) {
    const int kc = min(kVoChunk, Cin - c0);                     // a multiple of 8
    const int vecs = kc >> 3;
    __syncthreads();                                            // the previous chunk's reads are done
    for (int i = threadIdx.x; i < kVoHh * kVoHw * vecs; i += kVoThreads) {
      const int pix = i / vecs, v = i - pix * vecs;
      const int hy = pix / kVoHw, hx = pix - hy * kVoHw;
      const int gy = y0 + hy - 1, gx = x0 + hx - 1;
      uint4 val = make_uint4(0u, 0u, 0u, 0u);
      if (gy >= 0 && gy < H && gx >= 0 && gx < W)
        val = __ldg(reinterpret_cast<const uint4*>(xb + gy * sh + gx * sw + c0 + v * 8));
      *reinterpret_cast<uint4*>(tile + pix * kVoPitch + v * 8) = val;
    }
    for (int i = threadIdx.x; i < 27 * kc; i += kVoThreads) {   // w is [3][3][3][Cin]: (o, dy, dx) = i / kc
      const int ot = i / kc, c = i - ot * kc;
      wsm[ot * kVoChunk + c] = __bfloat162float(w[(size_t)ot * Cin + c0 + c]);
    }
    __syncthreads();
#pragma unroll 1
    for (int tap = 0; tap < 9; ++tap) {
      const int dy = tap / 3, dx = tap - dy * 3;
      const __nv_bfloat16* px = tile + ((ty + dy) * kVoHw + tx + dx) * kVoPitch;
      const float* w0 = wsm + tap * kVoChunk;
      for (int v = 0; v < vecs; ++v) {
        const uint4 raw = *reinterpret_cast<const uint4*>(px + v * 8);
        const __nv_bfloat162* h2 = reinterpret_cast<const __nv_bfloat162*>(&raw);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 hf = __bfloat1622float2(h2[j]);
          const int c = v * 8 + 2 * j;
#pragma unroll
          for (int o = 0; o < 3; ++o) {
            acc[o] = fmaf(hf.x, w0[o * 9 * kVoChunk + c], acc[o]);
            acc[o] = fmaf(hf.y, w0[o * 9 * kVoChunk + c + 1], acc[o]);
          }
        }
      }
    }
  }
  const int gy = y0 + ty, gx = x0 + tx;
  if (gy >= H || gx >= W) return;
  const size_t p = ((size_t)b * H + gy) * W + gx;
#pragma unroll
  for (int o = 0; o < 3; ++o) {
    const float y = __fadd_rn(acc[o], bias[o]);
    if (out_f32) out_f32[p * 3 + o] = y;
    out_u8[p * 3 + o] = vae_out_u8(y);
  }
}

}  // namespace pxa

extern "C" int pxa_vae_out_u8(const PxaVaeOutArgs* args, void* stream) {
  using namespace pxa;
  if (!args) return fail(PXA_ERR_ARG, "null args");
  const PxaVaeOutArgs& a = *args;
  if (!a.x || !a.w || !a.bias || !a.out_u8) return fail(PXA_ERR_ARG, "null pointer");
  if (a.B <= 0 || a.H <= 0 || a.W <= 0) return fail(PXA_ERR_ARG, "B, H, W must be positive (B=%d H=%d W=%d)", a.B, a.H, a.W);
  if (a.B > 65535 || (a.H + kVoTh - 1) / kVoTh > 65535) return fail(PXA_ERR_ARG, "B <= 65535 and H <= %d required", 65535 * kVoTh);
  if (a.Cin <= 0 || a.Cin % 8) return fail(PXA_ERR_ARG, "Cin must be a positive multiple of 8 (Cin=%d)", a.Cin);
  if (a.x_sw < a.Cin || a.x_sh < (long long)a.W * a.x_sw || a.x_sb < (long long)a.H * a.x_sh)
    return fail(PXA_ERR_ARG, "x strides overlap (sb=%lld sh=%lld sw=%lld)", (long long)a.x_sb, (long long)a.x_sh, (long long)a.x_sw);
  if ((reinterpret_cast<uintptr_t>(a.x) & 15) || ((a.x_sw | a.x_sh | a.x_sb) & 7))
    return fail(PXA_ERR_ALIGN, "x must be 16-byte aligned and its strides multiples of 8 elements");
  if ((reinterpret_cast<uintptr_t>(a.w) & 1) || (reinterpret_cast<uintptr_t>(a.bias) & 3) || (reinterpret_cast<uintptr_t>(a.out_f32) & 3))
    return fail(PXA_ERR_ALIGN, "w / bias / out_f32 must be aligned to their element size");
  PXA_REQUIRE_SM90();
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const dim3 grid((a.W + kVoTw - 1) / kVoTw, (a.H + kVoTh - 1) / kVoTh, a.B);
  vae_out_u8_kernel<<<grid, kVoThreads, 0, st>>>(reinterpret_cast<const __nv_bfloat16*>(a.x), reinterpret_cast<const __nv_bfloat16*>(a.w),
                                                 a.bias, a.out_u8, a.out_f32, a.x_sb, a.x_sh, a.x_sw, a.H, a.W, a.Cin);
  launch_counter()++;
  PXA_CHECK_CUDA(cudaGetLastError());
  return PXA_OK;
}
