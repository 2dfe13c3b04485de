// DoRA kernels (include/pixart_sm100.h): the per-row weight norm of an adapted projection and the magnitude backward.
//
//   dora_norm    wn[n] = ||W[n,:] + (b a)[n,:]||_2, c[n] = m[n] / wn[n].  A CTA owns 32 rows of one item; per 64-column slice of K
//                it stages a [T, 64] (fp32) next to b^T [T, 32] of its rows; each warp owns 4 rows and each lane 2 columns, so one
//                t step is one 8-byte load of a, one broadcast 16-byte load of the warp's 4 b values and 8 FMAs.
//                Work N K T FMA per item, bytes N K 2 (W) + the small adapter operands: bandwidth-bound on W.
//   dora_bwd     dz = bf16(c g), per-chunk partial sums of g (y - bias) (pass 1, one read of g and y, one write of dz) and their
//                ordered sum over chunks, divided by m (pass 2, added into dm).  Bytes 3 M N 2.
#include "host_common.cuh"
#include "ptx.cuh"

namespace pxa {

constexpr int kNormRows = 32;       // rows of W per CTA
constexpr int kNormKc = 64;         // columns of K per smem slice
constexpr int kNormMaxItems = 64;   // items per launch (kernel parameter space)
constexpr int kNormMaxT = 256;

struct DoraNormBatch {
  PxaDoraNormItem it[kNormMaxItems];
};

__global__ void __launch_bounds__(256) dora_norm_kernel(const __grid_constant__ DoraNormBatch batch, int N, int K, int T) {
  extern __shared__ float norm_smem[];
  float* sa = norm_smem;                          // [T][kNormKc]
  float* sb = norm_smem + T * kNormKc;            // [T][kNormRows]: b^T of the CTA's rows
  const PxaDoraNormItem& item = batch.it[blockIdx.y];
  const __nv_bfloat16* W = reinterpret_cast<const __nv_bfloat16*>(item.w);
  const __nv_bfloat16* A = reinterpret_cast<const __nv_bfloat16*>(item.a);
  const __nv_bfloat16* Bm = reinterpret_cast<const __nv_bfloat16*>(item.b);
  const int n0 = blockIdx.x * kNormRows;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int i = threadIdx.x; i < kNormRows * T; i += blockDim.x) {
    const int r = i / T, t = i - r * T;
    sb[t * kNormRows + r] = n0 + r < N ? __bfloat162float(Bm[(size_t)(n0 + r) * T + t]) : 0.f;
  }
  float ss[4] = {0.f, 0.f, 0.f, 0.f};
  for (int k0 = 0; k0 < K; k0 += kNormKc) {
    __syncthreads();
    for (int i = threadIdx.x; i < T * (kNormKc / 2); i += blockDim.x) {
      const int t = i / (kNormKc / 2), kk = 2 * (i - t * (kNormKc / 2));
      float2 v = make_float2(0.f, 0.f);
      if (k0 + kk < K) {
        const uint32_t u = *reinterpret_cast<const uint32_t*>(A + (size_t)t * K + k0 + kk);
        v = make_float2(bf16_lo(u), bf16_hi(u));
      }
      *reinterpret_cast<float2*>(sa + t * kNormKc + kk) = v;
    }
    __syncthreads();
    const int k = k0 + 2 * lane;
    if (k >= K) continue;
    float d0[4] = {0.f, 0.f, 0.f, 0.f}, d1[4] = {0.f, 0.f, 0.f, 0.f};
    for (int t = 0; t < T; ++t) {
      const float2 av = *reinterpret_cast<const float2*>(sa + t * kNormKc + 2 * lane);
      const float4 bv = *reinterpret_cast<const float4*>(sb + t * kNormRows + 4 * warp);
      const float bb[4] = {bv.x, bv.y, bv.z, bv.w};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        d0[i] = fmaf(bb[i], av.x, d0[i]);
        d1[i] = fmaf(bb[i], av.y, d1[i]);
      }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int r = 4 * warp + i;
      if (n0 + r >= N) continue;
      const uint32_t u = *reinterpret_cast<const uint32_t*>(W + (size_t)(n0 + r) * K + k);
      const float e0 = bf16_lo(u) + d0[i], e1 = bf16_hi(u) + d1[i];
      ss[i] = fmaf(e0, e0, fmaf(e1, e1, ss[i]));
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float v = ss[i];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    const int n = n0 + 4 * warp + i;
    if (lane == 0 && n < N) {
      const float wn = sqrtf(v);
      if (item.wn) item.wn[n] = wn;
      if (item.c) item.c[n] = item.m[n] / wn;
    }
  }
}

// pass 1: CTA = 256 columns (32 lanes x 8) x PXA_DORA_BWD_ROWS rows (8 row lanes); partial[chunk][col] = sum over the chunk
__global__ void __launch_bounds__(256) dora_bwd_partial_kernel(const __nv_bfloat16* g, const __nv_bfloat16* __restrict__ y,
                                                              const __nv_bfloat16* __restrict__ bias, const float* __restrict__ c,
                                                              __nv_bfloat16* dz, float* __restrict__ partial, int M, int N,
                                                              long long ldg, long long ldy, long long ldz) {
  __shared__ float part[8][256 + 8];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int col = (blockIdx.x * 32 + tx) * 8;
  const int r0 = blockIdx.y * PXA_DORA_BWD_ROWS;
  const int r1 = min(r0 + PXA_DORA_BWD_ROWS, M);
  float acc[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = 0.f;
  if (col < N) {
    float cs[8], bs[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      cs[j] = __ldg(c + col + j);
      bs[j] = bias ? __bfloat162float(bias[col + j]) : 0.f;
    }
    for (int r = r0 + ty; r < r1; r += 8) {
      const uint4 gu = *reinterpret_cast<const uint4*>(g + (size_t)r * ldg + col);
      const uint4 yu = *reinterpret_cast<const uint4*>(y + (size_t)r * ldy + col);
      const uint32_t gw[4] = {gu.x, gu.y, gu.z, gu.w}, yw[4] = {yu.x, yu.y, yu.z, yu.w};
      uint32_t o[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float g0 = bf16_lo(gw[j]), g1 = bf16_hi(gw[j]);
        acc[2 * j] = fmaf(g0, bf16_lo(yw[j]) - bs[2 * j], acc[2 * j]);
        acc[2 * j + 1] = fmaf(g1, bf16_hi(yw[j]) - bs[2 * j + 1], acc[2 * j + 1]);
        o[j] = pack_bf16x2(cs[2 * j] * g0, cs[2 * j + 1] * g1);
      }
      *reinterpret_cast<uint4*>(dz + (size_t)r * ldz + col) = make_uint4(o[0], o[1], o[2], o[3]);
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) part[ty][tx * 8 + j] = acc[j];
  __syncthreads();
  const int gcol = blockIdx.x * 256 + threadIdx.x;
  if (gcol < N) {
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) s += part[j][threadIdx.x];
    partial[(size_t)blockIdx.y * N + gcol] = s;
  }
}

// pass 2: dm[n] += (sum over chunks, in chunk order) / m[n]
__global__ void __launch_bounds__(256) dora_bwd_final_kernel(const float* __restrict__ partial, const float* __restrict__ m,
                                                            float* __restrict__ dm, int chunks, int N) {
  const int n = blockIdx.x * 256 + threadIdx.x;
  if (n >= N) return;
  float s = 0.f;
  for (int i = 0; i < chunks; ++i) s += partial[(size_t)i * N + n];
  dm[n] += s / m[n];
}

}  // namespace pxa

extern "C" int pxa_dora_norm(const PxaDoraNormArgs* args, void* stream) {
  using namespace pxa;
  if (!args) return fail(PXA_ERR_ARG, "null args");
  const PxaDoraNormArgs& a = *args;
  if (a.n_items <= 0) return PXA_OK;
  if (!a.items) return fail(PXA_ERR_ARG, "null items");
  if (a.N <= 0 || a.K <= 0 || (a.N & 7) || (a.K & 7)) return fail(PXA_ERR_ARG, "N, K must be positive multiples of 8 (N=%d K=%d)", a.N, a.K);
  if (a.T <= 0 || (a.T & 7) || a.T > kNormMaxT) return fail(PXA_ERR_ARG, "T must be a multiple of 8 in [8, %d] (got %d)", kNormMaxT, a.T);
  for (int i = 0; i < a.n_items; ++i) {
    const PxaDoraNormItem& it = a.items[i];
    if (!it.w || !it.a || !it.b) return fail(PXA_ERR_ARG, "item %d: null w / a / b", i);
    if (it.c && !it.m) return fail(PXA_ERR_ARG, "item %d: c needs m", i);
    if ((reinterpret_cast<uintptr_t>(it.w) | reinterpret_cast<uintptr_t>(it.a) | reinterpret_cast<uintptr_t>(it.b)) & 3)
      return fail(PXA_ERR_ALIGN, "item %d: w / a / b must be 4-byte aligned", i);
  }
  PXA_REQUIRE_SM90();
  const int smem = (a.T * kNormKc + a.T * kNormRows) * (int)sizeof(float);
  PXA_CHECK_CUDA(cudaFuncSetAttribute(dora_norm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  for (int i0 = 0; i0 < a.n_items; i0 += kNormMaxItems) {
    const int n = a.n_items - i0 < kNormMaxItems ? a.n_items - i0 : kNormMaxItems;
    DoraNormBatch b = {};
    for (int i = 0; i < n; ++i) b.it[i] = a.items[i0 + i];
    dora_norm_kernel<<<dim3((a.N + kNormRows - 1) / kNormRows, n), 256, smem, s>>>(b, a.N, a.K, a.T);
    launch_counter()++;
    PXA_CHECK_CUDA(cudaGetLastError());
  }
  return PXA_OK;
}

extern "C" int pxa_dora_bwd(const PxaDoraBwdArgs* args, void* stream) {
  using namespace pxa;
  if (!args) return fail(PXA_ERR_ARG, "null args");
  const PxaDoraBwdArgs& a = *args;
  if (!a.g || !a.y || !a.c || !a.m || !a.dz || !a.dm || !a.partials) return fail(PXA_ERR_ARG, "null g / y / c / m / dz / dm / partials");
  if (a.M <= 0 || a.N <= 0 || (a.N & 7)) return fail(PXA_ERR_ARG, "bad shape M=%d N=%d (N must be a multiple of 8)", a.M, a.N);
  if ((a.ldg & 7) || (a.ldy & 7) || (a.ldz & 7) || a.ldg < a.N || a.ldy < a.N || a.ldz < a.N)
    return fail(PXA_ERR_ALIGN, "ldg / ldy / ldz must be multiples of 8 and >= N");
  if ((reinterpret_cast<uintptr_t>(a.g) | reinterpret_cast<uintptr_t>(a.y) | reinterpret_cast<uintptr_t>(a.dz)) & 15)
    return fail(PXA_ERR_ALIGN, "g / y / dz must be 16-byte aligned");
  if (a.dz == a.g && a.ldz != a.ldg) return fail(PXA_ERR_ARG, "dz aliases g with a different row stride");
  PXA_REQUIRE_SM90();
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const int chunks = (a.M + PXA_DORA_BWD_ROWS - 1) / PXA_DORA_BWD_ROWS;
  const int cblocks = (a.N + 255) / 256;
  dora_bwd_partial_kernel<<<dim3(cblocks, chunks), 256, 0, s>>>(
      reinterpret_cast<const __nv_bfloat16*>(a.g), reinterpret_cast<const __nv_bfloat16*>(a.y),
      reinterpret_cast<const __nv_bfloat16*>(a.bias), a.c, reinterpret_cast<__nv_bfloat16*>(a.dz), a.partials, a.M, a.N, a.ldg,
      a.ldy, a.ldz);
  launch_counter()++;
  PXA_CHECK_CUDA(cudaGetLastError());
  dora_bwd_final_kernel<<<cblocks, 256, 0, s>>>(a.partials, a.m, a.dm, chunks, a.N);
  launch_counter()++;
  PXA_CHECK_CUDA(cudaGetLastError());
  return PXA_OK;
}
