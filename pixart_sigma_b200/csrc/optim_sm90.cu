// Training-side optimizer kernels on the flat gradient buckets: gradient-norm clipping (pxa_grad_clip_flat) and the CAME
// step (pxa_came_flat) of the PixArt-Sigma configs.  Both are HBM-bound and deterministic: partial sums go to caller-owned
// workspace and are reduced in a fixed order, never with floating-point atomics.
#include <cuda_runtime.h>
#include <math.h>

#include "host_common.cuh"

namespace pxa {

constexpr int kOptThreads = 256;
constexpr int kOptWarps = kOptThreads / 32;

// Deterministic block sum (fixed shuffle tree, then warp partials in warp order); every thread receives the result.
__device__ __forceinline__ float block_sum(float v, float* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();  // `red` may still be read by a previous call
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float s = 0.f;
#pragma unroll
  for (int w = 0; w < kOptWarps; ++w) s += red[w];
  return s;
}

// ------------------------------------------------------------------------------------------------- gradient clipping
struct ClipBuckets {
  float* ptr[PXA_GRAD_CLIP_MAX_BUCKETS];
  long long n[PXA_GRAD_CLIP_MAX_BUCKETS];
  int count;
};

__global__ void __launch_bounds__(kOptThreads) grad_sumsq_kernel(const ClipBuckets b, float scale, float* __restrict__ partials) {
  __shared__ float red[kOptWarps];
  const long long stride = (long long)gridDim.x * kOptThreads;
  const long long first = (long long)blockIdx.x * kOptThreads + threadIdx.x;
  float acc = 0.f;
  for (int k = 0; k < b.count; ++k) {
    const float4* p4 = reinterpret_cast<const float4*>(b.ptr[k]);
    const long long n4 = b.n[k] >> 2;
    for (long long i = first; i < n4; i += stride) {
      const float4 v = p4[i];
      const float x = v.x * scale, y = v.y * scale, z = v.z * scale, w = v.w * scale;
      acc = fmaf(x, x, acc); acc = fmaf(y, y, acc); acc = fmaf(z, z, acc); acc = fmaf(w, w, acc);
    }
    const long long tail = (n4 << 2) + first;
    if (tail < b.n[k]) {
      const float x = b.ptr[k][tail] * scale;
      acc = fmaf(x, x, acc);
    }
  }
  const float s = block_sum(acc, red);
  if (threadIdx.x == 0) partials[blockIdx.x] = s;
}

__global__ void __launch_bounds__(kOptThreads) grad_clip_scale_kernel(const ClipBuckets b, float scale, float max_norm,
                                                                   const float* __restrict__ partials, float* __restrict__ total_norm) {
  __shared__ float red[kOptWarps];
  float acc = 0.f;
  for (int i = threadIdx.x; i < PXA_GRAD_CLIP_PARTS; i += kOptThreads) acc += partials[i];
  const float total = sqrtf(block_sum(acc, red));
  const float coef = fminf(max_norm / (total + 1e-6f), 1.0f);
  if (blockIdx.x == 0 && threadIdx.x == 0) *total_norm = total;
  const long long stride = (long long)gridDim.x * kOptThreads;
  const long long first = (long long)blockIdx.x * kOptThreads + threadIdx.x;
  for (int k = 0; k < b.count; ++k) {
    float4* p4 = reinterpret_cast<float4*>(b.ptr[k]);
    const long long n4 = b.n[k] >> 2;
    for (long long i = first; i < n4; i += stride) {
      float4 v = p4[i];
      v.x = (v.x * scale) * coef; v.y = (v.y * scale) * coef; v.z = (v.z * scale) * coef; v.w = (v.w * scale) * coef;
      p4[i] = v;
    }
    const long long tail = (n4 << 2) + first;
    if (tail < b.n[k]) b.ptr[k][tail] = (b.ptr[k][tail] * scale) * coef;
  }
}

// ------------------------------------------------------------------------------------------------- CAME
// Tiles: kind 0 = 1-D parameter, kVecTile consecutive elements; kind 1 = matrices of at most 4 x 4, kSmallTile whole matrices
// (one per thread); kind 2 = larger matrices, kTR x kTC blocks (warp w: rows w, w + 8, ...; lane: columns lane + 32 q).
constexpr int kVecTile = 2048;
constexpr int kSmallTile = kOptThreads;
constexpr int kSmallMax = 4;
constexpr int kTR = 128, kTC = 128, kColsPerLane = kTC / 32, kRowsPerWarp = kTR / kOptWarps;

struct CameGeom {
  int kind;
  long long rowtiles, coltiles;  // kind 2
  long long tiles, fin, ws;      // tiles, finalisation items (one per matrix, kind 2), workspace floats
};

__host__ __device__ inline CameGeom came_geom(const PxaCameParam& e) {
  CameGeom g{};
  if (!e.factored) {
    g.kind = 0;
    g.tiles = (e.numel + kVecTile - 1) / kVecTile;
    g.ws = g.tiles;
  } else if (e.R <= kSmallMax && e.C <= kSmallMax) {
    g.kind = 1;
    g.tiles = ((long long)e.lead + kSmallTile - 1) / kSmallTile;
    g.ws = g.tiles;
  } else {
    g.kind = 2;
    g.rowtiles = (e.R + kTR - 1) / kTR;
    g.coltiles = (e.C + kTC - 1) / kTC;
    g.tiles = (long long)e.lead * g.rowtiles * g.coltiles;
    g.fin = e.lead;
    // [tile sums: tiles][row partials: coltiles x lead*R][column partials: lead*rowtiles x C][row means: 2 x lead]
    g.ws = g.tiles + g.coltiles * e.lead * e.R + (long long)e.lead * g.rowtiles * e.C + 2LL * e.lead;
  }
  return g;
}

struct CameHyper {
  float eps1, eps2, clip, b1, omb1, b2, omb2, b3, omb3, wd;
};

// Entry whose [begin, next begin) range holds `item` (entries are planned in order, so the begins are non-decreasing).
template <bool kFin>
__device__ __forceinline__ int find_entry(const PxaCameParam* __restrict__ t, int n, long long item) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    const long long b = kFin ? t[mid].fin_begin : t[mid].tile_begin;
    if (b <= item) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// The clip divisor max(RMS(u) / clip_threshold, 1) from the parameter's per-tile sums of u^2 (same order in every CTA).
__device__ __forceinline__ float clip_divisor(const float* __restrict__ tile_sums, long long tiles, long long numel, float clip,
                                              float* red) {
  float acc = 0.f;
  for (long long i = threadIdx.x; i < tiles; i += kOptThreads) acc += tile_sums[i];
  const float s = block_sum(acc, red);
  return fmaxf(sqrtf(s) / (float)sqrt((double)numel) / clip, 1.0f);
}

// Phases (one launch each): 0 = second-moment sums (1-D / small: EMA, u and sum u^2 complete), 1 = sum u^2 (kind 2),
// 2 = clip divisor, exp_avg, instability sums (small: EMA complete), 3 = parameter update + sum p^2.
template <int kPhase>
__global__ void __launch_bounds__(kOptThreads, 2) came_tile_kernel(PxaCameArgs a, CameHyper h) {
  __shared__ float red[kOptWarps];
  __shared__ float colbuf[kOptWarps][kTC];
  const long long tile = blockIdx.x;
  const PxaCameParam e = a.table[find_entry<false>(a.table, a.n_entries, tile)];
  const CameGeom G = came_geom(e);
  const long long t = tile - e.tile_begin;
  float* ws = reinterpret_cast<float*>(a.workspace) + e.ws_off;
  float* tile_sums = ws;
  const int tid = threadIdx.x;
  const float lr = (kPhase == 3) ? *a.lr : 0.f;
  const float decay = -h.wd * lr;

  if (G.kind == 0) {
    if (kPhase == 1) return;
    const long long base = t * kVecTile;
    float* v = a.exp_avg_sq + e.sq_off;
    float div = 1.f;
    if (kPhase == 2) div = clip_divisor(tile_sums, G.tiles, e.numel, h.clip, red);
    float acc = 0.f;
#pragma unroll 4
    for (int k = 0; k < kVecTile / kOptThreads; ++k) {
      const long long i = base + tid + k * kOptThreads;
      if (i >= e.numel) break;
      if (kPhase == 0) {
        const float g = e.grad[i];
        const float vv = v[i] * h.b2 + h.omb2 * (g * g + h.eps1);
        v[i] = vv;
        const float u = rsqrtf(vv) * g;
        acc = fmaf(u, u, acc);
      } else if (kPhase == 2) {
        const float u = (rsqrtf(v[i]) * e.grad[i]) / div;
        e.exp_avg[i] = e.exp_avg[i] * h.b1 + h.omb1 * u;
      } else {
        const float p = e.param[i];
        acc = fmaf(p, p, acc);
        float q = p;
        if (h.wd != 0.f) q = q + decay * q;
        e.param[i] = q - e.exp_avg[i] * lr;
      }
    }
    if (kPhase != 2) {
      const float s = block_sum(acc, red);
      if (tid == 0) tile_sums[t] = s;
    }
    return;
  }

  if (G.kind == 1) {
    if (kPhase == 1) return;
    const int R = e.R, Cc = e.C, RC = R * Cc;
    const long long mat = t * kSmallTile + tid;
    float div = 1.f;
    if (kPhase == 2) div = clip_divisor(tile_sums, G.tiles, e.numel, h.clip, red);
    float acc = 0.f;
    if (mat < e.lead) {
      float* row = (kPhase == 3 ? a.res_row : a.sq_row) + e.sq_off + mat * R;
      float* col = (kPhase == 3 ? a.res_col : a.sq_col) + e.col_off + mat * Cc;
      const long long off = mat * RC;
      float x[kSmallMax][kSmallMax], rf[kSmallMax], cf[kSmallMax], rowv[kSmallMax], colv[kSmallMax];
#pragma unroll
      for (int r = 0; r < kSmallMax; ++r) rowv[r] = r < R ? row[r] : 1.f;
#pragma unroll
      for (int c = 0; c < kSmallMax; ++c) colv[c] = c < Cc ? col[c] : 1.f;
      if (kPhase == 0) {
#pragma unroll
        for (int r = 0; r < kSmallMax; ++r)
#pragma unroll
          for (int c = 0; c < kSmallMax; ++c)
            if (r < R && c < Cc) { const float g = e.grad[off + r * Cc + c]; x[r][c] = g * g + h.eps1; }
        // EMAs of the row / column means of u = g^2 + eps1
#pragma unroll
        for (int r = 0; r < kSmallMax; ++r)
          if (r < R) {
            float s = 0.f;
#pragma unroll
            for (int c = 0; c < kSmallMax; ++c) if (c < Cc) s += x[r][c];
            rowv[r] = rowv[r] * h.b2 + h.omb2 * (s / (float)Cc);
            row[r] = rowv[r];
          }
#pragma unroll
        for (int c = 0; c < kSmallMax; ++c)
          if (c < Cc) {
            float s = 0.f;
#pragma unroll
            for (int r = 0; r < kSmallMax; ++r) if (r < R) s += x[r][c];
            colv[c] = colv[c] * h.b2 + h.omb2 * (s / (float)R);
            col[c] = colv[c];
          }
      }
      // r / c factors of the (updated) statistics: rsqrt(row / mean(row)), rsqrt(col)
      float rm = 0.f;
#pragma unroll
      for (int r = 0; r < kSmallMax; ++r) if (r < R) rm += rowv[r];
      rm = rm / (float)R;
#pragma unroll
      for (int r = 0; r < kSmallMax; ++r) rf[r] = r < R ? rsqrtf(rowv[r] / rm) : 0.f;
#pragma unroll
      for (int c = 0; c < kSmallMax; ++c) cf[c] = c < Cc ? rsqrtf(colv[c]) : 0.f;
      if (kPhase == 0) {
#pragma unroll
        for (int r = 0; r < kSmallMax; ++r)
#pragma unroll
          for (int c = 0; c < kSmallMax; ++c)
            if (r < R && c < Cc) { const float u = (rf[r] * cf[c]) * e.grad[off + r * Cc + c]; acc = fmaf(u, u, acc); }
      } else if (kPhase == 2) {
#pragma unroll
        for (int r = 0; r < kSmallMax; ++r)
#pragma unroll
          for (int c = 0; c < kSmallMax; ++c)
            if (r < R && c < Cc) {
              const long long i = off + r * Cc + c;
              const float u = ((rf[r] * cf[c]) * e.grad[i]) / div;
              const float m = e.exp_avg[i] * h.b1 + h.omb1 * u;
              e.exp_avg[i] = m;
              const float d = u - m;
              x[r][c] = d * d + h.eps2;
            }
        float* rrow = a.res_row + e.sq_off + mat * R;
        float* rcol = a.res_col + e.col_off + mat * Cc;
#pragma unroll
        for (int r = 0; r < kSmallMax; ++r)
          if (r < R) {
            float s = 0.f;
#pragma unroll
            for (int c = 0; c < kSmallMax; ++c) if (c < Cc) s += x[r][c];
            rrow[r] = rrow[r] * h.b3 + h.omb3 * (s / (float)Cc);
          }
#pragma unroll
        for (int c = 0; c < kSmallMax; ++c)
          if (c < Cc) {
            float s = 0.f;
#pragma unroll
            for (int r = 0; r < kSmallMax; ++r) if (r < R) s += x[r][c];
            rcol[c] = rcol[c] * h.b3 + h.omb3 * (s / (float)R);
          }
      } else {  // kPhase == 3: row / col are the instability statistics here
#pragma unroll
        for (int r = 0; r < kSmallMax; ++r)
#pragma unroll
          for (int c = 0; c < kSmallMax; ++c)
            if (r < R && c < Cc) {
              const long long i = off + r * Cc + c;
              const float p = e.param[i];
              acc = fmaf(p, p, acc);
              float q = p;
              if (h.wd != 0.f) q = q + decay * q;
              e.param[i] = q - ((rf[r] * cf[c]) * e.exp_avg[i]) * lr;
            }
      }
    }
    if (kPhase != 2) {
      const float s = block_sum(acc, red);
      if (tid == 0) tile_sums[t] = s;
    }
    return;
  }

  // kind 2: a kTR x kTC block of matrix `mat`
  const int R = e.R, Cc = e.C;
  const long long per_mat = G.rowtiles * G.coltiles;
  const long long mat = t / per_mat;
  const int rt = (int)((t % per_mat) / G.coltiles), ct = (int)(t % G.coltiles);
  const int warp = tid >> 5, lane = tid & 31;
  const int r0 = rt * kTR, c0 = ct * kTC;
  float* row_part = ws + G.tiles;                                   // [coltiles][lead * R]
  float* col_part = row_part + G.coltiles * e.lead * R;             // [lead * rowtiles][C]
  const float* rmean = col_part + (long long)e.lead * G.rowtiles * Cc;   // [2][lead]
  const float* srow = (kPhase == 3 ? a.res_row : a.sq_row) + e.sq_off + mat * R;
  const float* scol = (kPhase == 3 ? a.res_col : a.sq_col) + e.col_off + mat * Cc;
  const float rm = kPhase == 0 ? 0.f : rmean[(kPhase == 3 ? e.lead : 0) + mat];
  float div = 1.f;
  if (kPhase == 2) div = clip_divisor(tile_sums, G.tiles, e.numel, h.clip, red);
  float cf[kColsPerLane], colacc[kColsPerLane];
#pragma unroll
  for (int q = 0; q < kColsPerLane; ++q) {
    const int c = c0 + lane + 32 * q;
    cf[q] = (kPhase != 0 && c < Cc) ? rsqrtf(scol[c]) : 0.f;
    colacc[q] = 0.f;
  }
  float acc = 0.f;
#pragma unroll 2
  for (int j = 0; j < kRowsPerWarp; ++j) {
    const int r = r0 + warp + kOptWarps * j;
    if (r >= R) break;
    const long long rowbase = (mat * R + r) * Cc;
    const float rf = kPhase == 0 ? 0.f : rsqrtf(srow[r] / rm);
    float racc = 0.f;
#pragma unroll
    for (int q = 0; q < kColsPerLane; ++q) {
      const int c = c0 + lane + 32 * q;
      if (c < Cc) {
        const long long i = rowbase + c;
        if (kPhase == 0) {
          const float g = e.grad[i];
          const float x = g * g + h.eps1;
          racc += x;
          colacc[q] += x;
        } else if (kPhase == 1) {
          const float u = (rf * cf[q]) * e.grad[i];
          acc = fmaf(u, u, acc);
        } else if (kPhase == 2) {
          const float u = ((rf * cf[q]) * e.grad[i]) / div;
          const float m = e.exp_avg[i] * h.b1 + h.omb1 * u;
          e.exp_avg[i] = m;
          const float d = u - m;
          const float x = d * d + h.eps2;
          racc += x;
          colacc[q] += x;
        } else {
          const float p = e.param[i];
          acc = fmaf(p, p, acc);
          float pq = p;
          if (h.wd != 0.f) pq = pq + decay * pq;
          e.param[i] = pq - ((rf * cf[q]) * e.exp_avg[i]) * lr;
        }
      }
    }
    if (kPhase == 0 || kPhase == 2) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) racc += __shfl_xor_sync(0xffffffffu, racc, o);
      if (lane == 0) row_part[(long long)ct * e.lead * R + mat * R + r] = racc;
    }
  }
  if (kPhase == 0 || kPhase == 2) {
#pragma unroll
    for (int q = 0; q < kColsPerLane; ++q) colbuf[warp][lane + 32 * q] = colacc[q];
    __syncthreads();
    if (tid < kTC && c0 + tid < Cc) {
      float s = 0.f;
#pragma unroll
      for (int w = 0; w < kOptWarps; ++w) s += colbuf[w][tid];
      col_part[(mat * G.rowtiles + rt) * Cc + c0 + tid] = s;
    }
  } else {
    const float s = block_sum(acc, red);
    if (tid == 0) tile_sums[t] = s;
  }
}

// Finalisation of the factored statistics of one kind-2 matrix: the row / column EMAs from the partial sums (fixed order)
// and the mean of the updated row statistics.  kRes = 0: second moments (b2), 1: instability (b3).
template <int kRes>
__global__ void __launch_bounds__(kOptThreads) came_finalize_kernel(PxaCameArgs a, CameHyper h) {
  __shared__ float red[kOptWarps];
  const long long item = blockIdx.x;
  const PxaCameParam e = a.table[find_entry<true>(a.table, a.n_entries, item)];
  const CameGeom G = came_geom(e);
  const long long mat = item - e.fin_begin;
  float* ws = reinterpret_cast<float*>(a.workspace) + e.ws_off;
  const float* row_part = ws + G.tiles;
  const float* col_part = row_part + G.coltiles * e.lead * e.R;
  float* rmean = const_cast<float*>(col_part) + (long long)e.lead * G.rowtiles * e.C;
  float* row = (kRes ? a.res_row : a.sq_row) + e.sq_off + mat * e.R;
  float* col = (kRes ? a.res_col : a.sq_col) + e.col_off + mat * e.C;
  const float b = kRes ? h.b3 : h.b2, omb = kRes ? h.omb3 : h.omb2;
  float acc = 0.f;
  for (int r = threadIdx.x; r < e.R; r += kOptThreads) {
    float s = 0.f;
    for (long long ct = 0; ct < G.coltiles; ++ct) s += row_part[ct * e.lead * e.R + mat * e.R + r];
    const float v = row[r] * b + omb * (s / (float)e.C);
    row[r] = v;
    acc += v;
  }
  for (int c = threadIdx.x; c < e.C; c += kOptThreads) {
    float s = 0.f;
    for (long long rt = 0; rt < G.rowtiles; ++rt) s += col_part[(mat * G.rowtiles + rt) * e.C + c];
    col[c] = col[c] * b + omb * (s / (float)e.R);
  }
  const float s = block_sum(acc, red);
  if (threadIdx.x == 0) rmean[kRes * e.lead + mat] = s / (float)e.R;
}

// rms[e] = ||p before the update|| / sqrt(numel) from the per-tile sums of p^2 (one warp per parameter).
__global__ void __launch_bounds__(kOptThreads) came_rms_kernel(PxaCameArgs a) {
  const int entry = blockIdx.x * kOptWarps + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (entry >= a.n_entries) return;
  const PxaCameParam e = a.table[entry];
  const CameGeom G = came_geom(e);
  const float* tile_sums = reinterpret_cast<const float*>(a.workspace) + e.ws_off;
  float s = 0.f;
  for (long long i = lane; i < G.tiles; i += 32) s += tile_sums[i];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) a.rms[entry] = sqrtf(s) / (float)sqrt((double)e.numel);
}

inline bool misaligned16(const void* p) { return reinterpret_cast<uintptr_t>(p) & 15; }

}  // namespace pxa

extern "C" int pxa_grad_clip_flat(const PxaGradClipArgs* args, void* stream) {
  using namespace pxa;
  if (!args) return fail(PXA_ERR_ARG, "null args");
  const PxaGradClipArgs& a = *args;
  if (!a.buckets || !a.partials || !a.total_norm) return fail(PXA_ERR_ARG, "null pointer");
  if (a.n_buckets <= 0 || a.n_buckets > PXA_GRAD_CLIP_MAX_BUCKETS)
    return fail(PXA_ERR_ARG, "n_buckets must be in 1..%d (got %d)", PXA_GRAD_CLIP_MAX_BUCKETS, a.n_buckets);
  if (!(a.max_norm > 0.f)) return fail(PXA_ERR_ARG, "max_norm must be positive");
  if (misaligned16(a.partials) || (reinterpret_cast<uintptr_t>(a.total_norm) & 3))
    return fail(PXA_ERR_ALIGN, "partials must be 16-byte aligned, total_norm 4-byte");
  ClipBuckets b{};
  b.count = a.n_buckets;
  for (int k = 0; k < a.n_buckets; ++k) {
    if (!a.buckets[k].ptr || a.buckets[k].n <= 0) return fail(PXA_ERR_ARG, "bucket %d: null pointer or empty", k);
    if (misaligned16(a.buckets[k].ptr)) return fail(PXA_ERR_ALIGN, "bucket %d is not 16-byte aligned", k);
    b.ptr[k] = a.buckets[k].ptr;
    b.n[k] = a.buckets[k].n;
  }
  PXA_REQUIRE_SM90();
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  grad_sumsq_kernel<<<PXA_GRAD_CLIP_PARTS, kOptThreads, 0, s>>>(b, a.grad_scale, a.partials);
  launch_counter()++;
  PXA_CHECK_CUDA(cudaGetLastError());
  grad_clip_scale_kernel<<<PXA_GRAD_CLIP_PARTS, kOptThreads, 0, s>>>(b, a.grad_scale, a.max_norm, a.partials, a.total_norm);
  launch_counter()++;
  PXA_CHECK_CUDA(cudaGetLastError());
  return PXA_OK;
}

extern "C" int pxa_came_workspace_bytes(PxaCameArgs* args, PxaCameParam* t, int64_t* bytes) {
  using namespace pxa;
  if (!args || !t || !bytes) return fail(PXA_ERR_ARG, "null pointer");
  if (args->n_entries <= 0) return fail(PXA_ERR_ARG, "empty parameter table");
  long long tiles = 0, fin = 0, ws = 0;
  for (int i = 0; i < args->n_entries; ++i) {
    PxaCameParam& e = t[i];
    if (!e.param || !e.grad || !e.exp_avg) return fail(PXA_ERR_ARG, "entry %d: null pointer", i);
    if (e.lead <= 0 || e.R <= 0 || e.C <= 0 || e.numel != (int64_t)e.lead * e.R * e.C)
      return fail(PXA_ERR_ARG, "entry %d: numel %lld != lead %d x R %d x C %d", i, (long long)e.numel, e.lead, e.R, e.C);
    if (!e.factored && (e.lead != 1 || e.R != 1)) return fail(PXA_ERR_ARG, "entry %d: a 1-D entry has lead = R = 1", i);
    if (e.offset < 0 || e.offset + e.numel > e.bucket_numel)
      return fail(PXA_ERR_ARG, "entry %d: elements [%lld, %lld) overrun its bucket of %lld", i, (long long)e.offset,
                  (long long)(e.offset + e.numel), (long long)e.bucket_numel);
    if (e.factored) {
      if (e.sq_off < 0 || e.sq_off + (int64_t)e.lead * e.R > args->n_row || e.col_off < 0 ||
          e.col_off + (int64_t)e.lead * e.C > args->n_col)
        return fail(PXA_ERR_ARG, "entry %d: row / column statistics overrun n_row / n_col", i);
    } else if (e.sq_off < 0 || e.sq_off + e.numel > args->n_vec) {
      return fail(PXA_ERR_ARG, "entry %d: second moments overrun n_vec", i);
    }
    const CameGeom G = came_geom(e);
    e.tile_begin = tiles;
    e.fin_begin = fin;
    e.ws_off = ws;
    tiles += G.tiles;
    fin += G.fin;
    ws += (G.ws + 3) & ~3LL;
  }
  if (tiles > 0x7fffffffLL) return fail(PXA_ERR_ARG, "too many tiles (%lld)", tiles);
  args->n_tiles = tiles;
  args->n_fin = fin;
  args->ws_floats = ws;
  *bytes = ws * (int64_t)sizeof(float);
  return PXA_OK;
}

extern "C" int pxa_came_flat(const PxaCameArgs* args, void* stream) {
  using namespace pxa;
  if (!args) return fail(PXA_ERR_ARG, "null args");
  const PxaCameArgs& a = *args;
  if (!a.table || !a.rms || !a.lr || !a.workspace) return fail(PXA_ERR_ARG, "null pointer");
  if ((a.n_vec > 0 && !a.exp_avg_sq) || (a.n_row > 0 && (!a.sq_row || !a.res_row)) || (a.n_col > 0 && (!a.sq_col || !a.res_col)))
    return fail(PXA_ERR_ARG, "null state buffer");
  if (a.step <= 0) return fail(PXA_ERR_ARG, "step counts from 1");
  if (a.n_entries <= 0 || a.n_tiles <= 0) return fail(PXA_ERR_ARG, "no plan: call pxa_came_workspace_bytes first");
  if (a.workspace_bytes < a.ws_floats * (int64_t)sizeof(float))
    return fail(PXA_ERR_ARG, "workspace of %lld bytes, the plan needs %lld", (long long)a.workspace_bytes,
                (long long)(a.ws_floats * sizeof(float)));
  if (!(a.clip_threshold > 0.0)) return fail(PXA_ERR_ARG, "clip_threshold must be positive");
  if (misaligned16(a.table) || misaligned16(a.exp_avg_sq) || misaligned16(a.sq_row) || misaligned16(a.res_row) ||
      misaligned16(a.sq_col) || misaligned16(a.res_col) || misaligned16(a.rms) || misaligned16(a.workspace) ||
      (reinterpret_cast<uintptr_t>(a.lr) & 3))
    return fail(PXA_ERR_ALIGN, "table, state buffers, rms and workspace must be 16-byte aligned, lr 4-byte");
  PXA_REQUIRE_SM90();
  CameHyper h;
  h.eps1 = (float)a.eps1; h.eps2 = (float)a.eps2; h.clip = (float)a.clip_threshold;
  h.b1 = (float)a.beta1; h.omb1 = (float)(1.0 - a.beta1);
  h.b2 = (float)a.beta2; h.omb2 = (float)(1.0 - a.beta2);
  h.b3 = (float)a.beta3; h.omb3 = (float)(1.0 - a.beta3);
  h.wd = (float)a.weight_decay;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const unsigned tiles = (unsigned)a.n_tiles;
  came_tile_kernel<0><<<tiles, kOptThreads, 0, s>>>(a, h);
  launch_counter()++;
  PXA_CHECK_CUDA(cudaGetLastError());
  if (a.n_fin > 0) {
    came_finalize_kernel<0><<<(unsigned)a.n_fin, kOptThreads, 0, s>>>(a, h);
    launch_counter()++;
    PXA_CHECK_CUDA(cudaGetLastError());
  }
  came_tile_kernel<1><<<tiles, kOptThreads, 0, s>>>(a, h);
  launch_counter()++;
  PXA_CHECK_CUDA(cudaGetLastError());
  came_tile_kernel<2><<<tiles, kOptThreads, 0, s>>>(a, h);
  launch_counter()++;
  PXA_CHECK_CUDA(cudaGetLastError());
  if (a.n_fin > 0) {
    came_finalize_kernel<1><<<(unsigned)a.n_fin, kOptThreads, 0, s>>>(a, h);
    launch_counter()++;
    PXA_CHECK_CUDA(cudaGetLastError());
  }
  came_tile_kernel<3><<<tiles, kOptThreads, 0, s>>>(a, h);
  launch_counter()++;
  PXA_CHECK_CUDA(cudaGetLastError());
  came_rms_kernel<<<(unsigned)((a.n_entries + kOptWarps - 1) / kOptWarps), kOptThreads, 0, s>>>(a);
  launch_counter()++;
  PXA_CHECK_CUDA(cudaGetLastError());
  return PXA_OK;
}
