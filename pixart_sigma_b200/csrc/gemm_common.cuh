// Shared pieces of the wgmma GEMM kernel: parameters, shared-memory configuration and the epilogues.
#pragma once
#include "host_common.cuh"
#include "ptx.cuh"

namespace pxa {

constexpr int kBM = 128;
constexpr int kBK = 64;            // 64 bf16 = 128 B = one swizzle atom row
constexpr int kGemmThreads = 384;  // warp 0: TMA producer; warps 4-11: two consumer warpgroups (wgmma + epilogue)
constexpr int kEpiWarp0 = 4;       // first consumer warp
constexpr int kNumEpiThreads = 256;

struct GemmParams {
  const __nv_bfloat16* bias;
  void* out;
  __nv_bfloat16* out_aux;
  const void* residual;
  const float* gate;
  long long gate_batch_stride;
  int rows_per_batch;
  int row_base;         // row r of this call is row row_base + r of the batch (sample = (row_base + r) / rows_per_batch)
  int M, N, K, ldo;
  int num_m_tiles, num_n_tiles;
  int k_splits;         // > 1: split-K over tiles (reduce-add epilogue only)
  int aux_branch;       // residual epilogue: the bf16 aux output receives acc + bias (the branch output) instead of out
  int reverse_tiles;    // visit the tiles from the last row block to the first (L2 reuse of a just-written A operand)
  // fused LayerNorm-modulate, producer side (fp32 residual epilogue): aux = out * aux_scale[b], row partial sums of out
  const float* aux_scale;
  long long aux_scale_batch_stride;
  float* row_stats_out;
  // consumer side (PXA_EPI_LN_BIAS / _GELU): out = rstd * (acc - mu * u[b]) + v[b]
  const float* ln_stats;
  const float* ln_u;
  const float* ln_v;
  long long ln_uv_batch_stride;
  float ln_inv_dim, ln_eps;
  // implicit-GEMM 3x3 convolution mode (kConv): A is an NHWC image read through a 4-D tensor map
  int conv_H, conv_W, conv_tile_w, conv_tile_h, conv_cin_blocks;
  // widths that do not tile (neither a power of two <= 128 nor a multiple of 128): the M index runs over a VIRTUAL image of width
  // conv_Wp = W rounded up to 128 -- pixel columns >= W are TMA zero fill on the way in and are not stored on the way out
  int conv_Wp;
};

inline void fill_ln_params(GemmParams& p, const PxaGemmArgs& a) {
  p.aux_scale = a.aux_scale;
  p.aux_scale_batch_stride = a.aux_scale_batch_stride;
  p.row_stats_out = a.row_stats_out;
  p.ln_stats = a.ln_stats;
  p.ln_u = a.ln_u;
  p.ln_v = a.ln_v;
  p.ln_uv_batch_stride = a.ln_uv_batch_stride;
  p.ln_inv_dim = a.ln_dim > 0 ? 1.0f / (float)a.ln_dim : 0.f;
  p.ln_eps = a.ln_eps;
  p.reverse_tiles = a.reverse_tiles ? 1 : 0;
}


constexpr int kSmemBudget = 227 * 1024;

// Per-tile epilogue constants staged in smem while the tile's MMAs run: bias (fp32) and the gate rows of the (at most
// two) samples a 128-row tile can span.  Reading them per chunk is then an LDS broadcast instead of a chain of L2-latency
// global loads in the epilogue's critical path.  Double-buffered by tile parity.
struct EpiConst {
  float bias[256];     // LN consumer epilogue: v of the first sample
  float gate0[256];    // gate of the sample of the tile's first row (1.0 when there is no gate); LN consumer: v of the last sample
  float gate1[256];    // gate of the sample of the tile's last row
  float ex0[256];      // aux_scale of the first / last sample (1.0 when there is none); LN consumer: u of the first / last sample
  float ex1[256];
  int row_split;       // tile rows >= row_split belong to the second sample
  int pad[3];
};
constexpr int kEpiConstBytes = 2 * sizeof(EpiConst);    // 10272 B

// Shared memory of one CTA: the operand ring, one accumulator staging chunk per consumer warpgroup (128 rows x 32 fp32 columns:
// the wgmma fragments are re-read from it row per thread), the constants, the warpgroup-to-warpgroup row statistics and the
// barriers.  Each consumer warp's 4 KB transpose tile is the 32 staging rows that warp reads: it has them in registers before it
// writes the tile, and the named barrier at the top of the next chunk keeps the other warps' fragment stores behind it.  The
// 32 KB this saves is one more ring stage at BN 128 and 192 (5 and 4 stages).
template <int BN> struct GemmCfg {
  static constexpr int kStageA = kBM * kBK * 2;                 // 16 KB
  static constexpr int kStageB = BN * kBK * 2;
  static constexpr int kStage = kStageA + kStageB;
  static constexpr int kAccChunkBytes = 128 * 32 * 4;           // 16 KB per consumer warpgroup
  static constexpr int kEpiBufs = 2 * kAccChunkBytes;
  static constexpr int kStatBytes = 128 * 8;
  static constexpr int kEpiSmem = kEpiBufs + ((kEpiConstBytes + 127) / 128) * 128 + kStatBytes;
  static constexpr int kBarBytes = 256;
  static constexpr int kMaxStages = (kSmemBudget - kEpiSmem - kBarBytes - 1024) / kStage;
  static constexpr int kStages = kMaxStages > 6 ? 6 : kMaxStages;
  static constexpr int kSmem = kStages * kStage + kEpiSmem + kBarBytes + 1024;  // +1024 alignment slack
};

// ------------------------------------------------------------------------------------------------- epilogues
// Row-per-thread registers `v` hold acc for columns [col0, col0+32) of this thread's row.

// bf16 residual epilogue (EPI 2 of the VAE convolutions): fp32 acc transposed through smem (128 B per row), then in the coalesced
// layout out = residual + gate * (acc + bias); optional bf16 aux copy.
// In the coalesced layout lane l owns columns [4*(l&7), +4) of rows 4*it + (l>>3), it = 0..7.
// The residual fragment of a chunk is loaded before the chunk's transpose and stores (`residual` may alias `out`, so the compiler
// may not hoist the loads over the stores itself).
struct ResFrag {
  float4 r[8];
};

template <typename OutT>
PXA_DEVICE void load_residual_frag(ResFrag& f, const GemmParams& p, int lane, int row0, int col0, int m_limit = -1) {
  const int m_end = m_limit >= 0 ? m_limit : p.M;       // convolution with a virtual width: rows [row0, m_limit) exist
  const int gcol = col0 + (lane & 7) * 4;
  const bool col_ok = gcol < p.N;
#pragma unroll
  for (int it = 0; it < 8; ++it) {
    const int grow = row0 + it * 4 + (lane >> 3);
    f.r[it] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (grow < m_end && col_ok) {
      const size_t off = (size_t)grow * p.ldo + gcol;
      if constexpr (sizeof(OutT) == 4) {
        f.r[it] = *reinterpret_cast<const float4*>(reinterpret_cast<const float*>(p.residual) + off);
      } else {
        uint2 u = *reinterpret_cast<const uint2*>(reinterpret_cast<const __nv_bfloat16*>(p.residual) + off);
        f.r[it] = make_float4(bf16_lo(u.x), bf16_hi(u.x), bf16_lo(u.y), bf16_hi(u.y));
      }
    }
  }
}

template <typename OutT>
PXA_DEVICE void epilogue_chunk_residual(uint32_t (&v)[32], const ResFrag& res, const GemmParams& p, uint8_t* stile,
                                        int lane, int row0, int col0, int m_limit = -1) {
  const int m_end = m_limit >= 0 ? m_limit : p.M;
  // smem tile: 32 rows x 128 B; 16-byte chunk c of row r lives at r*128 + ((c ^ (r & 7)) * 16)
  {
    const int sw = lane & 7;
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      uint4 u = make_uint4(v[4 * c], v[4 * c + 1], v[4 * c + 2], v[4 * c + 3]);
      *reinterpret_cast<uint4*>(stile + lane * 128 + ((c ^ sw) << 4)) = u;
    }
  }
  __syncwarp();
  const int c = lane & 7;
  const int gcol = col0 + c * 4;
  const bool col_ok = gcol < p.N;
  float b0 = 0.f, b1 = 0.f, b2 = 0.f, b3 = 0.f;
  if (p.bias != nullptr && col_ok) {
    uint2 u = __ldg(reinterpret_cast<const uint2*>(p.bias + gcol));
    b0 = bf16_lo(u.x); b1 = bf16_hi(u.x); b2 = bf16_lo(u.y); b3 = bf16_hi(u.y);
  }
  // gate: all loads first (tiny table, L1/L2 resident), then compute + store
  float4 g[8];
#pragma unroll
  for (int it = 0; it < 8; ++it) {
    const int grow = row0 + it * 4 + (lane >> 3);
    g[it] = make_float4(1.f, 1.f, 1.f, 1.f);
    if (p.gate != nullptr && grow < m_end && col_ok) {
      const int bidx = (p.row_base + grow) / p.rows_per_batch;
      g[it] = __ldg(reinterpret_cast<const float4*>(p.gate + (size_t)bidx * p.gate_batch_stride + gcol));
    }
  }
#pragma unroll
  for (int it = 0; it < 8; ++it) {
    const int r = it * 4 + (lane >> 3);
    const int grow = row0 + r;
    const float4 a = *reinterpret_cast<const float4*>(stile + r * 128 + ((c ^ (r & 7)) << 4));
    if (grow < m_end && col_ok) {
      const size_t off = (size_t)grow * p.ldo + gcol;
      float4 o;
      const float4 yb = make_float4(a.x + b0, a.y + b1, a.z + b2, a.w + b3);     // the branch output
      o.x = fmaf(g[it].x, yb.x, res.r[it].x);
      o.y = fmaf(g[it].y, yb.y, res.r[it].y);
      o.z = fmaf(g[it].z, yb.z, res.r[it].z);
      o.w = fmaf(g[it].w, yb.w, res.r[it].w);
      if constexpr (sizeof(OutT) == 4) {
        *reinterpret_cast<float4*>(reinterpret_cast<float*>(p.out) + off) = o;
      } else {
        *reinterpret_cast<uint2*>(reinterpret_cast<__nv_bfloat16*>(p.out) + off) =
            make_uint2(pack_bf16x2(o.x, o.y), pack_bf16x2(o.z, o.w));
      }
      if (p.out_aux != nullptr) {
        const float4 ax = p.aux_branch ? yb : o;
        *reinterpret_cast<uint2*>(p.out_aux + off) = make_uint2(pack_bf16x2(ax.x, ax.y), pack_bf16x2(ax.z, ax.w));
      }
    }
  }
  __syncwarp();
}

// Per-tile constants in two phases so that their L2 latency hides behind the PREVIOUS tile's work: the 256
// consumer threads issue the global loads of tile i + 1 (load_epi_consts) right after tile i's barrier and park the values in
// registers; at the top of tile i + 1 they are stored to the tile's EpiConst buffer (store_epi_consts), followed by a named
// barrier.  (Loading and storing in one go would put one L2 round trip in front of every tile's epilogue.)
template <int BN> struct EpiRegs {
  static constexpr int kCols = (BN + kNumEpiThreads - 1) / kNumEpiThreads;
  float v[kCols][5];
  int row_split;
};

template <int BN, bool kLn = false>
PXA_DEVICE void load_epi_consts(EpiRegs<BN>& r, const GemmParams& p, int tid, int m0, int n0) {
  const int b0 = (p.row_base + m0) / p.rows_per_batch;
  const int last = (m0 + kBM - 1 < p.M ? m0 + kBM - 1 : p.M - 1);
  const int b1 = (p.row_base + last) / p.rows_per_batch;
#pragma unroll
  for (int i = 0; i < EpiRegs<BN>::kCols; ++i) {
    const int col = n0 + tid + i * kNumEpiThreads;
    const bool ok = col < p.N && tid + i * kNumEpiThreads < BN;
    if constexpr (kLn) {
      r.v[i][0] = ok ? __ldg(p.ln_v + (size_t)b0 * p.ln_uv_batch_stride + col) : 0.f;
      r.v[i][1] = ok ? __ldg(p.ln_v + (size_t)b1 * p.ln_uv_batch_stride + col) : 0.f;
      r.v[i][2] = 1.f;
      r.v[i][3] = ok ? __ldg(p.ln_u + (size_t)b0 * p.ln_uv_batch_stride + col) : 0.f;
      r.v[i][4] = ok ? __ldg(p.ln_u + (size_t)b1 * p.ln_uv_batch_stride + col) : 0.f;
    } else {
      r.v[i][0] = (ok && p.bias != nullptr) ? __bfloat162float(p.bias[col]) : 0.f;
      r.v[i][1] = (ok && p.gate != nullptr) ? __ldg(p.gate + (size_t)b0 * p.gate_batch_stride + col) : 1.f;
      r.v[i][2] = (ok && p.gate != nullptr) ? __ldg(p.gate + (size_t)b1 * p.gate_batch_stride + col) : 1.f;
      r.v[i][3] = (ok && p.aux_scale != nullptr) ? __ldg(p.aux_scale + (size_t)b0 * p.aux_scale_batch_stride + col) : 1.f;
      r.v[i][4] = (ok && p.aux_scale != nullptr) ? __ldg(p.aux_scale + (size_t)b1 * p.aux_scale_batch_stride + col) : 1.f;
    }
  }
  r.row_split = (b0 + 1) * p.rows_per_batch - (p.row_base + m0);
}

template <int BN>
PXA_DEVICE void store_epi_consts(EpiConst* cb, const EpiRegs<BN>& r, int tid) {
#pragma unroll
  for (int i = 0; i < EpiRegs<BN>::kCols; ++i) {
    const int c = tid + i * kNumEpiThreads;
    if (c < BN) {
      cb->bias[c] = r.v[i][0];
      cb->gate0[c] = r.v[i][1];
      cb->gate1[c] = r.v[i][2];
      cb->ex0[c] = r.v[i][3];
      cb->ex1[c] = r.v[i][4];
    }
  }
  if (tid == 0) cb->row_split = r.row_split;
}

// The PXA_LN_STAT_PARTS partial (sum, sum of squares) pairs of row `row` (fused LayerNorm consumer), loaded one tile ahead.
struct LnStatRegs {
  float4 t[PXA_LN_STAT_PARTS / 2];
};
PXA_DEVICE void load_ln_stats(LnStatRegs& r, const GemmParams& p, int row) {
  const float4* sp = reinterpret_cast<const float4*>(p.ln_stats + (size_t)(row < p.M ? row : p.M - 1) * (2 * PXA_LN_STAT_PARTS));
#pragma unroll
  for (int i = 0; i < PXA_LN_STAT_PARTS / 2; ++i) r.t[i] = __ldg(sp + i);
}
// (rstd, -rstd * mean), so that the normalised accumulator is fma(rstd, acc, fma(-rstd * mean, u, v)).
PXA_DEVICE float2 ln_row_coeffs(const GemmParams& p, const LnStatRegs& r) {
  float s = 0.f, q = 0.f;
#pragma unroll
  for (int i = 0; i < PXA_LN_STAT_PARTS / 2; ++i) {
    s += r.t[i].x + r.t[i].z;
    q += r.t[i].y + r.t[i].w;
  }
  const float mean = s * p.ln_inv_dim;
  const float var = fmaxf(q * p.ln_inv_dim - mean * mean, 0.f);
  const float rstd = rsqrtf(var + p.ln_eps);
  return make_float2(rstd, -rstd * mean);
}

// bf16 output (EPI 0/1/3/4) with staged constants: bias from smem (LDS broadcast).
//   PXA_EPI_BIAS_GELU_AUX: out = gelu(acc + bias) and, through the same smem transpose, out_aux = acc + bias (the
//                          pre-activation the GELU backward needs) -- the MLP's first GEMM in training;
//   PXA_EPI_MUL_DGELU:     out = acc * gelu'(pre), pre = p.residual read as bf16 [M, N] (row stride ldo) -- the dgrad GEMM of
//                          the MLP's second layer producing the gradient of the pre-activation directly.
//   PXA_EPI_LN_BIAS(_GELU): out = [gelu](rstd * (acc - mu * u) + v) -- the fused LayerNorm-modulate (see the header); `ln` =
//                          (rstd, -rstd * mu) of this thread's row, u / v of the row's sample from the staged constants.
template <int EPI>
PXA_DEVICE void epilogue_chunk_bf16_c(uint32_t (&v)[32], const GemmParams& p, const EpiConst* cb, uint8_t* stile, int lane,
                                      int row0, int col0, int ccol, float2 ln = make_float2(1.f, 0.f), bool second = false,
                                      int m_limit = -1) {
  constexpr bool kLn = (EPI == PXA_EPI_LN_BIAS || EPI == PXA_EPI_LN_BIAS_GELU);
  const int m_end = m_limit >= 0 ? m_limit : p.M;
  uint32_t pk[16];
  [[maybe_unused]] uint32_t pk2[16];
  const float4* bp = reinterpret_cast<const float4*>((kLn && second ? cb->gate0 : cb->bias) + ccol);
  [[maybe_unused]] const float4* up = reinterpret_cast<const float4*>((second ? cb->ex1 : cb->ex0) + ccol);
  [[maybe_unused]] uint4 pre[4];
  if constexpr (EPI == PXA_EPI_MUL_DGELU) {
    const __nv_bfloat16* pr = reinterpret_cast<const __nv_bfloat16*>(p.residual) + (size_t)(row0 + lane) * p.ldo + col0;
#pragma unroll
    for (int i = 0; i < 4; ++i)
      pre[i] = (row0 + lane < p.M && col0 + 8 * i < p.N) ? *reinterpret_cast<const uint4*>(pr + 8 * i) : make_uint4(0u, 0u, 0u, 0u);
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const float4 b = bp[i];
    float x0, x1, x2, x3;
    if constexpr (kLn) {
      const float4 u = up[i];
      x0 = fmaf(ln.x, __uint_as_float(v[4 * i]), fmaf(ln.y, u.x, b.x));
      x1 = fmaf(ln.x, __uint_as_float(v[4 * i + 1]), fmaf(ln.y, u.y, b.y));
      x2 = fmaf(ln.x, __uint_as_float(v[4 * i + 2]), fmaf(ln.y, u.z, b.z));
      x3 = fmaf(ln.x, __uint_as_float(v[4 * i + 3]), fmaf(ln.y, u.w, b.w));
    } else {
      x0 = __uint_as_float(v[4 * i]) + b.x; x1 = __uint_as_float(v[4 * i + 1]) + b.y;
      x2 = __uint_as_float(v[4 * i + 2]) + b.z; x3 = __uint_as_float(v[4 * i + 3]) + b.w;
    }
    if constexpr (EPI == PXA_EPI_BIAS_GELU_AUX) {
      pk2[2 * i] = pack_bf16x2(x0, x1);
      pk2[2 * i + 1] = pack_bf16x2(x2, x3);
    }
    if (EPI == PXA_EPI_BIAS_GELU || EPI == PXA_EPI_BIAS_GELU_AUX || EPI == PXA_EPI_LN_BIAS_GELU) {
      x0 = gelu_tanh(x0); x1 = gelu_tanh(x1); x2 = gelu_tanh(x2); x3 = gelu_tanh(x3);
    }
    if constexpr (EPI == PXA_EPI_MUL_DGELU) {
      const uint32_t w0 = (i & 1) ? pre[i >> 1].z : pre[i >> 1].x, w1 = (i & 1) ? pre[i >> 1].w : pre[i >> 1].y;
      x0 *= gelu_tanh_grad(bf16_lo(w0)); x1 *= gelu_tanh_grad(bf16_hi(w0));
      x2 *= gelu_tanh_grad(bf16_lo(w1)); x3 *= gelu_tanh_grad(bf16_hi(w1));
    }
    pk[2 * i] = pack_bf16x2(x0, x1);
    pk[2 * i + 1] = pack_bf16x2(x2, x3);
  }
  {
    const int sw = (lane >> 1) & 3;
#pragma unroll
    for (int c = 0; c < 4; ++c)
      *reinterpret_cast<uint4*>(stile + lane * 64 + ((c ^ sw) << 4)) = make_uint4(pk[4 * c], pk[4 * c + 1], pk[4 * c + 2], pk[4 * c + 3]);
  }
  __syncwarp();
  __nv_bfloat16* out = reinterpret_cast<__nv_bfloat16*>(p.out);
  const int c = lane & 3;
  uint4 u[4];
#pragma unroll
  for (int it = 0; it < 4; ++it) {
    const int r = it * 8 + (lane >> 2);
    u[it] = *reinterpret_cast<const uint4*>(stile + r * 64 + ((c ^ ((r >> 1) & 3)) << 4));
  }
#pragma unroll
  for (int it = 0; it < 4; ++it) {
    const int grow = row0 + it * 8 + (lane >> 2);
    const int gcol = col0 + c * 8;
    if (grow < m_end && gcol < p.N) *reinterpret_cast<uint4*>(out + (size_t)grow * p.ldo + gcol) = u[it];
  }
  __syncwarp();
  if constexpr (EPI == PXA_EPI_BIAS_GELU_AUX) {              // second pass of the same transpose for the pre-activation
    const int sw = (lane >> 1) & 3;
#pragma unroll
    for (int cc = 0; cc < 4; ++cc)
      *reinterpret_cast<uint4*>(stile + lane * 64 + ((cc ^ sw) << 4)) = make_uint4(pk2[4 * cc], pk2[4 * cc + 1], pk2[4 * cc + 2], pk2[4 * cc + 3]);
    __syncwarp();
#pragma unroll
    for (int it = 0; it < 4; ++it) {
      const int r = it * 8 + (lane >> 2);
      const uint4 w = *reinterpret_cast<const uint4*>(stile + r * 64 + ((c ^ ((r >> 1) & 3)) << 4));
      const int grow = row0 + r;
      const int gcol = col0 + c * 8;
      if (grow < p.M && gcol < p.N) *reinterpret_cast<uint4*>(p.out_aux + (size_t)grow * p.ldo + gcol) = w;
    }
    __syncwarp();
  }
}

// One chunk (32 columns) of the fp32 residual epilogue for the calling thread's row: out = residual + gate * (acc + bias), read and
// written straight from / to global memory in 16-byte pieces (every thread touches the four full 32-byte sectors of its own row).
// `reduce` (split-K weight gradients): the update is ADDED into `out` with vector reductions, so that the partial sums of the K
// splits meet in L2.  `st` accumulates this row's (sum, sum of squares) of the new residual values over the chunks of a tile (the
// fused LayerNorm's statistics, p.row_stats_out); with p.aux_scale the bf16 aux copy is out * (1 + scale of the next modulate).
PXA_DEVICE void residual_chunk_row_c(uint32_t (&v)[32], const GemmParams& p, const EpiConst* cb, int r, int ccol, int grow,
                                     int gcol0, bool reduce, float2& st) {
  if (grow >= p.M) return;
  const float4* bp = reinterpret_cast<const float4*>(cb->bias + ccol);
  const float4* gp = reinterpret_cast<const float4*>((r >= cb->row_split ? cb->gate1 : cb->gate0) + ccol);
  const float4* ep = reinterpret_cast<const float4*>((r >= cb->row_split ? cb->ex1 : cb->ex0) + ccol);
  const bool scaled_aux = p.aux_scale != nullptr;
  // samples shorter than a tile (rows_per_batch < 128, tiny images): a tile may span more than two samples, so the
  // gate row is looked up per thread in global memory instead of the two staged rows
  const bool per_row_gate = p.gate != nullptr && p.rows_per_batch < kBM;
  const float* gg = nullptr;
  if (per_row_gate) gg = p.gate + (size_t)((p.row_base + grow) / p.rows_per_batch) * p.gate_batch_stride + gcol0;
  const size_t off = (size_t)grow * p.ldo + gcol0;
  float* orow = reinterpret_cast<float*>(p.out) + off;
  const float* rrow = reinterpret_cast<const float*>(p.residual) + off;
  float4 res[8];
#pragma unroll
  for (int c = 0; c < 8; ++c)                                                                        // all loads first
    res[c] = (reduce || gcol0 + 4 * c >= p.N) ? make_float4(0.f, 0.f, 0.f, 0.f) : *reinterpret_cast<const float4*>(rrow + 4 * c);
  uint32_t aux[16];
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    const float4 b = bp[c];
    float4 g = gp[c];
    const bool col_ok = gcol0 + 4 * c < p.N;
    if (per_row_gate) g = col_ok ? __ldg(reinterpret_cast<const float4*>(gg + 4 * c)) : make_float4(1.f, 1.f, 1.f, 1.f);
    float4 o;
    const float4 yb = make_float4(__uint_as_float(v[4 * c + 0]) + b.x, __uint_as_float(v[4 * c + 1]) + b.y,
                                  __uint_as_float(v[4 * c + 2]) + b.z, __uint_as_float(v[4 * c + 3]) + b.w);
    o.x = fmaf(g.x, yb.x, res[c].x);
    o.y = fmaf(g.y, yb.y, res[c].y);
    o.z = fmaf(g.z, yb.z, res[c].z);
    o.w = fmaf(g.w, yb.w, res[c].w);
    if (col_ok) {
      st.x += (o.x + o.y) + (o.z + o.w);
      st.y = fmaf(o.x, o.x, fmaf(o.y, o.y, fmaf(o.z, o.z, fmaf(o.w, o.w, st.y))));
      if (reduce) red_add_f32x4(orow + 4 * c, o.x, o.y, o.z, o.w);
      else *reinterpret_cast<float4*>(orow + 4 * c) = o;
    }
    float4 ax = p.aux_branch ? yb : o;
    if (scaled_aux) {
      const float4 e = ep[c];
      ax = make_float4(ax.x * e.x, ax.y * e.y, ax.z * e.z, ax.w * e.w);
    }
    aux[2 * c] = pack_bf16x2(ax.x, ax.y);
    aux[2 * c + 1] = pack_bf16x2(ax.z, ax.w);
  }
  if (p.out_aux != nullptr) {
#pragma unroll
    for (int c = 0; c < 4; ++c)
      if (gcol0 + 8 * c < p.N)
        *reinterpret_cast<uint4*>(p.out_aux + off + 8 * c) = make_uint4(aux[4 * c], aux[4 * c + 1], aux[4 * c + 2], aux[4 * c + 3]);
  }
}

template <int BN>
PXA_DEVICE int chunks_of_tile(const GemmParams& p, int n0) {
  const int rem = (p.N - n0 + 31) / 32;
  return rem < BN / 32 ? rem : BN / 32;
}

}  // namespace pxa
