// Shared pieces of the wgmma GEMM kernel: parameters, shared-memory configuration and the epilogue constants.
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
  // per-output-column scale of the accumulator (kScale, pxa_gemm_dora_bf16): staged in EpiConst::ex1, which the scaled forms
  // do not otherwise use (they take no aux_scale)
  const float* col_scale;
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
// two) samples a 128-row tile can span.  Reading them per fragment is then an LDS broadcast instead of a chain of L2-latency
// global loads in the epilogue's critical path.  Double-buffered by tile parity.
template <int BN> struct EpiConst {
  float bias[BN];      // LN consumer epilogue: v of the first sample
  float gate0[BN];     // gate of the sample of the tile's first row (1.0 when there is no gate); LN consumer: v of the last sample
  float gate1[BN];     // gate of the sample of the tile's last row
  float ex0[BN];       // aux_scale of the first / last sample (1.0 when there is none); LN consumer: u of the first / last sample
  float ex1[BN];
  int row_split;       // tile rows >= row_split belong to the second sample
  int pad[3];
};

// Shared memory of one CTA: the operand ring, the output tile, the constants, one per-row float2 array per tile parity and the
// barriers.  The output tile is BN / 32 slabs of 128 rows x 32 columns of OutT (the TMA box of the output; 128-byte swizzle for
// fp32, 64-byte swizzle for bf16); consumer warpgroup g owns the slabs of its column half.  It receives the tile's epilogue
// operand (residual / pre-activation, loaded by the producer) and the results are written over it, then stored by TMA.
//   BN   out    ring stages   dynamic smem
//   128  bf16   5             205088 B
//   128  fp32   4             205088 B
//   192  bf16   4             224032 B
//   192  fp32   3             232224 B
//   256  bf16   3             226592 B     (fp32 output runs at BN 128: at 256 the ring would have 2 stages)
template <int BN, typename OutT> struct GemmCfg {
  static constexpr int kStageA = kBM * kBK * 2;                 // 16 KB
  static constexpr int kStageB = BN * kBK * 2;
  static constexpr int kStage = kStageA + kStageB;
  static constexpr int kSlabBytes = kBM * 32 * (int)sizeof(OutT);
  static constexpr int kEpiTile = kBM * BN * (int)sizeof(OutT);
  static constexpr int kConstBytes = 2 * (int)sizeof(EpiConst<BN>);
  static constexpr int kRowBytes = 2 * kBM * 8;                 // LN row coefficients / warpgroup row statistics
  static constexpr int kEpiSmem = kEpiTile + kConstBytes + kRowBytes;
  static constexpr int kBarBytes = 256;
  static constexpr int kMaxStages = (kSmemBudget - kEpiSmem - kBarBytes - 1024) / kStage;
  static constexpr int kStages = kMaxStages > 6 ? 6 : kMaxStages;
  static constexpr int kSmem = kStages * kStage + kEpiSmem + kBarBytes + 1024;  // +1024 alignment slack
  static_assert(kStages >= 3, "the operand ring needs 3 stages or more");
};

// Byte offset of element (row, col) of a 128 x 32 output slab, in the TMA swizzle of the slab's store: 16-byte chunk c of row r
// at chunk c ^ (r & 7) for fp32 (128-byte rows), c ^ ((r >> 1) & 3) for bf16 (64-byte rows).  Both are conflict-free for the
// wgmma fragment layout (8 rows x 2 columns per quad of lanes).
template <typename T> PXA_DEVICE uint32_t slab_offset(int row, int col) {
  if constexpr (sizeof(T) == 4) return row * 128 + ((((col >> 2) ^ (row & 7))) << 4) + (col & 3) * 4;
  else return row * 64 + (((col >> 3) ^ ((row >> 1) & 3)) << 4) + (col & 7) * 2;
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

template <int BN, bool kLn = false, bool kScale = false>
PXA_DEVICE void load_epi_consts(EpiRegs<BN>& r, const GemmParams& p, int tid, int m0, int n0) {
  const int b0 = m0 / p.rows_per_batch;
  const int last = (m0 + kBM - 1 < p.M ? m0 + kBM - 1 : p.M - 1);
  const int b1 = last / p.rows_per_batch;
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
      if constexpr (kScale) r.v[i][4] = ok ? __ldg(p.col_scale + col) : 1.f;
      else r.v[i][4] = (ok && p.aux_scale != nullptr) ? __ldg(p.aux_scale + (size_t)b1 * p.aux_scale_batch_stride + col) : 1.f;
    }
  }
  r.row_split = (b0 + 1) * p.rows_per_batch - m0;
}

template <int BN>
PXA_DEVICE void store_epi_consts(EpiConst<BN>* cb, const EpiRegs<BN>& r, int tid) {
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

}  // namespace pxa
