// wgmma GEMM for the linear layer:  C[M,N] = A[M,K] * B[N,K]^T   (bf16 in, fp32
// accumulate in registers, bf16 out), its dgrad form C = A[M,K] * B[K,N] (B read
// MN-major in place), and the fused form where the B operand is the rank-average of
// every rank's weight and is produced INSIDE the same kernel by communication warps
// (fused_allreduce_gemm, below).
//
// Structure: see wgmma_pipeline.cuh (persistent CTAs, 128x256 tiles - 128x128 in the fused
// kernel -, TMA producer warp, two consumer warpgroups).  Fused kernel only: four
// communication warps run the NVLS reduce of weight panels (multimem.ld_reduce over all
// ranks' weights -> x 1/size -> multimem.st into every rank's W_avg -> multimem.red on the
// panel counter).  The TMA producer polls that counter before loading from a panel, so the
// all-reduce of panel p+1.. overlaps the MMAs on panel p.
#include <cuda.h>

#include "kernels.h"
#include "fused_comm.cuh"
#include "tma_host.h"
#include "wgmma_pipeline.cuh"

namespace m4t {

namespace {

using namespace wg;

constexpr int kPanel = 256;  // weight rows per all-reduce panel of the fused kernel (one counter each)

// Epilogues of gemm_bf16_wgmma_kernel, its EPI template argument (an int, so the kernels' symbol names stay plain):
//   kStore          C = acc
//   kMse            C = grad_scale * (acc - T), loss_scale * sum((acc - T)^2) added to *loss_acc
//   kBiasGelu ...   the MLP epilogues, see mlp_epilogue and xent_epilogue
enum : int { kStore = 0, kMse = 1, kBiasGelu = 2, kBiasMseColsum = 3, kGeluBwdColsum = 4, kBiasXent = 5, kBias = 6 };
constexpr bool epi_adds_loss(int epi) { return epi == kMse || epi == kBiasMseColsum; }
constexpr bool epi_reads_t(int epi) { return epi == kMse || epi == kBiasMseColsum || epi == kGeluBwdColsum; }
// The MLP epilogues hold bias, target / z values and column sums next to the accumulators: the producer warpgroup
// hands registers to the consumers (40 + 2 x 232 per thread fits the register file).
constexpr bool epi_reallocs(int epi) { return epi >= kBiasGelu; }

struct GemmArgs {
  void* C;
  int M, N, K;
  int ldc;
  // fused MSE epilogue (kMse): C receives dL/dy = grad_scale * (y - T),
  // loss_acc accumulates loss_scale * sum((y - T)^2); y itself is never stored
  const void* T;
  int ldt;
  float* loss_acc;
  float loss_scale, grad_scale;
  // fused mode ----------------------------------------------------------------
  union {
    const uint32_t* panel_flags;  // [N / kPanel] counters in local HBM (written through multicast)
    const int* group_counts;      // GROUPED (never fused): [groups] rows of each group, int32 on the device
  };
  uint32_t panel_target;        // a panel is ready when its counter >= target (wrap-safe)
  // batched kernels: rows of one expert (a multiple of BM); grouped kernels: the number of groups.  Placed in the
  // tail padding, so the other kernels' parameter layout is unchanged.
  union {
    int expert_rows;
    int groups;
  };
};

// Epilogues of the two-layer MLP (unused by kStore / kMse):
//   kBiasGelu       TN  z = acc + bias -> C,  h = gelu_tanh(z) -> h_out
//   kBiasMseColsum  TN  d = acc + bias - T:  C = grad_scale * d, loss as kMse, column-sum partials of C
//   kGeluBwdColsum  NN  C = gscale * acc * gelu_tanh'(z), z read from T (bf16), column-sum partials of C
//   kBiasXent       TN  C = logits = acc + bias, per-tile softmax partials (xent_epilogue; xent_finish completes them)
//   kBias           TN  C = acc + bias (kBiasGelu without h)
// Column sums are deterministic: a warp adds its 16 rows in registers (h pair, then lane bits 2-4) and
// lanes 0-3 store one fp32 row of colsum[ceil(M/16), N]; column_sum_kernel adds those rows in a fixed order.
struct MlpEpiArgs {
  const float* bias;    // [N] fp32
  void* h_out;          // kBiasGelu: bf16, same layout as C
  float* colsum;        // kBiasMseColsum, kGeluBwdColsum: [ceil(M/16), N] fp32, row-major
  const float* gscale;  // kGeluBwdColsum: optional device scalar
  float2* xent_ms;      // kBiasXent: [ceil(N/256), M] (max, sum of exp) per row and column tile
};

constexpr float kGeluBeta = 0.7978845608028654f;  // sqrt(2/pi)
constexpr float kGeluKappa = 0.044715f;

__device__ __forceinline__ float gelu_tanh(float v) {
  const float t = tanhf(kGeluBeta * fmaf(kGeluKappa * v, v * v, v));
  return 0.5f * v * (1.f + t);
}

// d gelu_tanh / dv, written as torch's GeluBackward (approximate="tanh")
__device__ __forceinline__ float gelu_tanh_grad(float v) {
  const float v2 = v * v;
  const float t = tanhf(kGeluBeta * fmaf(kGeluKappa * v, v2, v));
  return 0.5f * (1.f + t) + 0.5f * v * (1.f - t * t) * kGeluBeta * fmaf(3.f * kGeluKappa, v2, 1.f);
}

// Epilogue of one consumer warpgroup's 64 x BN accumulators for kStore and kMse; returns this thread's part of the
// kMse loss.  N is a multiple of 8, so a column pair is either wholly inside or wholly outside.
template <int EPI, int BN>
__device__ __forceinline__ float store_epilogue(const float (&acc)[BN / 2], const GemmArgs& g, int m_blk, int n_blk,
                                                int wgi) {
  float loss_part = 0.f;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = m_blk * BM + wgi * 64 + frag_row(h);
    if (row >= g.M) continue;
    uint16_t* crow = static_cast<uint16_t*>(g.C) + static_cast<int64_t>(row) * g.ldc;
    const uint16_t* trow = epi_reads_t(EPI) ? static_cast<const uint16_t*>(g.T) + static_cast<int64_t>(row) * g.ldt : nullptr;
#pragma unroll
    for (int j0 = 0; j0 < BN / 8; j0 += 8) {
      uint32_t tv[8];  // the targets of eight column pairs are requested before the first is used
      if (epi_reads_t(EPI)) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int col = n_blk * BN + frag_col(j0 + j);
          tv[j] = col < g.N ? __ldcs(reinterpret_cast<const unsigned int*>(trow + col)) : 0u;
        }
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int col = n_blk * BN + frag_col(j0 + j);
        if (col >= g.N) continue;
        float v0 = acc[4 * (j0 + j) + 2 * h], v1 = acc[4 * (j0 + j) + 2 * h + 1];
        if (EPI == kMse) {
          const float d0 = v0 - bf16_bits_to_float(static_cast<uint16_t>(tv[j] & 0xffffu));
          const float d1 = v1 - bf16_bits_to_float(static_cast<uint16_t>(tv[j] >> 16));
          loss_part = fmaf(d0, d0, loss_part);
          loss_part = fmaf(d1, d1, loss_part);
          v0 = d0 * g.grad_scale;
          v1 = d1 * g.grad_scale;
        }
        *reinterpret_cast<uint32_t*>(crow + col) = pack_bf16x2(v0, v1);
      }
    }
  }
  return loss_part;
}

// Epilogue of one consumer warpgroup's 64 x BN accumulators for kBiasGelu, kBiasMseColsum, kGeluBwdColsum and kBias.
// Column pairs are handled in groups of kGroup, small enough that the bias / target / z values and the column sums
// fit next to acc.
template <int EPI, int BN>
__device__ __forceinline__ void mlp_epilogue(const float (&acc)[BN / 2], const GemmArgs& g, const MlpEpiArgs& e,
                                             int m_blk, int n_blk, int wgi, float& loss_part) {
  constexpr int kGroup = 4;
  constexpr bool kAddBias = EPI != kGeluBwdColsum, kColsum = EPI == kBiasMseColsum || EPI == kGeluBwdColsum;
  const int lane = threadIdx.x & 31;
  const int row0 = m_blk * BM + wgi * 64 + frag_row(0);
  const bool row_ok[2] = {row0 < g.M, row0 + 8 < g.M};
  const float gs = (EPI == kGeluBwdColsum && e.gscale != nullptr) ? *e.gscale : 1.f;
  const int prow = (m_blk * BM + wgi * 64) / 16 + ((threadIdx.x >> 5) & 3);  // this warp's colsum row
#pragma unroll
  for (int j0 = 0; j0 < BN / 8; j0 += kGroup) {
    // N is a multiple of 8: a group's column pairs are in range as a whole warp, and so are all earlier ones
    if (n_blk * BN + 8 * j0 >= g.N) break;
    float2 bv[kGroup];
    uint32_t tv[2][kGroup];
#pragma unroll
    for (int j = 0; j < kGroup; ++j) {
      const int col = n_blk * BN + frag_col(j0 + j);
      const bool col_ok = col < g.N;
      if (kAddBias) bv[j] = col_ok ? *reinterpret_cast<const float2*>(e.bias + col) : make_float2(0.f, 0.f);
      if (epi_reads_t(EPI)) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const uint16_t* trow = static_cast<const uint16_t*>(g.T) + static_cast<int64_t>(row0 + 8 * h) * g.ldt;
          tv[h][j] = (col_ok && row_ok[h]) ? __ldcs(reinterpret_cast<const unsigned int*>(trow + col)) : 0u;
        }
      }
    }
    float cs[kGroup][2];
#pragma unroll
    for (int j = 0; j < kGroup; ++j) {
      const int col = n_blk * BN + frag_col(j0 + j);
      cs[j][0] = cs[j][1] = 0.f;
      if (col >= g.N) continue;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float v0 = acc[4 * (j0 + j) + 2 * h], v1 = acc[4 * (j0 + j) + 2 * h + 1];
        if (kAddBias) {
          v0 += bv[j].x;
          v1 += bv[j].y;
        }
        if (!row_ok[h]) continue;
        const int64_t off = static_cast<int64_t>(row0 + 8 * h) * g.ldc + col;
        const float t0 = bf16_bits_to_float(static_cast<uint16_t>(tv[h][j] & 0xffffu));
        const float t1 = bf16_bits_to_float(static_cast<uint16_t>(tv[h][j] >> 16));
        if (EPI == kBiasGelu) {
          *reinterpret_cast<uint32_t*>(static_cast<uint16_t*>(e.h_out) + off) = pack_bf16x2(gelu_tanh(v0), gelu_tanh(v1));
        } else if (EPI == kBiasMseColsum) {
          const float d0 = v0 - t0, d1 = v1 - t1;
          loss_part = fmaf(d0, d0, loss_part);
          loss_part = fmaf(d1, d1, loss_part);
          v0 = d0 * g.grad_scale;
          v1 = d1 * g.grad_scale;
        } else if (EPI == kGeluBwdColsum) {
          v0 = gs * v0 * gelu_tanh_grad(t0);
          v1 = gs * v1 * gelu_tanh_grad(t1);
        }
        *reinterpret_cast<uint32_t*>(static_cast<uint16_t*>(g.C) + off) = pack_bf16x2(v0, v1);
        cs[j][0] += v0;
        cs[j][1] += v1;
      }
    }
    if (kColsum) {
#pragma unroll
      for (int j = 0; j < kGroup; ++j) {
#pragma unroll
        for (int o = 4; o < 32; o <<= 1) {
          cs[j][0] += __shfl_xor_sync(0xffffffffu, cs[j][0], o);
          cs[j][1] += __shfl_xor_sync(0xffffffffu, cs[j][1], o);
        }
        const int col = n_blk * BN + frag_col(j0 + j);
        if (lane < 4 && col < g.N && prow * 16 < g.M)
          *reinterpret_cast<float2*>(e.colsum + static_cast<int64_t>(prow) * g.N + col) = make_float2(cs[j][0], cs[j][1]);
      }
    }
  }
}

// The one exponential of the cross-entropy path: the epilogue's tile sums and xent_finish's probabilities must use
// the same function, or the softmax of a row would not add up to one.
__device__ __forceinline__ float xent_exp(float v) { return expf(v); }

// kBiasXent  TN  logit = bf16(acc + bias) -> C, and for each row the pair (m, s) of this 256-column tile: m the max of
// the row's stored (bf16-rounded) logits over the valid columns, s = sum exp(logit - m).  A thread reduces its 64
// values of a row, the quad (lanes 4r .. 4r+3 hold one row) combines them, and its first lane stores the pair.
// A -inf logit adds nothing to s without evaluating exp: a tile of -inf gives (-inf, 0), never exp(-inf - -inf).
// NaN is dropped by fmaxf but reaches s through exp(NaN - m); +inf gives m = +inf and s = exp(inf - inf) = NaN.
template <int BN>
__device__ __forceinline__ void xent_epilogue(float (&acc)[BN / 2], const GemmArgs& g, const MlpEpiArgs& e, int m_blk,
                                              int n_blk, int wgi) {
  const int row0 = m_blk * BM + wgi * 64 + frag_row(0);
  const bool row_ok[2] = {row0 < g.M, row0 + 8 < g.M};
  float m[2] = {-INFINITY, -INFINITY};
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    const int col = n_blk * BN + frag_col(j);
    if (col >= g.N) continue;  // N is a multiple of 8: a column pair is wholly in or out
    const float2 bv = *reinterpret_cast<const float2*>(e.bias + col);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const uint32_t p = pack_bf16x2(acc[4 * j + 2 * h] + bv.x, acc[4 * j + 2 * h + 1] + bv.y);
      const float v0 = bf16_bits_to_float(static_cast<uint16_t>(p & 0xffffu));
      const float v1 = bf16_bits_to_float(static_cast<uint16_t>(p >> 16));
      acc[4 * j + 2 * h] = v0;
      acc[4 * j + 2 * h + 1] = v1;
      m[h] = fmaxf(m[h], fmaxf(v0, v1));
      if (row_ok[h])
        *reinterpret_cast<uint32_t*>(static_cast<uint16_t*>(g.C) + static_cast<int64_t>(row0 + 8 * h) * g.ldc + col) = p;
    }
  }
  float s[2] = {0.f, 0.f};
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    m[h] = fmaxf(m[h], __shfl_xor_sync(0xffffffffu, m[h], 1));
    m[h] = fmaxf(m[h], __shfl_xor_sync(0xffffffffu, m[h], 2));
  }
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    if (n_blk * BN + frag_col(j) >= g.N) continue;
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const float v = acc[4 * j + 2 * h + i];
        s[h] += v == -INFINITY ? 0.f : xent_exp(v - m[h]);
      }
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    s[h] += __shfl_xor_sync(0xffffffffu, s[h], 1);
    s[h] += __shfl_xor_sync(0xffffffffu, s[h], 2);
    if ((threadIdx.x & 3) == 0 && row_ok[h]) e.xent_ms[static_cast<int64_t>(n_blk) * g.M + row0 + 8 * h] = make_float2(m[h], s[h]);
  }
}

// Grouped tiles: this warpgroup's rows at or past `valid` (an absolute row) of the tile become zero in C, and in
// h_out for kBiasGelu.  C is [g.M, g.N] contiguous with g.M a multiple of BM, so every row of the tile exists.
template <int EPI, int BN>
__device__ __forceinline__ void zero_rows_epilogue(const GemmArgs& g, const MlpEpiArgs& e, int m_blk, int n_blk, int wgi,
                                                   int valid) {
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = m_blk * BM + wgi * 64 + frag_row(h);
    if (row < valid) continue;
    const int64_t off = static_cast<int64_t>(row) * g.ldc;
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      const int col = n_blk * BN + frag_col(j);
      if (col >= g.N) break;
      *reinterpret_cast<uint32_t*>(static_cast<uint16_t*>(g.C) + off + col) = 0u;
      if (EPI == kBiasGelu) *reinterpret_cast<uint32_t*>(static_cast<uint16_t*>(e.h_out) + off + col) = 0u;
    }
  }
}

// Tile t of the grouped kernel: the used * n_tiles tiles of the groups come first, M fastest, then the zero tiles of the
// m-blocks behind the last group, so the persistent CTAs share the real tiles evenly.
__device__ __forceinline__ void grouped_tile(int t, int m_tiles, int used, int n_tiles, int& m_blk, int& n_blk) {
  const int live = used * n_tiles;
  if (t < live) {
    n_blk = t / used;
    m_blk = t - n_blk * used;
  } else {
    const int z = t - live, rest = m_tiles - used;
    n_blk = z / rest;
    m_blk = used + (z - n_blk * rest);
  }
}

// Producer and consumer roles of the grouped kernel (see gemm_bf16_wgmma_kernel).  A tile of group ge reads B at row
// offset ge * (N, or K if B_MN), the bias at ge * N, and stores its rows below the group's end.
template <int EPI, bool B_MN, int BN>
__device__ __forceinline__ void grouped_roles(uint8_t* smem, Pipe* pipe, const CUtensorMap* tmap_a,
                                              const CUtensorMap* tmap_b, const GemmArgs& g, const MlpEpiArgs& e,
                                              int first_tile, int tile_stride, int m_tiles, int num_tiles, int k_blocks) {
  const GroupTable* grp = group_table_of(pipe);
  const int n_tiles = num_tiles / m_tiles;
  const int warp = threadIdx.x >> 5;
  const int used = grp->pfx[g.groups];  // m-blocks holding groups; the rest are zero tiles
  if (warp < 4) {
    if constexpr (epi_reallocs(EPI)) tc::setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int t = first_tile; t < used * n_tiles; t += tile_stride) {
        int m_blk, n_blk;
        grouped_tile(t, m_tiles, used, n_tiles, m_blk, n_blk);
        const int b_row0 = group_of(grp, g.groups, m_blk) * (B_MN ? g.K : g.N);
        for (int kb = 0; kb < k_blocks; ++kb)
          load_stage<false, B_MN, BN>(smem, pipe, stage, phase, tmap_a, tmap_b, m_blk * BM, n_blk * BN, kb * BK, b_row0);
      }
    }
  } else {
    if constexpr (epi_reallocs(EPI)) tc::setmaxnreg_inc<232>();
    const int wgi = warp / 4 - 1;
    int stage = 0;
    uint32_t phase = 0;
    float acc[BN / 2];
    for (int t = first_tile; t < num_tiles; t += tile_stride) {
      int m_blk, n_blk;
      grouped_tile(t, m_tiles, used, n_tiles, m_blk, n_blk);
      int valid = m_blk * BM;  // rows below this one are stored from acc, the tile's others as zero
      if (m_blk < used) {
        const int ge = group_of(grp, g.groups, m_blk);
        valid = grp->end[ge];
        mma_tile<false, B_MN, BN>(acc, smem, pipe, stage, phase, k_blocks, wgi);
        GemmArgs gg = g;
        gg.M = valid;
        if constexpr (EPI == kStore) {
          store_epilogue<EPI, BN>(acc, gg, m_blk, n_blk, wgi);
        } else {
          float unused = 0.f;
          MlpEpiArgs ex = e;
          if (e.bias != nullptr) ex.bias = e.bias + static_cast<int64_t>(ge) * g.N;
          mlp_epilogue<EPI, BN>(acc, gg, ex, m_blk, n_blk, wgi, unused);
        }
      }
      zero_rows_epilogue<EPI, BN>(g, e, m_blk, n_blk, wgi, valid);
    }
  }
}

// BATCHED: E experts stacked along M (g.M = E * g.expert_rows); the tile's expert is m0 / expert_rows.  Only B and
// the bias depend on it: B is one map over the stacked weights, read at row offset expert * (N, or K if B_MN).
// GROUPED: g.groups groups of g.group_counts[e] rows in the grouped layout of the g.M rows (GroupTable, built once per
// CTA in shared memory).  The tile space is every m-block of g.M (grouped_tile): a tile's group comes from the table,
// its rows at or past the group's count are stored as zero, and m-blocks behind the last group are zero tiles that
// load nothing and come after all the others.  Epilogues kStore, kBiasGelu, kGeluBwdColsum and kBias.
template <bool FUSED, int EPI, bool B_MN, bool BATCHED = false, bool GROUPED = false>
__global__ void __launch_bounds__(kGemmThreads + (FUSED ? kCommWarps * 32 : 0), 1)
gemm_bf16_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                       const GemmArgs g, const CommArgs cm, const MlpEpiArgs e) {
  static_assert(!GROUPED || (!FUSED && !BATCHED && (EPI == kStore || EPI == kBiasGelu || EPI == kGeluBwdColsum ||
                                                    EPI == kBias)),
                "grouped GEMM epilogues");
  constexpr int BN = tile_n<FUSED>();
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = aligned_smem(smem_raw);
  Pipe* pipe = pipe_of<BN>(smem);
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  // read once for both roles: reading them inside each branch costs the fused kernel ten registers
  const int first_tile = blockIdx.x, tile_stride = gridDim.x;

  const int m_tiles = (g.M + BM - 1) / BM;
  const int n_tiles = (g.N + BN - 1) / BN;
  const int num_tiles = m_tiles * n_tiles;
  const int k_blocks = (g.K + BK - 1) / BK;

  if (warp == 0 && lane == 0) {
    tc::prefetch_tmap(&tmap_a);
    tc::prefetch_tmap(&tmap_b);
    init_pipe<BN>(pipe);
  }
  if constexpr (GROUPED) {
    if (threadIdx.x == 32) build_group_table(group_table_of(pipe), g.group_counts, g.groups, g.M);
  }
  __syncthreads();
  if constexpr (GROUPED) {
    grouped_roles<EPI, B_MN, BN>(smem, pipe, &tmap_a, &tmap_b, g, e, first_tile, tile_stride, m_tiles, num_tiles,
                                 k_blocks);
    __syncthreads();
    return;
  }

  if (warp < 4) {
    // =========================== TMA producer ===========================
    if constexpr (epi_reallocs(EPI)) tc::setmaxnreg_dec<40>();
    if (warp == 0 && lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int t = first_tile; t < num_tiles; t += tile_stride) {
        const int n_blk = t / m_tiles;  // M fastest: a wave works on few weight panels
        const int m_blk = t - n_blk * m_tiles;
        if (FUSED) {
          // the weight panel must have been all-reduced (by every rank) first
          bounded_wait_ge(g.panel_flags + n_blk * BN / kPanel, g.panel_target, cm.sync);
          tc::fence_proxy_async();  // generic-proxy writes (multimem.st) -> async-proxy reads (TMA)
        }
        const int b_row0 = BATCHED ? (m_blk * BM / g.expert_rows) * (B_MN ? g.K : g.N) : 0;
        for (int kb = 0; kb < k_blocks; ++kb)
          load_stage<false, B_MN, BN>(smem, pipe, stage, phase, &tmap_a, &tmap_b, m_blk * BM, n_blk * BN, kb * BK,
                                      b_row0);
      }
    }
  } else if (warp < kGemmThreads / 32) {
    // ====================== consumers: wgmma + epilogue ======================
    if constexpr (epi_reallocs(EPI)) tc::setmaxnreg_inc<232>();
    const int wgi = warp / 4 - 1;
    int stage = 0;
    uint32_t phase = 0;
    float acc[BN / 2];
    for (int t = first_tile; t < num_tiles; t += tile_stride) {
      const int n_blk = t / m_tiles;
      const int m_blk = t - n_blk * m_tiles;
      mma_tile<false, B_MN, BN>(acc, smem, pipe, stage, phase, k_blocks, wgi);
      float loss_part = 0.f;
      if constexpr (EPI == kStore || EPI == kMse) {
        loss_part = store_epilogue<EPI, BN>(acc, g, m_blk, n_blk, wgi);
      } else if constexpr (EPI == kBiasXent) {
        xent_epilogue<BN>(acc, g, e, m_blk, n_blk, wgi);
      } else if constexpr (BATCHED) {
        MlpEpiArgs ex = e;
        if (e.bias != nullptr) ex.bias = e.bias + static_cast<int64_t>(m_blk * BM / g.expert_rows) * g.N;
        mlp_epilogue<EPI, BN>(acc, g, ex, m_blk, n_blk, wgi, loss_part);
      } else {
        mlp_epilogue<EPI, BN>(acc, g, e, m_blk, n_blk, wgi, loss_part);
      }
      if (epi_adds_loss(EPI)) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) loss_part += __shfl_xor_sync(0xffffffffu, loss_part, o);
        if (lane == 0) atomicAdd(g.loss_acc, loss_part * g.loss_scale);
      }
    }
  } else if (FUSED) {
    // =========================== communication ==========================
    comm_allreduce_panels<kCommWarps, kPanel>(cm, kGemmThreads, g.N / kPanel, g.K);
  }
  __syncthreads();
}

// ---------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------
// Row-major [rows, cols] bf16 matrix, box = [box_rows, 64 cols], 128-byte swizzle.
CUtensorMap make_tmap(const void* base, int64_t rows, int64_t cols, int64_t ld, int box_rows) {
  return make_tmap_bf16_sw128(base, rows, cols, ld, BK, box_rows);
}

// ctas: the SM count, of which the persistent grid uses no more than g has tiles; the fused kernel's grid
// (fused_gemm_grid), which it uses whole.
template <bool FUSED, int EPI, bool B_MN, bool BATCHED = false, bool GROUPED = false>
void launch(int ctas, const CUtensorMap& ta, const CUtensorMap& tb, const GemmArgs& g, cudaStream_t stream,
            const char* what, const MlpEpiArgs& e = MlpEpiArgs{}, const CommArgs& cm = CommArgs{}) {
  constexpr int BN = tile_n<FUSED>();
  const int64_t M = g.M, N = g.N;
  const int grid = FUSED ? ctas : persistent_grid(((M + BM - 1) / BM) * ((N + BN - 1) / BN), ctas);
  launch_kernel<gemm_bf16_wgmma_kernel<FUSED, EPI, B_MN, BATCHED, GROUPED>>(
      grid, kGemmThreads + (FUSED ? kCommWarps * 32 : 0), Tile<BN>::kSmemBytes + (GROUPED ? kGroupTableBytes : 0), stream,
      what, ta, tb, g, cm, e);
}

void set_mse(GemmArgs& g, const MseEpilogue* mse) {
  g.T = mse->target;
  g.ldt = static_cast<int>(mse->ldt);
  g.loss_acc = mse->loss_acc;
  g.loss_scale = mse->loss_scale;
  g.grad_scale = mse->grad_scale;
}

// out[n] = gscale * sum_i partial[i, n] over i = 0, 1, .. in a fixed order: a block covers 32 columns,
// its 8 row groups each add every 8th row, and row group 0 adds the 8 results in order.
// BATCHED: expert e = blockIdx.y reduces partial[e] [rows, N] into out[e] [N] in that same order.
template <bool BATCHED = false>
__global__ void __launch_bounds__(256) column_sum_kernel(const float* __restrict__ partial, int rows, int N,
                                                         float* __restrict__ out, const float* gscale) {
  __shared__ float part[8][33];
  if (BATCHED) {
    partial += static_cast<int64_t>(blockIdx.y) * rows * N;
    out += static_cast<int64_t>(blockIdx.y) * N;
  }
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int n = blockIdx.x * 32 + tx;
  float s = 0.f;
  if (n < N)
    for (int i = ty; i < rows; i += 8) s += partial[static_cast<int64_t>(i) * N + n];
  part[ty][tx] = s;
  __syncthreads();
  if (ty == 0 && n < N) {
    float t = part[0][tx];
#pragma unroll
    for (int k = 1; k < 8; ++k) t += part[k][tx];
    out[n] = gscale != nullptr ? t * *gscale : t;
  }
}

constexpr int kXentRows = 16;  // rows per block: one row of the column-sum partials, as EPI 3 writes them
constexpr int kXentThreads = 256;
constexpr int kXentCols = 8 * kXentThreads;  // columns per block: 8 per thread, one 16-byte load per row

// Completes EPI 5 in place over the logits y [M, N] (bf16, leading dimension ldy).  Block b covers rows
// [16 r, 16 r + 16) and columns [2048 c, 2048 c + 2048) with r = b / col_blocks, c = b % col_blocks.
//   1. lse of its 16 rows from the tile pairs ms[tile, row] = (m, s): M = max m, lse = M + log sum s exp(m - M).
//      Thread (slot, row) visits tiles slot, slot + 16, ..; the 16 slots are then added in order.  A tile with
//      s = 0 (all its logits -inf) is skipped, so exp(-inf - -inf) is never evaluated.
//   2. dy = grad_scale (exp(logit - lse) - [col == label]) over the logits, and colsum[r, col] = sum of the 16 rows'
//      fp32 dy in row order.  A row whose label is ignore_index gets dy = 0; one whose label is outside [0, N) NaN.
//   3. The loss of row i is lse - logit[i, label] (0 if ignored, NaN if the label is out of range), stored in
//      row_loss.  The last block to finish (an integer counter) adds row_loss in a fixed order: the same bits on
//      every call, with no float atomics.
__global__ void __launch_bounds__(kXentThreads) xent_finish_kernel(uint16_t* __restrict__ y, int64_t ldy,
                                                                   const float2* __restrict__ ms, int tiles,
                                                                   const int64_t* __restrict__ labels, int M, int N,
                                                                   int64_t ignore_index, float loss_scale, float grad_scale,
                                                                   float* __restrict__ row_loss, unsigned int* done,
                                                                   float* __restrict__ loss, float* __restrict__ colsum) {
  __shared__ float red[kXentThreads];
  __shared__ float lse_s[kXentRows];
  __shared__ int64_t lab_s[kXentRows];
  __shared__ bool last;
  const int t = threadIdx.x;
  const int col_blocks = (N + kXentCols - 1) / kXentCols;
  const int rg = static_cast<int>(blockIdx.x / col_blocks), cb = static_cast<int>(blockIdx.x % col_blocks);
  const int r0 = rg * kXentRows;
  {
    const int row = t % kXentRows, slot = t / kXentRows, r = r0 + row;
    constexpr int kSlots = kXentThreads / kXentRows;
    float mx = -INFINITY;
    if (r < M)
      for (int j = slot; j < tiles; j += kSlots) mx = fmaxf(mx, ms[static_cast<int64_t>(j) * M + r].x);
    red[t] = mx;
    __syncthreads();
    float big = -INFINITY;
#pragma unroll
    for (int k = 0; k < kSlots; ++k) big = fmaxf(big, red[k * kXentRows + row]);
    __syncthreads();
    float sum = 0.f;
    if (r < M)
      for (int j = slot; j < tiles; j += kSlots) {
        const float2 p = ms[static_cast<int64_t>(j) * M + r];
        if (p.y != 0.f) sum += p.y * xent_exp(p.x - big);
      }
    red[t] = sum;
    __syncthreads();
    if (slot == 0) {
      float tot = 0.f;
#pragma unroll
      for (int k = 0; k < kSlots; ++k) tot += red[k * kXentRows + row];
      lse_s[row] = big + logf(tot);
      lab_s[row] = r < M ? labels[r] : ignore_index;
    }
    __syncthreads();
  }
  const int c = cb * kXentCols + 8 * t;
  float cs[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  for (int i = 0; i < kXentRows && r0 + i < M; ++i) {
    const int r = r0 + i;
    const int64_t lab = lab_s[i];
    const bool ignored = lab == ignore_index;
    const bool valid = !ignored && lab >= 0 && lab < N;
    // a label that is no column of the row: its loss is written once, by the first thread of column block 0
    if (!valid && cb == 0 && t == 0) row_loss[r] = ignored ? 0.f : NAN;
    if (c >= N) continue;
    uint16_t* yr = y + static_cast<int64_t>(r) * ldy + c;
    const uint4 raw = *reinterpret_cast<const uint4*>(yr);
    const uint32_t w[4] = {raw.x, raw.y, raw.z, raw.w};
    float v[8];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      v[2 * k] = bf16_bits_to_float(static_cast<uint16_t>(w[k] & 0xffffu));
      v[2 * k + 1] = bf16_bits_to_float(static_cast<uint16_t>(w[k] >> 16));
    }
    const float lse = lse_s[i];
    // In place: the store below overwrites logit[r, label], which the row's loss needs.  Only this thread holds
    // that column, so it reads the logit here, from the registers loaded before its own store.
    if (valid && lab >= c && lab < c + 8) {
      float vl = 0.f;
#pragma unroll
      for (int k = 0; k < 8; ++k)
        if (c + k == lab) vl = v[k];
      row_loss[r] = lse - vl;
    }
    float d[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      d[k] = ignored ? 0.f : valid ? grad_scale * (xent_exp(v[k] - lse) - (c + k == lab ? 1.f : 0.f)) : NAN;
      cs[k] += d[k];
    }
    *reinterpret_cast<uint4*>(yr) = make_uint4(pack_bf16x2(d[0], d[1]), pack_bf16x2(d[2], d[3]), pack_bf16x2(d[4], d[5]),
                                               pack_bf16x2(d[6], d[7]));
  }
  if (c < N) {
    float4* out = reinterpret_cast<float4*>(colsum + static_cast<int64_t>(rg) * N + c);
    out[0] = make_float4(cs[0], cs[1], cs[2], cs[3]);
    out[1] = make_float4(cs[4], cs[5], cs[6], cs[7]);
  }
  // every block's row losses are visible before its arrival on the counter
  __threadfence();
  __syncthreads();
  if (t == 0) last = atomicAdd(done, 1u) == gridDim.x - 1;
  __syncthreads();
  if (!last) return;
  __threadfence();
  float part = 0.f;
  for (int r = t; r < M; r += kXentThreads) part += __ldcg(row_loss + r);
  red[t] = part;
  __syncthreads();
#pragma unroll
  for (int s = kXentThreads / 2; s > 0; s >>= 1) {
    if (t < s) red[t] += red[t + s];
    __syncthreads();
  }
  if (t == 0) *loss = loss_scale * red[0];
}

GemmArgs plain_args(void* C, int64_t M, int64_t N, int64_t K, int64_t ldc) {
  GemmArgs g{};
  g.C = C;
  g.M = static_cast<int>(M);
  g.N = static_cast<int>(N);
  g.K = static_cast<int>(K);
  g.ldc = static_cast<int>(ldc);
  return g;
}

GemmArgs batched_args(void* C, int64_t E, int64_t M, int64_t N, int64_t K) {
  GemmArgs g = plain_args(C, E * M, N, K, N);
  g.expert_rows = static_cast<int>(M);
  return g;
}

}  // namespace

bool gemm_bf16_tn_supported(int64_t M, int64_t N, int64_t K, const void* A, const void* B, const void* C, int64_t lda,
                            int64_t ldb, int64_t ldc) {
  return M > 0 && N > 0 && K > 0 && (K % 8) == 0 && (N % 8) == 0 && (lda % 8) == 0 && (ldb % 8) == 0 && (ldc % 8) == 0 &&
         lda >= K && ldb >= K && ldc >= N && aligned16(A) && aligned16(B) && aligned16(C) && M < (1ll << 31) &&
         N < (1ll << 31) && K < (1ll << 31);
}

bool epilogue_bf16_pairs_ok(const void* p, int64_t ld) {
  return (reinterpret_cast<uintptr_t>(p) & 3u) == 0 && ld % 2 == 0 && ld >= 0 && ld < (1ll << 31);
}

bool epilogue_bias_ok(const float* bias) { return (reinterpret_cast<uintptr_t>(bias) & 7u) == 0; }

void launch_gemm_bf16_tn(const void* A, const void* B, void* C, int64_t M, int64_t N, int64_t K, int64_t lda,
                         int64_t ldb, int64_t ldc, int sm_count, cudaStream_t stream, const MseEpilogue* mse) {
  M4T_CHECK(gemm_bf16_tn_supported(M, N, K, A, B, C, lda, ldb, ldc), "unsupported GEMM shape/alignment for the wgmma path");
  M4T_CHECK(mse == nullptr || epilogue_bf16_pairs_ok(mse->target, mse->ldt),
            "the MSE target needs a 4-byte-aligned base and an even row stride");
  const CUtensorMap ta = make_tmap(A, M, K, lda, BM);
  const CUtensorMap tb = make_tmap(B, N, K, ldb, tile_n<false>());
  GemmArgs g = plain_args(C, M, N, K, ldc);
  if (mse) {
    set_mse(g, mse);
    launch<false, kMse, false>(sm_count, ta, tb, g, stream, "gemm_mse_epilogue");
  } else {
    launch<false, kStore, false>(sm_count, ta, tb, g, stream, "gemm_bf16_tn");
  }
}

bool gemm_bf16_nn_supported(int64_t M, int64_t N, int64_t K, const void* A, const void* B, const void* C, int64_t lda,
                            int64_t ldb, int64_t ldc) {
  return M > 0 && N > 0 && K > 0 && N % 8 == 0 && K % 8 == 0 && aligned16(A) && aligned16(B) && aligned16(C) &&
         lda % 8 == 0 && ldb % 8 == 0 && ldc % 8 == 0 && lda >= K && ldb >= N && ldc >= N && M < (1ll << 31) &&
         N < (1ll << 31) && K < (1ll << 31);
}

// C[M,N] = A[M,K] * B[K,N], both row-major (the dgrad shape: gy @ W).
void launch_gemm_bf16_nn(const void* A, const void* B, void* C, int64_t M, int64_t N, int64_t K, int64_t lda,
                         int64_t ldb, int64_t ldc, int sm_count, cudaStream_t stream) {
  M4T_CHECK(gemm_bf16_nn_supported(M, N, K, A, B, C, lda, ldb, ldc), "unsupported GEMM shape/alignment for the wgmma NN path");
  const CUtensorMap ta = make_tmap(A, M, K, lda, BM);
  const CUtensorMap tb = make_tmap_bf16_sw128(B, K, N, ldb, 64, BK);  // boxes of {64 n, BK k-rows}
  launch<false, kStore, true>(sm_count, ta, tb, plain_args(C, M, N, K, ldc), stream, "gemm_nn");
}

// y = x @ mean_ranks(W)^T in ONE kernel.  `w_off`/`wavg_off`/`flags_off` are
// byte offsets inside the symmetric heap (identical on all ranks); the weight
// must already be staged at w_off on every rank.
void launch_fused_allreduce_gemm(const DeviceComm& dc, const void* x, void* y, int64_t M, int64_t N, int64_t K,
                                 int64_t ldx, int64_t ldy, int64_t w_off, int64_t wavg_off, int64_t flags_off,
                                 uint32_t panel_target, float scale, cudaStream_t stream, const MseEpilogue* mse) {
  M4T_CHECK(dc.mc_heap != nullptr, "the fused Allreduce->GEMM kernel needs the NVLS multicast mapping");
  const int P = dc.sync.size;
  M4T_CHECK(kPanel % P == 0 && N % kPanel == 0 && (K * 2) % 16 == 0,
            "fused Allreduce->GEMM: N must be a multiple of 256 and 256 % ranks == 0");
  const char* wavg = dc.heap[dc.sync.rank] + wavg_off;
  M4T_CHECK(gemm_bf16_tn_supported(M, N, K, x, wavg, y, ldx, K, ldy), "unsupported GEMM shape/alignment for the fused path");
  M4T_CHECK(mse == nullptr || epilogue_bf16_pairs_ok(mse->target, mse->ldt),
            "the MSE target needs a 4-byte-aligned base and an even row stride");
  constexpr int BN = tile_n<true>();
  const CUtensorMap ta = make_tmap(x, M, K, ldx, BM);
  const CUtensorMap tb = make_tmap(wavg, N, K, K, BN);
  GemmArgs g = plain_args(y, M, N, K, ldy);
  g.panel_flags = reinterpret_cast<const uint32_t*>(dc.heap[dc.sync.rank] + flags_off);
  g.panel_target = panel_target;
  CommArgs cm{};
  cm.sync = dc.sync;
  cm.mc_heap = dc.mc_heap;
  cm.my_heap = dc.heap[dc.sync.rank];
  cm.w_off = w_off;
  cm.wavg_off = wavg_off;
  cm.flags_off = flags_off;
  cm.scale = scale;
  cm.do_barrier = 1;
  static const int fused_debug = static_cast<int>(env_i64("M4T_FUSED_DEBUG", 0));  // read once
  cm.debug_skip = fused_debug;
  if (cm.debug_skip & 2) g.M = 0;  // timing experiment: communication only, no GEMM tiles
  // the grid must be identical on every rank (per-block barrier + counter targets)
  const int grid = fused_gemm_grid(dc);
  if (mse) {
    set_mse(g, mse);
    launch<true, kMse, false>(grid, ta, tb, g, stream, "fused_allreduce_gemm_mse", MlpEpiArgs{}, cm);
  } else {
    launch<true, kStore, false>(grid, ta, tb, g, stream, "fused_allreduce_gemm", MlpEpiArgs{}, cm);
  }
}

int64_t colsum_rows(int64_t M) { return (M + 15) / 16; }

void launch_gemm_bias_gelu(const void* A, const void* B, const float* bias, void* z, void* h, int64_t M, int64_t N,
                           int64_t K, int64_t lda, int64_t ldb, int64_t ldc, int sm_count, cudaStream_t stream) {
  M4T_CHECK(gemm_bf16_tn_supported(M, N, K, A, B, z, lda, ldb, ldc) && aligned16(h),
            "unsupported GEMM shape/alignment for the wgmma bias+GELU path");
  M4T_CHECK(epilogue_bias_ok(bias), "the bias needs an 8-byte-aligned base");
  MlpEpiArgs e{};
  e.bias = bias;
  e.h_out = h;
  launch<false, kBiasGelu, false>(sm_count, make_tmap(A, M, K, lda, BM), make_tmap(B, N, K, ldb, tile_n<false>()),
                           plain_args(z, M, N, K, ldc), stream, "gemm_bias_gelu", e);
}

void launch_gemm_bias_mse_colsum(const void* A, const void* B, const float* bias, void* dy, float* colsum, int64_t M,
                                 int64_t N, int64_t K, int64_t lda, int64_t ldb, int64_t ldc, int sm_count,
                                 cudaStream_t stream, const MseEpilogue& mse) {
  M4T_CHECK(gemm_bf16_tn_supported(M, N, K, A, B, dy, lda, ldb, ldc), "unsupported GEMM shape/alignment for the wgmma bias+MSE path");
  M4T_CHECK(epilogue_bf16_pairs_ok(mse.target, mse.ldt), "the MSE target needs a 4-byte-aligned base and an even row stride");
  M4T_CHECK(epilogue_bias_ok(bias), "the bias needs an 8-byte-aligned base");
  GemmArgs g = plain_args(dy, M, N, K, ldc);
  set_mse(g, &mse);
  MlpEpiArgs e{};
  e.bias = bias;
  e.colsum = colsum;
  launch<false, kBiasMseColsum, false>(sm_count, make_tmap(A, M, K, lda, BM), make_tmap(B, N, K, ldb, tile_n<false>()), g,
                                stream, "gemm_bias_mse_colsum", e);
}

void launch_gemm_nn_gelu_bwd_colsum(const void* A, const void* B, const void* z, void* dz, float* colsum, int64_t M,
                                    int64_t N, int64_t K, int64_t lda, int64_t ldb, int64_t ldz, int64_t ldc,
                                    int sm_count, cudaStream_t stream, const float* gscale) {
  M4T_CHECK(gemm_bf16_nn_supported(M, N, K, A, B, dz, lda, ldb, ldc),
            "unsupported GEMM shape/alignment for the wgmma GELU-backward path");
  M4T_CHECK(epilogue_bf16_pairs_ok(z, ldz), "z needs a 4-byte-aligned base and an even row stride");
  GemmArgs g = plain_args(dz, M, N, K, ldc);
  g.T = z;
  g.ldt = static_cast<int>(ldz);
  MlpEpiArgs e{};
  e.colsum = colsum;
  e.gscale = gscale;
  launch<false, kGeluBwdColsum, true>(sm_count, make_tmap(A, M, K, lda, BM), make_tmap_bf16_sw128(B, K, N, ldb, 64, BK), g,
                               stream, "gemm_nn_gelu_bwd_colsum", e);
}

void launch_column_sum(const float* partial, int64_t rows, int64_t N, float* out, const float* gscale, cudaStream_t stream) {
  M4T_CHECK(rows > 0 && N > 0 && N < (1ll << 31) && rows < (1ll << 31), "column_sum: empty or oversized workspace");
  launch_kernel<column_sum_kernel<>>(static_cast<unsigned>((N + 31) / 32), 256, 0, stream, "column_sum", partial,
                                     static_cast<int>(rows), static_cast<int>(N), out, gscale);
}

int64_t xent_tiles(int64_t N) { return (N + tile_n<false>() - 1) / tile_n<false>(); }

void launch_gemm_bias_xent(const void* A, const void* B, const float* bias, void* logits, float2* ms, int64_t M,
                           int64_t N, int64_t K, int64_t lda, int64_t ldb, int64_t ldc, int sm_count, cudaStream_t stream) {
  M4T_CHECK(gemm_bf16_tn_supported(M, N, K, A, B, logits, lda, ldb, ldc),
            "unsupported GEMM shape/alignment for the wgmma bias+cross-entropy path");
  M4T_CHECK(epilogue_bias_ok(bias), "the bias needs an 8-byte-aligned base");
  MlpEpiArgs e{};
  e.bias = bias;
  e.xent_ms = ms;
  launch<false, kBiasXent, false>(sm_count, make_tmap(A, M, K, lda, BM), make_tmap(B, N, K, ldb, tile_n<false>()),
                           plain_args(logits, M, N, K, ldc), stream, "gemm_bias_xent", e);
}

void launch_xent_finish(void* y, int64_t M, int64_t N, int64_t ldy, const float2* ms, const int64_t* labels,
                        int64_t ignore_index, float loss_scale, float grad_scale, float* row_loss, unsigned int* done,
                        float* loss, float* colsum, cudaStream_t stream) {
  M4T_CHECK(M > 0 && N > 0 && N % 8 == 0 && ldy % 8 == 0 && ldy >= N && aligned16(y) && aligned16(colsum) &&
                M < (1ll << 31) && N < (1ll << 31),
            "xent_finish: unsupported shape or alignment");
  const int64_t blocks = ((M + kXentRows - 1) / kXentRows) * ((N + kXentCols - 1) / kXentCols);
  M4T_CHECK(blocks < (1ll << 31), "xent_finish: too many blocks");
  launch_kernel<xent_finish_kernel>(static_cast<unsigned>(blocks), kXentThreads, 0, stream, "xent_finish",
                                    static_cast<uint16_t*>(y), ldy, ms, static_cast<int>(xent_tiles(N)), labels,
                                    static_cast<int>(M), static_cast<int>(N), ignore_index, loss_scale, grad_scale,
                                    row_loss, done, loss, colsum);
}

int fused_gemm_grid(const DeviceComm& dc) { return std::min(dc.sm_count, kMaxChannels) & ~1; }

// ---- batched experts ---------------------------------------------------------------------------------------------
// Every operand is contiguous and stacked along its leading dimension, so expert e's A rows are rows [e M, e M + M) of
// one [E M, K] matrix and the whole call is ONE GEMM of E M rows against a B that changes at every M rows.
bool batched_gemm_supported(int64_t E, int64_t M, int64_t N, int64_t K, const void* A, const void* B, const void* C) {
  return E > 0 && M > 0 && N > 0 && K > 0 && M % BM == 0 && N % 128 == 0 && K % 128 == 0 && aligned16(A) &&
         aligned16(B) && aligned16(C) && E * M < (1ll << 31) && E * N < (1ll << 31) && E * K < (1ll << 31);
}

void launch_gemm_bias_gelu_batched(const void* A, const void* B, const float* bias, void* z, void* h, int64_t E,
                                   int64_t M, int64_t N, int64_t K, int sm_count, cudaStream_t stream) {
  M4T_CHECK(batched_gemm_supported(E, M, N, K, A, B, z) && aligned16(h) && epilogue_bias_ok(bias),
            "unsupported shape/alignment for the batched bias+GELU GEMM");
  MlpEpiArgs e{};
  e.bias = bias;
  e.h_out = h;
  launch<false, kBiasGelu, false, true>(sm_count, make_tmap(A, E * M, K, K, BM), make_tmap(B, E * N, K, K, tile_n<false>()),
                                 batched_args(z, E, M, N, K), stream, "gemm_bias_gelu_batched", e);
}

void launch_gemm_bias_batched(const void* A, const void* B, const float* bias, void* y, int64_t E, int64_t M, int64_t N,
                              int64_t K, int sm_count, cudaStream_t stream) {
  M4T_CHECK(batched_gemm_supported(E, M, N, K, A, B, y) && epilogue_bias_ok(bias),
            "unsupported shape/alignment for the batched bias GEMM");
  MlpEpiArgs e{};
  e.bias = bias;
  launch<false, kBias, false, true>(sm_count, make_tmap(A, E * M, K, K, BM), make_tmap(B, E * N, K, K, tile_n<false>()),
                             batched_args(y, E, M, N, K), stream, "gemm_bias_batched", e);
}

void launch_gemm_nn_gelu_bwd_colsum_batched(const void* A, const void* B, const void* z, void* dz, float* colsum,
                                            int64_t E, int64_t M, int64_t N, int64_t K, int sm_count, cudaStream_t stream,
                                            const float* gscale) {
  M4T_CHECK(batched_gemm_supported(E, M, N, K, A, B, dz) && epilogue_bf16_pairs_ok(z, N),
            "unsupported shape/alignment for the batched GELU-backward GEMM");
  GemmArgs g = batched_args(dz, E, M, N, K);
  g.T = z;
  g.ldt = static_cast<int>(N);
  MlpEpiArgs e{};
  e.colsum = colsum;
  e.gscale = gscale;
  launch<false, kGeluBwdColsum, true, true>(sm_count, make_tmap(A, E * M, K, K, BM), make_tmap_bf16_sw128(B, E * K, N, N, 64, BK),
                                     g, stream, "gemm_nn_gelu_bwd_colsum_batched", e);
}

void launch_gemm_nn_batched(const void* A, const void* B, void* C, int64_t E, int64_t M, int64_t N, int64_t K,
                            int sm_count, cudaStream_t stream) {
  M4T_CHECK(batched_gemm_supported(E, M, N, K, A, B, C), "unsupported shape/alignment for the batched NN GEMM");
  launch<false, kStore, true, true>(sm_count, make_tmap(A, E * M, K, K, BM), make_tmap_bf16_sw128(B, E * K, N, N, 64, BK),
                             batched_args(C, E, M, N, K), stream, "gemm_nn_batched");
}

void launch_column_sum_batched(const float* partial, int64_t E, int64_t rows, int64_t N, float* out, const float* gscale,
                               cudaStream_t stream) {
  M4T_CHECK(E > 0 && E < 65536 && rows > 0 && N > 0 && N < (1ll << 31) && rows * N < (1ll << 31),
            "column_sum_batched: empty or oversized workspace");
  const dim3 grid(static_cast<unsigned>((N + 31) / 32), static_cast<unsigned>(E));
  launch_kernel<column_sum_kernel<true>>(grid, 256, 0, stream, "column_sum_batched", partial, static_cast<int>(rows),
                                         static_cast<int>(N), out, gscale);
}

// ---- grouped experts ---------------------------------------------------------------------------------------------
// A [R, K] in the grouped layout of `counts` (GroupTable), B [E, N, K] (TN) or [E, K, N] (NN), C [R, N], bias [E, N].
// The tile space is all R / 128 m-blocks, so C is fully written: rows past a group's count and behind the last group
// are zero.
namespace {

GemmArgs grouped_args(void* C, const int* counts, int64_t E, int64_t R, int64_t N, int64_t K) {
  GemmArgs g = plain_args(C, R, N, K, N);
  g.group_counts = counts;
  g.groups = static_cast<int>(E);
  return g;
}

// Expert e sums rows [first_e, first_e + n_e) of in [.., N] (fp32, or bf16 read as fp32) into out[e] in column_sum's
// order, with first_e = start_e / row_div and n_e = ceil((end_e - start_e) / row_div) from the grouped layout of
// `counts` over R rows.  row_div 16 reduces the GELU-backward epilogue's column-sum partials, row_div 1 the rows
// themselves.  No atomics: the same bits on every call.
template <typename T>
__global__ void __launch_bounds__(256) grouped_column_sum_kernel(const T* __restrict__ in, int N, const int* counts,
                                                                 int R, int row_div, float* __restrict__ out) {
  __shared__ float part[8][33];
  __shared__ int span[2];
  if (threadIdx.x == 0) {
    int p = 0, start = 0, end = 0;
    for (int e = 0; e <= static_cast<int>(blockIdx.y); ++e) {  // build_group_table's rule, up to this group
      const int c = min(max(counts[e], 0), R);
      start = p * BM;
      p = min(p + (c + BM - 1) / BM, R / BM);
      end = min(start + c, R);
    }
    span[0] = start / row_div;
    span[1] = (end - start + row_div - 1) / row_div;
  }
  __syncthreads();
  const int first = span[0], rows = span[1];
  out += static_cast<int64_t>(blockIdx.y) * N;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int n = blockIdx.x * 32 + tx;
  float s = 0.f;
  if (n < N)
    for (int i = ty; i < rows; i += 8) {
      const T v = in[static_cast<int64_t>(first + i) * N + n];
      if constexpr (sizeof(T) == 2) s += bf16_bits_to_float(v);
      else s += v;
    }
  part[ty][tx] = s;
  __syncthreads();
  if (ty == 0 && n < N) {
    float t = part[0][tx];
#pragma unroll
    for (int k = 1; k < 8; ++k) t += part[k][tx];
    out[n] = t;
  }
}

}  // namespace

bool grouped_gemm_supported(int64_t E, int64_t R, int64_t N, int64_t K, const void* A, const void* B, const void* C,
                            const void* counts) {
  return E > 0 && E <= kMaxGroups && R > 0 && N > 0 && K > 0 && R % BM == 0 && N % 128 == 0 && K % 128 == 0 &&
         aligned16(A) && aligned16(B) && aligned16(C) && (reinterpret_cast<uintptr_t>(counts) & 3u) == 0 &&
         R < (1ll << 31) && R / BM * ((N + tile_n<false>() - 1) / tile_n<false>()) < (1ll << 31) && E * N < (1ll << 31) &&
         E * K < (1ll << 31);
}

void launch_gemm_bias_gelu_grouped(const void* A, const void* B, const float* bias, void* z, void* h, const int* counts,
                                   int64_t E, int64_t R, int64_t N, int64_t K, int sm_count, cudaStream_t stream) {
  M4T_CHECK(grouped_gemm_supported(E, R, N, K, A, B, z, counts) && aligned16(h) && epilogue_bias_ok(bias),
            "unsupported shape/alignment for the grouped bias+GELU GEMM");
  MlpEpiArgs e{};
  e.bias = bias;
  e.h_out = h;
  launch<false, kBiasGelu, false, false, true>(sm_count, make_tmap(A, R, K, K, BM), make_tmap(B, E * N, K, K, tile_n<false>()),
                                               grouped_args(z, counts, E, R, N, K), stream, "gemm_bias_gelu_grouped", e);
}

void launch_gemm_bias_grouped(const void* A, const void* B, const float* bias, void* y, const int* counts, int64_t E,
                              int64_t R, int64_t N, int64_t K, int sm_count, cudaStream_t stream) {
  M4T_CHECK(grouped_gemm_supported(E, R, N, K, A, B, y, counts) && epilogue_bias_ok(bias),
            "unsupported shape/alignment for the grouped bias GEMM");
  MlpEpiArgs e{};
  e.bias = bias;
  launch<false, kBias, false, false, true>(sm_count, make_tmap(A, R, K, K, BM), make_tmap(B, E * N, K, K, tile_n<false>()),
                                           grouped_args(y, counts, E, R, N, K), stream, "gemm_bias_grouped", e);
}

void launch_gemm_nn_gelu_bwd_colsum_grouped(const void* A, const void* B, const void* z, void* dz, float* colsum,
                                            const int* counts, int64_t E, int64_t R, int64_t N, int64_t K, int sm_count,
                                            cudaStream_t stream) {
  M4T_CHECK(grouped_gemm_supported(E, R, N, K, A, B, dz, counts) && epilogue_bf16_pairs_ok(z, N),
            "unsupported shape/alignment for the grouped GELU-backward GEMM");
  GemmArgs g = grouped_args(dz, counts, E, R, N, K);
  g.T = z;
  g.ldt = static_cast<int>(N);
  MlpEpiArgs e{};
  e.colsum = colsum;
  launch<false, kGeluBwdColsum, true, false, true>(sm_count, make_tmap(A, R, K, K, BM),
                                                   make_tmap_bf16_sw128(B, E * K, N, N, 64, BK), g, stream,
                                                   "gemm_nn_gelu_bwd_colsum_grouped", e);
}

void launch_gemm_nn_grouped(const void* A, const void* B, void* C, const int* counts, int64_t E, int64_t R, int64_t N,
                            int64_t K, int sm_count, cudaStream_t stream) {
  M4T_CHECK(grouped_gemm_supported(E, R, N, K, A, B, C, counts), "unsupported shape/alignment for the grouped NN GEMM");
  launch<false, kStore, true, false, true>(sm_count, make_tmap(A, R, K, K, BM), make_tmap_bf16_sw128(B, E * K, N, N, 64, BK),
                                           grouped_args(C, counts, E, R, N, K), stream, "gemm_nn_grouped");
}

void launch_column_sum_grouped(const void* in, bool bf16_rows, const int* counts, int64_t E, int64_t R, int64_t N,
                               float* out, cudaStream_t stream) {
  M4T_CHECK(E > 0 && E <= kMaxGroups && R > 0 && R % BM == 0 && N > 0 && R * N < (1ll << 31),
            "column_sum_grouped: empty or oversized input");
  const dim3 grid(static_cast<unsigned>((N + 31) / 32), static_cast<unsigned>(E));
  if (bf16_rows)
    launch_kernel<grouped_column_sum_kernel<uint16_t>>(grid, 256, 0, stream, "row_sum_grouped",
                                                       static_cast<const uint16_t*>(in), static_cast<int>(N), counts,
                                                       static_cast<int>(R), 1, out);
  else
    launch_kernel<grouped_column_sum_kernel<float>>(grid, 256, 0, stream, "column_sum_grouped",
                                                    static_cast<const float*>(in), static_cast<int>(N), counts,
                                                    static_cast<int>(R), 16, out);
}

}  // namespace m4t
