// Weight-gradient GEMM on wgmma, optionally fused with the gradient all-reduce and
// the SGD update, or accumulated into an fp32 gradient buffer.
//
//   G[N,K] = dY[Mb,N]^T * X[Mb,K]          (bf16 in, fp32 accumulate in registers)
//
// The contraction runs over the batch dimension Mb, which is the STRIDED
// dimension of both row-major operands, so both wgmma operands are MN-major:
// TMA boxes are {64 contiguous elements (128 B swizzle span), BK batch rows} and
// the shared-memory descriptors use the MN-major SWIZZLE_128B canonical layout
// (LBO = one 64-wide chunk = BK*128 B, SBO = one 8-row swizzle atom = 1024 B);
// the wgmma transpose bits select MN-major A and B.  No transposed copy of dY or
// X is ever made.  Pipeline: wgmma_pipeline.cuh (128x256 tiles, 128x128 in the fused kernel).
//
// Fused mode (the backward of the data-parallel linear layer, where the
// reference does wgrad GEMM -> MPI_Allreduce -> optimizer step as three passes
// over the gradient, csrc/extension.cpp:197-260 + the example's SGD loop):
//   * tiles that fill whole waves of the CTAs run over the full batch; only the
//     tiles of the last, partial wave are split in `ksplit` batch halves, so
//     only those tiles produce two partial buffers;
//   * the epilogue writes each partial tile as bf16 into the staging buffer and
//     bumps the tile's counter ON THE OWNER rank (tile t is owned by rank
//     t % P) with a release-scoped remote red;
//   * four communication warps per CTA wait for owned tiles to be complete on
//     all ranks, pull the sum through the NVSwitch (multimem.ld_reduce), apply
//     W -= lr/P * sum in fp32 and multicast the new bf16 weights into every
//     rank's copy (multimem.st) - reduce-scatter + update + all-gather, hidden
//     under the GEMM of later tiles;
//   * a multicast "done" counter makes kernel completion imply that every
//     rank's weights are final.
#include <cuda.h>

#include <atomic>

#include "kernels.h"
#include "tma_host.h"
#include "wgmma_pipeline.cuh"

namespace m4t {

namespace {

using namespace wg;

constexpr int kSignalsPerUnit = kConsumerWarps;  // every consumer warp of the CTA arrives on the tile counter
constexpr int kMaxUnicastRanks = 3;  // peer-load mode keeps ranks x rows x partial buffers requests in registers

struct WgradArgs {
  void* out;            // plain: G [N, K] (bf16; fp32 when ACC32); fused: unused (the staging buffers live in
                        // the heaps of WgradComm)
  int Mb, N, K;
  int ldo;              // leading dimension of out (elements)
  union {
    int ksplit;
    const int* group_counts;  // GROUPED (ksplit 1): [experts] rows of each group, int32 on the device.  The slot of
                              // ksplit and its padding, so the parameter layout is unchanged.
  };
  const float* gscale;  // optional device scalar multiplied into every output element (the upstream
                        // gradient of the loss: autograd hands it over as a tensor, never through the host)
  float axpy;           // plain mode with axpy != 0: out <- out + axpy * gscale * G  (single-rank SGD epilogue)
  int experts;          // BATCHED, GROUPED: E (in the tail padding: the other kernels' parameter layout is unchanged)
};

struct WgradComm {
  SyncCtx sync;
  char* heap[kMaxGpuPeers];
  char* mc_heap;
  int64_t stage_off;     // partial-gradient staging (same offset on every rank)
  int64_t stage_stride;  // bytes between the ksplit partial buffers
  int64_t src_stride;    // peer-store mode: bytes between the per-source-rank copies of the staging area in the
                         // OWNER's heap (the epilogue pushes its partial tile there; the owner only reads locally)
  int64_t w_off;         // bf16 weights [N, K] (contiguous) inside every rank's heap
  int64_t cnt_off;       // u32 tile counters [tiles]
  int64_t done_off;      // u32 completion counter
  uint32_t tile_target;  // counters are monotonic: targets of THIS call when epoch_off < 0 ...
  uint32_t done_target;
  int64_t epoch_off;     // ... otherwise per-call increments; the call index is read from this local
                         // device word (and advanced by the kernel), which makes the launch graph-capturable
  float scale;           // W += scale * sum_ranks G   (scale = -lr / P)
  // optional: all-reduce the UPDATED weights for the next forward while the GEMM is still running
  int prefetch;          // 1: W_avg[tile] = avg_scale * sum_ranks W[tile] after the update of the tile
  int64_t wavg_off;      // bf16 [N, K] buffer receiving the averaged weights on every rank
  float avg_scale;       // 1 / P
  int unicast;           // 1: peer loads / peer stores instead of multimem (no NVLS, or too few ranks for it to pay)
  int debug;             // timing experiments (M4T_WGRAD_DEBUG): 1 no comm data movement, 2 no GEMM,
                         // 4 local loads instead of multimem.ld_reduce, 8 local stores instead of multimem.st,
                         // 16 no tile signals and no owner work, 32 no completion barrier
};

// Work-unit schedule shared by every role (and by the host for the counter targets): tiles
// [0, whole) run over the full batch, tiles [whole, num_tiles) are split in `split` batch slices.
struct UnitSched {
  int whole, split, num_units;
};
__host__ __device__ inline UnitSched make_sched(int num_tiles, int num_ctas, int ksplit) {
  UnitSched s;
  s.split = ksplit;
  s.whole = ksplit > 1 ? (num_tiles / num_ctas) * num_ctas : num_tiles;
  s.num_units = s.whole + (num_tiles - s.whole) * ksplit;
  return s;
}
// unit u -> tile t, slice h of `parts` slices
__host__ __device__ inline void unit_to_tile(const UnitSched& s, int u, int& t, int& h, int& parts) {
  if (u < s.whole) {
    t = u;
    h = 0;
    parts = 1;
  } else {
    const int j = u - s.whole;
    t = s.whole + j / s.split;
    h = j - (j / s.split) * s.split;
    parts = s.split;
  }
}

// Owner side of the fused mode; runs on kCommWarps warps of every CTA.
// MC: reduce through the NVSwitch (multimem.ld_reduce / multimem.st); otherwise NSRC peer loads in rank
// order and one store per peer (2-3 ranks, or no multicast mapping).
// A tile row is 128 * 2 = 256 bytes: half a warp (16 lanes x 16 bytes) per row, two rows per warp access.
template <bool MC, int NSRC>
__device__ __forceinline__ void comm_reduce_update(const WgradComm& wc, int first_thread, int num_tiles, int k_tiles,
                                                   int K, const UnitSched sched) {
  const SyncCtx& c = wc.sync;
  const int P = c.size, r = c.rank;
  const int ct = threadIdx.x - first_thread;
  const int lane = ct & 31;
  const int cw = ct >> 5;
  constexpr int kCommThreads = kCommWarps * 32;
  constexpr int kU = NSRC <= 2 ? 4 : 2;  // row pairs in flight per warp (x partial buffers x peers independent round trips)
  constexpr int kRowSplit = 2;    // CTAs sharing one owned tile: shortens the tail after the last GEMM wave
  constexpr int kPairs = BM / kRowSplit / 2;  // row pairs of one work item
  const uint32_t* my_cnt = reinterpret_cast<const uint32_t*>(wc.heap[r] + wc.cnt_off);
  const int64_t row_bytes = static_cast<int64_t>(K) * 2;
  // device-resident call counter: every communication thread reads it before any CTA can pass the
  // completion barrier below, and only CTA 0 advances it after that barrier
  uint32_t* epoch_ptr = wc.epoch_off >= 0 ? reinterpret_cast<uint32_t*>(wc.heap[r] + wc.epoch_off) : nullptr;
  const uint32_t epoch = epoch_ptr ? *reinterpret_cast<volatile uint32_t*>(epoch_ptr) : 0u;
  const uint32_t calls = epoch_ptr ? epoch + 1u : 1u;
  const uint32_t done_target = epoch_ptr ? calls * wc.done_target : wc.done_target;
  const bool skip = (wc.debug & 1) != 0;
  // Work item w = (j-th owned tile, row slice s); item w is served by CTA w % gridDim.x.
  // Owned tiles (t = r + j*P) finish in GEMM order, so consecutive items land on different CTAs
  // and their round trips overlap.
  const int owned = r < num_tiles ? (num_tiles - r + P - 1) / P : 0;
  for (int w_item = blockIdx.x; w_item < owned * kRowSplit && !(wc.debug & 16); w_item += gridDim.x) {
    const int j = w_item / kRowSplit;
    const int slice = w_item - j * kRowSplit;
    const int t = r + j * P;
    const int parts = t < sched.whole ? 1 : sched.split;
    // every rank's `parts` partial tiles are complete: kSignalsPerUnit signals per unit and rank, per call
    const uint32_t tile_target = (epoch_ptr ? calls : 1u) * wc.tile_target * static_cast<uint32_t>(parts);
    if (lane == 0) bounded_wait_ge(my_cnt + t, tile_target, c);
    __syncwarp();
    const int n_blk = t / k_tiles;
    const int k_blk = t - n_blk * k_tiles;
    // this item's rows: kPairs pairs x 2 rows x 256 bytes
    const int64_t tile_off = (static_cast<int64_t>(n_blk) * BM + slice * (2 * kPairs) + (lane >> 4)) * row_bytes +
                             static_cast<int64_t>(k_blk) * tile_n<true>() * 2 + (lane & 15) * 16;
    for (int pair0 = cw; pair0 < kPairs && !skip; pair0 += kCommWarps * kU) {
      // all loads of the kU row pairs (x partial buffers x peers) are issued before the first one is consumed
      constexpr int kSrc = NSRC;
      Vec16 s[kU][kSrc][2], w[kU];
#pragma unroll
      for (int u = 0; u < kU; ++u) {
        const int pair = pair0 + u * kCommWarps;
        if (pair < kPairs) {
          const int64_t off = tile_off + 2 * pair * row_bytes;
          if (MC) {
            if (wc.debug & 4) {
              s[u][0][0] = ld_vec(wc.heap[r] + wc.stage_off + off);
              if (parts > 1) s[u][0][1] = ld_vec(wc.heap[r] + wc.stage_off + wc.stage_stride + off);
            } else {
              s[u][0][0] = multimem_ld_reduce_vec<NvlsKind::ADD_BF16>(wc.mc_heap + wc.stage_off + off);
              if (parts > 1) s[u][0][1] = multimem_ld_reduce_vec<NvlsKind::ADD_BF16>(wc.mc_heap + wc.stage_off + wc.stage_stride + off);
            }
          } else {
#pragma unroll
            for (int p = 0; p < kSrc; ++p) {
              if (p < P) {
                // pushed here by rank p's epilogue: local reads
                const char* src = wc.heap[r] + wc.stage_off + static_cast<int64_t>(p) * wc.src_stride + off;
                s[u][p][0] = ld_vec(src);
                if (parts > 1) s[u][p][1] = ld_vec(src + wc.stage_stride);
              }
            }
          }
          w[u] = ld_vec(wc.heap[r] + wc.w_off + off);
        }
      }
#pragma unroll
      for (int u = 0; u < kU; ++u) {
        const int pair = pair0 + u * kCommWarps;
        if (pair < kPairs) {
          const int64_t off = tile_off + 2 * pair * row_bytes;
          float a[8], b[8], wv[8];
#pragma unroll
          for (int e = 0; e < 8; ++e) a[e] = 0.f;
#pragma unroll
          for (int p = 0; p < kSrc; ++p) {  // fixed rank order: every run adds in the same order
            if (MC || p < P) {
              VecOf<DType::BF16>::unpack(s[u][p][0], b);
#pragma unroll
              for (int e = 0; e < 8; ++e) a[e] += b[e];
              if (parts > 1) {
                VecOf<DType::BF16>::unpack(s[u][p][1], b);
#pragma unroll
                for (int e = 0; e < 8; ++e) a[e] += b[e];
              }
            }
          }
          VecOf<DType::BF16>::unpack(w[u], wv);
#pragma unroll
          for (int e = 0; e < 8; ++e) wv[e] = fmaf(wc.scale, a[e], wv[e]);
          const Vec16 o = VecOf<DType::BF16>::pack(wv);
          if (MC && !(wc.debug & 8)) {
            multimem_st_vec(wc.mc_heap + wc.w_off + off, o);
          } else if (MC) {
            st_vec(wc.heap[r] + wc.w_off + off, o);
          } else {
#pragma unroll
            for (int p = 0; p < kSrc; ++p)
              if (p < P) st_vec(wc.heap[p] + wc.w_off + off, o);
          }
        }
      }
    }
    if (wc.prefetch && !skip) {
      // Next step's forward needs Allreduce(W) / P.  The rows this lane just wrote into every rank's
      // copy are the final values of this step, so the parameter all-reduce of the NEXT step can run here,
      // under the GEMM of later tiles.  Every address read below was written above by THIS lane:
      //  * peer-store mode: plain stores followed by loads of the same addresses - program order to the
      //    same location from one thread is coherent without a fence;
      //  * multicast mode: the write fans out inside the switch, so the fence stays.
      if (MC) __threadfence_system();
      for (int pair0 = cw; pair0 < kPairs; pair0 += kCommWarps * kU) {
        constexpr int kSrc = NSRC;
        Vec16 x[kU][kSrc];
#pragma unroll
        for (int u = 0; u < kU; ++u) {
          const int pair = pair0 + u * kCommWarps;
          if (pair < kPairs) {
            const int64_t off = tile_off + 2 * pair * row_bytes;
            if (MC) {
              x[u][0] = multimem_ld_reduce_vec<NvlsKind::ADD_BF16>(wc.mc_heap + wc.w_off + off);
            } else {
#pragma unroll
              for (int p = 0; p < kSrc; ++p)
                if (p < P) x[u][p] = ld_vec_sys(wc.heap[p] + wc.w_off + off);
            }
          }
        }
#pragma unroll
        for (int u = 0; u < kU; ++u) {
          const int pair = pair0 + u * kCommWarps;
          if (pair < kPairs) {
            const int64_t off = tile_off + 2 * pair * row_bytes;
            float a[8], b[8];
#pragma unroll
            for (int e = 0; e < 8; ++e) a[e] = 0.f;
#pragma unroll
            for (int p = 0; p < kSrc; ++p) {
              if (MC || p < P) {
                VecOf<DType::BF16>::unpack(x[u][p], b);
#pragma unroll
                for (int e = 0; e < 8; ++e) a[e] += b[e];
              }
            }
#pragma unroll
            for (int e = 0; e < 8; ++e) a[e] *= wc.avg_scale;
            const Vec16 o = VecOf<DType::BF16>::pack(a);
            if (MC) {
              multimem_st_vec(wc.mc_heap + wc.wavg_off + off, o);
            } else {
#pragma unroll
              for (int p = 0; p < kSrc; ++p)
                if (p < P) st_vec(wc.heap[p] + wc.wavg_off + off, o);
            }
          }
        }
      }
    }
  }
  // completion: every CTA of every rank reports once; leaving the kernel means all weights are final
  asm volatile("bar.sync 1, %0;" ::"n"(kCommThreads));
  if (ct == 0 && !(wc.debug & 32)) {
    if (MC) {
      asm volatile("multimem.red.release.sys.global.add.u32 [%0], %1;" ::"l"(wc.mc_heap + wc.done_off), "r"(1u) : "memory");
    } else {
      __threadfence_system();
      for (int p = 0; p < P; ++p)
        asm volatile("red.release.sys.global.add.u32 [%0], %1;" ::"l"(wc.heap[p] + wc.done_off), "r"(1u) : "memory");
    }
    bounded_wait_ge(reinterpret_cast<const uint32_t*>(wc.heap[r] + wc.done_off), done_target, c);
    if (epoch_ptr && blockIdx.x == 0) *reinterpret_cast<volatile uint32_t*>(epoch_ptr) = epoch + 1u;
  }
  asm volatile("bar.sync 1, %0;" ::"n"(kCommThreads));
}

// Epilogues of one consumer warpgroup's 64 rows of the tile (n_blk, k_blk) of out (leading dimension ldo, K columns).
// The tile's columns are a multiple of 128: a last tile of K may be half.
// bf16 out <- gs * acc, or out <- out + gs * acc when axpy.
template <int BN>
__device__ __forceinline__ void bf16_epilogue(const float (&acc)[BN / 2], char* obase, int ldo, int K, float gs, bool axpy,
                                              int n_blk, int k_blk, int wgi) {
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    const int row = n_blk * BM + wgi * 64 + frag_row(hr);
    uint16_t* orow = reinterpret_cast<uint16_t*>(obase) + static_cast<int64_t>(row) * ldo + k_blk * BN;
    const int cols = min(BN, K - k_blk * BN);
#pragma unroll
    for (int j0 = 0; j0 < BN / 8; j0 += 8) {
      if (j0 * 8 >= cols) continue;
      uint32_t prev[8];
      if (axpy) {  // the eight pieces of the row are requested before any is consumed
#pragma unroll
        for (int j = 0; j < 8; ++j) prev[j] = *reinterpret_cast<const uint32_t*>(orow + frag_col(j0 + j));
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        float v0 = gs * acc[4 * (j0 + j) + 2 * hr], v1 = gs * acc[4 * (j0 + j) + 2 * hr + 1];
        if (axpy) {
          v0 += bf16_bits_to_float(static_cast<uint16_t>(prev[j] & 0xffffu));
          v1 += bf16_bits_to_float(static_cast<uint16_t>(prev[j] >> 16));
        }
        *reinterpret_cast<uint32_t*>(orow + frag_col(j0 + j)) = pack_bf16x2(v0, v1);
      }
    }
  }
}

// fp32 out <- fmaf(gs, acc, out): ONE rounding per micro-batch (the product is not rounded on its own), so a
// contribution far below the buffer's ulp still moves it by its correctly rounded share.
template <int BN>
__device__ __forceinline__ void acc32_epilogue(const float (&acc)[BN / 2], char* obase, int ldo, int K, float gs,
                                               int n_blk, int k_blk, int wgi) {
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    const int row = n_blk * BM + wgi * 64 + frag_row(hr);
    float* orow = reinterpret_cast<float*>(obase) + static_cast<int64_t>(row) * ldo + k_blk * BN;
    const int cols = min(BN, K - k_blk * BN);
#pragma unroll
    for (int j0 = 0; j0 < BN / 8; j0 += 8) {
      if (j0 * 8 >= cols) continue;
      float2 prev[8];  // the eight column pairs of the row are requested before any is consumed
#pragma unroll
      for (int j = 0; j < 8; ++j) prev[j] = *reinterpret_cast<const float2*>(orow + frag_col(j0 + j));
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float2 o = make_float2(fmaf(gs, acc[4 * (j0 + j) + 2 * hr], prev[j].x),
                                     fmaf(gs, acc[4 * (j0 + j) + 2 * hr + 1], prev[j].y));
        *reinterpret_cast<float2*>(orow + frag_col(j0 + j)) = o;
      }
    }
  }
}

// The grouped wgrad (wgrad_bf16_wgmma_kernel with GROUPED): tile t of E * n_tiles * k_tiles is (expert, n, k) as in the
// batched kernel, contracted over the expert's rows [128 pfx[e], end[e]) of the grouped layout.  The epilogue is chosen
// at compile time: G (bf16), the SGD step W <- bf16(W + g.axpy * gscale * G) (SGD), or the fp32 accumulation (ACC32).
// In the two updating modes an expert without rows stores nothing, so its weight or buffer keeps its exact bits.
template <int BN, bool ACC32, bool SGD>
__device__ __forceinline__ void grouped_wgrad_roles(uint8_t* smem, Pipe* pipe, const CUtensorMap* tmap_a,
                                                    const CUtensorMap* tmap_b, const WgradArgs& g, int n_tiles,
                                                    int k_tiles) {
  GroupTable* grp = group_table_of(pipe);
  const int warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) {
    tc::prefetch_tmap(tmap_a);
    tc::prefetch_tmap(tmap_b);
    init_pipe<BN>(pipe);
  }
  if (threadIdx.x == 32) build_group_table(grp, g.group_counts, g.experts, g.Mb);
  __syncthreads();
  const int num_tiles = n_tiles * k_tiles * g.experts;
  if (warp < 4) {
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
        const int n_blk = t / k_tiles;
        const int k_blk = t - n_blk * k_tiles;
        const int expert = n_blk / n_tiles;
        const int row0 = grp->pfx[expert] * BM;
        const int kbs = (max(grp->end[expert] - row0, 0) + BK - 1) / BK;
        for (int kb = 0; kb < kbs; ++kb)
          load_stage<true, true, BN>(smem, pipe, stage, phase, tmap_a, tmap_b, (n_blk - expert * n_tiles) * BM,
                                     k_blk * BN, row0 + kb * BK);
      }
    }
  } else {
    const int wgi = warp / 4 - 1;
    int stage = 0;
    uint32_t phase = 0;
    float acc[BN / 2];
    // SGD: the plain kernel's axpy scale, (gscale * axpy), so both round the same products
    const float gs = SGD ? (g.gscale ? __ldg(g.gscale) : 1.0f) * g.axpy : (g.gscale ? __ldg(g.gscale) : 1.0f);
    for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
      const int n_blk = t / k_tiles;
      const int k_blk = t - n_blk * k_tiles;
      const int expert = n_blk / n_tiles;
      const int rows = max(grp->end[expert] - grp->pfx[expert] * BM, 0);
      const int kbs = (rows + BK - 1) / BK;
      if (kbs > 0) {
        mma_tile<true, true, BN, true>(acc, smem, pipe, stage, phase, kbs, wgi, rows - (kbs - 1) * BK);
        if constexpr (ACC32) acc32_epilogue<BN>(acc, static_cast<char*>(g.out), g.ldo, g.K, gs, n_blk, k_blk, wgi);
        else bf16_epilogue<BN>(acc, static_cast<char*>(g.out), g.ldo, g.K, gs, SGD, n_blk, k_blk, wgi);
        continue;
      }
      if constexpr (ACC32 || SGD) continue;  // updating modes: an expert without rows leaves its tile untouched
      // an expert without rows: a zero gradient (zeroing acc instead makes ptxas spill it)
      const int cols = min(BN, g.K - k_blk * BN);
#pragma unroll 1
      for (int hr = 0; hr < 2; ++hr) {
        uint16_t* orow = static_cast<uint16_t*>(g.out) + static_cast<int64_t>(n_blk * BM + wgi * 64 + frag_row(hr)) * g.ldo +
                         k_blk * BN;
#pragma unroll 1
        for (int j = 0; j < cols / 8; ++j) *reinterpret_cast<uint32_t*>(orow + frag_col(j)) = 0u;
      }
    }
  }
  __syncthreads();
}

// ACC32 (not FUSED): out is an fp32 [N, K] buffer and the epilogue is out <- fmaf(gscale, G, out), the
// gradient accumulation of micro-batches.  A compile-time mode, so the other instantiations are unchanged.
// BATCHED (not FUSED): E = g.experts problems G_e = dY_e^T X_e of the same shape, with dY [E Mb, N], X [E Mb, K]
// and out [E N, K] stacked.  Tile rows of the stacked output run over E * N / 128 blocks: block n_blk belongs to
// expert n_blk / (N / 128), whose contraction rows start at row expert * Mb of both operands.
// GROUPED (not FUSED, not BATCHED): the same tiles and output, with dY [Mb, N] and X [Mb, K] in the grouped layout of
// g.group_counts over Mb rows (GroupTable).  Expert e contracts over the ceil(rows_e / 64) k-blocks from its first
// row; the last one's rows past the group are zeroed in both operands, and an expert without rows stores zeros (G) or
// nothing (ACC32, SGD).
// SGD (GROUPED only): the SGD epilogue out <- bf16(out + axpy * gscale * G) as a compile-time mode; the other kernels
// select it at run time through g.axpy.
template <bool FUSED, bool ACC32 = false, bool BATCHED = false, bool GROUPED = false, bool SGD = false>
__global__ void __launch_bounds__(kGemmThreads + (FUSED ? kCommWarps * 32 : 0), 1)
wgrad_bf16_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                        const WgradArgs g, const WgradComm wc) {
  static_assert(!GROUPED || (!FUSED && !BATCHED && !(ACC32 && SGD)), "grouped wgrad: one epilogue, not fused");
  static_assert(!SGD || GROUPED, "the compile-time SGD epilogue is the grouped kernel's");
  constexpr int BN = tile_n<FUSED>();
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = aligned_smem(smem_raw);
  Pipe* pipe = pipe_of<BN>(smem);
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  const int n_tiles = g.N / BM;  // tiles along the rows of G
  const int k_tiles = (g.K + BN - 1) / BN;  // tiles along the columns of G (K % 128 == 0: a last tile may be half)
  if constexpr (GROUPED) {
    grouped_wgrad_roles<BN, ACC32, SGD>(smem, pipe, &tmap_a, &tmap_b, g, n_tiles, k_tiles);
    return;
  }
  const int num_tiles = n_tiles * k_tiles * (BATCHED ? g.experts : 1);
  const UnitSched sched = make_sched(num_tiles, gridDim.x, g.ksplit);
  const int num_units = sched.num_units;
  const int kb_total = g.Mb / BK;

  if (warp == 0 && lane == 0) {
    tc::prefetch_tmap(&tmap_a);
    tc::prefetch_tmap(&tmap_b);
    init_pipe<BN>(pipe);
  }
  __syncthreads();

  if (warp < 4) {
    // =========================== TMA producer ===========================
    if (warp == 0 && lane == 0 && !(FUSED && (wc.debug & 2))) {
      int stage = 0;
      uint32_t phase = 0;
      for (int u = blockIdx.x; u < num_units; u += gridDim.x) {
        int t, h, parts;
        unit_to_tile(sched, u, t, h, parts);
        const int kb_per_unit = kb_total / parts;
        const int n_blk = t / k_tiles;
        const int k_blk = t - n_blk * k_tiles;
        const int expert = BATCHED ? n_blk / n_tiles : 0;
        for (int kb = 0; kb < kb_per_unit; ++kb)
          load_stage<true, true, BN>(smem, pipe, stage, phase, &tmap_a, &tmap_b, (n_blk - expert * n_tiles) * BM,
                                     k_blk * BN, expert * g.Mb + (h * kb_per_unit + kb) * BK);
      }
    }
  } else if (warp < kGemmThreads / 32) {
    // ====================== consumers: wgmma + epilogue ======================
    const int wgi = warp / 4 - 1;
    int stage = 0;
    uint32_t phase = 0;
    float acc[BN / 2];
    const int r = wc.sync.rank;
    for (int u = blockIdx.x; u < num_units; u += gridDim.x) {
      int t, h, parts;
      unit_to_tile(sched, u, t, h, parts);
      const int n_blk = t / k_tiles;
      const int k_blk = t - n_blk * k_tiles;
      const int owner = FUSED ? t % wc.sync.size : 0;
      if (FUSED && (wc.debug & 2)) {  // timing experiment: no GEMM, only the tile signals
        __syncwarp();
        if (lane == 0) {
          uint32_t* cnt = reinterpret_cast<uint32_t*>(wc.heap[owner] + wc.cnt_off) + t;
          asm volatile("red.release.sys.global.add.u32 [%0], %1;" ::"l"(cnt), "r"(1u) : "memory");
        }
        continue;
      }
      mma_tile<true, true, BN>(acc, smem, pipe, stage, phase, u < sched.whole ? kb_total : kb_total / sched.split, wgi);
      // plain mode: G.  Multicast mode: this rank's own staging buffer.  Peer-store mode: the OWNER's staging area
      // for this source rank - posted writes over NVLink, spread over the whole GEMM, so the owner never has to
      // pull (no read round trips on the reduction path).
      char* obase = static_cast<char*>(g.out);
      int ldo = g.ldo;
      if (FUSED) {
        obase = wc.unicast ? wc.heap[owner] + wc.stage_off + static_cast<int64_t>(r) * wc.src_stride : wc.heap[r] + wc.stage_off;
        obase += h * wc.stage_stride;
        ldo = g.K;
      }
      const float gs = (g.gscale ? __ldg(g.gscale) : 1.0f) * (g.axpy != 0.0f ? g.axpy : 1.0f);
      const bool axpy = !FUSED && g.axpy != 0.0f;
      if constexpr (ACC32) acc32_epilogue<BN>(acc, obase, ldo, g.K, gs, n_blk, k_blk, wgi);
      else bf16_epilogue<BN>(acc, obase, ldo, g.K, gs, axpy, n_blk, k_blk, wgi);
      if (FUSED && !(wc.debug & 16)) {
        // this warp's 16 rows of the partial tile are written: tell the owner.  The release
        // (a system-scope fence + the add) is cumulative over the warp's stores through __syncwarp.
        __syncwarp();
        if (lane == 0) {
          uint32_t* cnt = reinterpret_cast<uint32_t*>(wc.heap[owner] + wc.cnt_off) + t;
          asm volatile("red.release.sys.global.add.u32 [%0], %1;" ::"l"(cnt), "r"(1u) : "memory");
        }
      }
    }
  } else if (FUSED) {
    // ===================== reduce + update =====================
    if (!wc.unicast) comm_reduce_update<true, 1>(wc, kGemmThreads, num_tiles, k_tiles, g.K, sched);
    else if (wc.sync.size <= 2) comm_reduce_update<false, 2>(wc, kGemmThreads, num_tiles, k_tiles, g.K, sched);
    else comm_reduce_update<false, kMaxUnicastRanks>(wc, kGemmThreads, num_tiles, k_tiles, g.K, sched);
  }
  __syncthreads();
}

// Row-major [rows, cols] bf16 tensor, boxes of {64 columns, BK rows}.
CUtensorMap make_tmap_mn(const void* base, int64_t rows, int64_t cols, int64_t ld) {
  return make_tmap_bf16_sw128(base, rows, cols, ld, 64, BK);
}

WgradArgs wgrad_args(void* out, int64_t Mb, int64_t N, int64_t K, int64_t ldo, int ksplit, const float* gscale,
                     float axpy, int64_t experts = 0) {
  WgradArgs g{};
  g.out = out;
  g.Mb = static_cast<int>(Mb);
  g.N = static_cast<int>(N);
  g.K = static_cast<int>(K);
  g.ldo = static_cast<int>(ldo);
  g.ksplit = ksplit;
  g.gscale = gscale;
  g.axpy = axpy;
  g.experts = static_cast<int>(experts);
  return g;
}

}  // namespace

// timing experiments only (scripts/wgrad_diag.py): initial value from M4T_WGRAD_DEBUG, changeable at run time
static std::atomic<int> g_wgrad_debug{static_cast<int>(env_i64("M4T_WGRAD_DEBUG", 0))};
void set_wgrad_debug(int mask) { g_wgrad_debug.store(mask, std::memory_order_relaxed); }

bool wgrad_bf16_supported(int64_t Mb, int64_t N, int64_t K, const void* dy, const void* x, const void* g, int64_t ldy,
                          int64_t ldx, int64_t ldg) {
  return Mb > 0 && N > 0 && K > 0 && N % BM == 0 && K % 128 == 0 && Mb % BK == 0 && aligned16(dy) && aligned16(x) &&
         aligned16(g) && ldy % 8 == 0 && ldx % 8 == 0 && ldg % 8 == 0 && ldy >= N && ldx >= K && ldg >= K &&
         Mb < (1ll << 31) && N < (1ll << 31) && K < (1ll << 31);
}

void launch_wgrad_bf16(const void* dy, const void* x, void* gout, int64_t Mb, int64_t N, int64_t K, int64_t ldy,
                       int64_t ldx, int64_t ldg, int sm_count, cudaStream_t stream, const float* gscale, float axpy) {
  M4T_CHECK(wgrad_bf16_supported(Mb, N, K, dy, x, gout, ldy, ldx, ldg),
            "unsupported wgrad shape/alignment for the wgmma path (N % 128, K % 128, batch % 64)");
  constexpr int BN = tile_n<false>();
  launch_kernel<wgrad_bf16_wgmma_kernel<false>>(
      persistent_grid((N / BM) * ((K + BN - 1) / BN), sm_count), kGemmThreads, Tile<BN>::kSmemBytes, stream,
      axpy != 0.0f ? "wgrad_sgd_epilogue" : "wgrad", make_tmap_mn(dy, Mb, N, ldy), make_tmap_mn(x, Mb, K, ldx),
      wgrad_args(gout, Mb, N, K, ldg, 1, gscale, axpy), WgradComm{});
}

void launch_wgrad_accumulate(const void* dy, const void* x, float* acc, int64_t Mb, int64_t N, int64_t K, int64_t ldy,
                             int64_t ldx, int sm_count, cudaStream_t stream, const float* gscale) {
  M4T_CHECK(wgrad_bf16_supported(Mb, N, K, dy, x, acc, ldy, ldx, K),
            "unsupported wgrad_accumulate shape/alignment (N % 128, K % 128, batch % 64, 16-byte aligned operands)");
  constexpr int BN = tile_n<false>();
  launch_kernel<wgrad_bf16_wgmma_kernel<false, true>>(
      persistent_grid((N / BM) * ((K + BN - 1) / BN), sm_count), kGemmThreads, Tile<BN>::kSmemBytes, stream,
      "wgrad_accumulate", make_tmap_mn(dy, Mb, N, ldy), make_tmap_mn(x, Mb, K, ldx),
      wgrad_args(acc, Mb, N, K, K, 1, gscale, 0.0f), WgradComm{});
}

bool wgrad_bf16_batched_supported(int64_t E, int64_t Mb, int64_t N, int64_t K, const void* dy, const void* x,
                                  const void* g) {
  return E > 0 && wgrad_bf16_supported(Mb, N, K, dy, x, g, N, K, K) && E * Mb < (1ll << 31) &&
         E * N / BM * ((K + tile_n<false>() - 1) / tile_n<false>()) < (1ll << 31);
}

void launch_wgrad_bf16_batched(const void* dy, const void* x, void* gout, int64_t E, int64_t Mb, int64_t N, int64_t K,
                               int sm_count, cudaStream_t stream, const float* gscale, float axpy) {
  M4T_CHECK(wgrad_bf16_batched_supported(E, Mb, N, K, dy, x, gout),
            "unsupported shape/alignment for the batched wgrad (N % 128, K % 128, batch % 64, 16-byte-aligned operands)");
  constexpr int BN = tile_n<false>();
  launch_kernel<wgrad_bf16_wgmma_kernel<false, false, true>>(
      persistent_grid(E * (N / BM) * ((K + BN - 1) / BN), sm_count), kGemmThreads, Tile<BN>::kSmemBytes, stream,
      axpy != 0.0f ? "wgrad_sgd_batched" : "wgrad_bf16_batched", make_tmap_mn(dy, E * Mb, N, N),
      make_tmap_mn(x, E * Mb, K, K), wgrad_args(gout, Mb, N, K, K, 1, gscale, axpy, E), WgradComm{});
}

void launch_wgrad_accumulate_batched(const void* dy, const void* x, float* acc, int64_t E, int64_t Mb, int64_t N,
                                     int64_t K, int sm_count, cudaStream_t stream, const float* gscale) {
  M4T_CHECK(wgrad_bf16_batched_supported(E, Mb, N, K, dy, x, acc),
            "unsupported shape/alignment for the batched wgrad (N % 128, K % 128, batch % 64, 16-byte-aligned operands)");
  constexpr int BN = tile_n<false>();
  launch_kernel<wgrad_bf16_wgmma_kernel<false, true, true>>(
      persistent_grid(E * (N / BM) * ((K + BN - 1) / BN), sm_count), kGemmThreads, Tile<BN>::kSmemBytes, stream,
      "wgrad_accumulate_batched", make_tmap_mn(dy, E * Mb, N, N), make_tmap_mn(x, E * Mb, K, K),
      wgrad_args(acc, Mb, N, K, K, 1, gscale, 0.0f, E), WgradComm{});
}

bool wgrad_bf16_grouped_supported(int64_t E, int64_t R, int64_t N, int64_t K, const void* dy, const void* x,
                                  const void* g, const void* counts) {
  return E > 0 && E <= kMaxGroups && R % BM == 0 && wgrad_bf16_supported(R, N, K, dy, x, g, N, K, K) &&
         (reinterpret_cast<uintptr_t>(counts) & 3u) == 0 &&
         E * N / BM * ((K + tile_n<false>() - 1) / tile_n<false>()) < (1ll << 31) && E * N < (1ll << 31);
}

namespace {
// Mode of the grouped wgrad: G, the SGD step (axpy != 0) or the fp32 accumulation.
template <bool ACC32, bool SGD>
void launch_grouped(const char* what, const void* dy, const void* x, void* out, const int* counts, int64_t E, int64_t R,
                    int64_t N, int64_t K, int sm_count, cudaStream_t stream, const float* gscale, float axpy) {
  M4T_CHECK(wgrad_bf16_grouped_supported(E, R, N, K, dy, x, out, counts),
            "unsupported shape/alignment for the grouped wgrad (N % 128, K % 128, rows % 128, 16-byte-aligned operands)");
  constexpr int BN = tile_n<false>();
  WgradArgs g = wgrad_args(out, R, N, K, K, 1, gscale, axpy, E);
  g.group_counts = counts;
  launch_kernel<wgrad_bf16_wgmma_kernel<false, ACC32, false, true, SGD>>(
      persistent_grid(E * (N / BM) * ((K + BN - 1) / BN), sm_count), kGemmThreads, Tile<BN>::kSmemBytes + kGroupTableBytes,
      stream, what, make_tmap_mn(dy, R, N, N), make_tmap_mn(x, R, K, K), g, WgradComm{});
}
}  // namespace

void launch_wgrad_bf16_grouped(const void* dy, const void* x, void* gout, const int* counts, int64_t E, int64_t R,
                               int64_t N, int64_t K, int sm_count, cudaStream_t stream, const float* gscale, float axpy) {
  if (axpy != 0.0f)
    launch_grouped<false, true>("wgrad_sgd_grouped", dy, x, gout, counts, E, R, N, K, sm_count, stream, gscale, axpy);
  else
    launch_grouped<false, false>("wgrad_bf16_grouped", dy, x, gout, counts, E, R, N, K, sm_count, stream, gscale, 0.0f);
}

void launch_wgrad_accumulate_grouped(const void* dy, const void* x, float* acc, const int* counts, int64_t E, int64_t R,
                                     int64_t N, int64_t K, int sm_count, cudaStream_t stream, const float* gscale) {
  launch_grouped<true, false>("wgrad_accumulate_grouped", dy, x, acc, counts, E, R, N, K, sm_count, stream, gscale, 0.0f);
}

int64_t fused_wgrad_tiles(int64_t N, int64_t K) { return (N / BM) * (K / tile_n<true>()); }
int fused_wgrad_signals_per_unit() { return kSignalsPerUnit; }
int fused_wgrad_max_unicast_ranks() { return kMaxUnicastRanks; }

void launch_fused_wgrad_update(const DeviceComm& dc, const void* dy, const void* x, int64_t Mb, int64_t N, int64_t K,
                               int64_t ldy, int64_t ldx, int64_t w_off, int64_t stage_off, int64_t stage_stride,
                               int64_t cnt_off, int64_t done_off, int ksplit, uint32_t tile_target,
                               uint32_t done_target, float scale, int64_t wavg_off, cudaStream_t stream,
                               int64_t epoch_off, const float* gscale, bool use_multicast, int64_t src_stride) {
  M4T_CHECK(use_multicast ? dc.mc_heap != nullptr : dc.sync.size <= kMaxUnicastRanks,
            "the fused wgrad->Allreduce->SGD kernel needs the NVLS multicast mapping beyond " << kMaxUnicastRanks << " ranks");
  M4T_CHECK(ksplit == 1 || ksplit == 2, "ksplit must be 1 or 2");
  M4T_CHECK((Mb / BK) % ksplit == 0, "batch / 64 must be divisible by ksplit");
  char* stage = dc.heap[dc.sync.rank] + stage_off;
  M4T_CHECK(wgrad_bf16_supported(Mb, N, K, dy, x, stage, ldy, ldx, K), "unsupported wgrad shape/alignment for the fused path");
  M4T_CHECK(use_multicast || stage_stride == N * K * 2, "peer-store mode expects densely packed partial buffers");
  const CUtensorMap ta = make_tmap_mn(dy, Mb, N, ldy);
  const CUtensorMap tb = make_tmap_mn(x, Mb, K, ldx);
  const WgradArgs g = wgrad_args(nullptr, Mb, N, K, K, ksplit, gscale, 0.0f);
  WgradComm wc{};
  wc.sync = dc.sync;
  for (int p = 0; p < dc.sync.size; ++p) wc.heap[p] = dc.heap[p];
  wc.mc_heap = dc.mc_heap;
  wc.stage_off = stage_off;
  wc.stage_stride = stage_stride;
  wc.src_stride = src_stride;
  wc.w_off = w_off;
  wc.cnt_off = cnt_off;
  wc.done_off = done_off;
  wc.tile_target = tile_target;
  wc.done_target = done_target;
  wc.epoch_off = epoch_off;
  wc.scale = scale;
  wc.prefetch = wavg_off >= 0 ? 1 : 0;
  wc.wavg_off = wavg_off >= 0 ? wavg_off : 0;
  wc.avg_scale = 1.0f / static_cast<float>(dc.sync.size);
  wc.unicast = use_multicast ? 0 : 1;
  wc.debug = g_wgrad_debug.load(std::memory_order_relaxed);
  const int grid = fused_gemm_grid(dc);  // identical on every rank
  launch_kernel<wgrad_bf16_wgmma_kernel<true>>(
      grid, kGemmThreads + kCommWarps * 32, Tile<tile_n<true>()>::kSmemBytes, stream,
      wc.prefetch ? "fused_wgrad_reduce_scatter_sgd_prefetch" : "fused_wgrad_reduce_scatter_sgd", ta, tb, g, wc);
}

}  // namespace m4t
