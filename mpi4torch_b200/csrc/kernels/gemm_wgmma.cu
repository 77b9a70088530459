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

#include <algorithm>
#include <mutex>

#include "kernels.h"
#include "fused_comm.cuh"
#include "tma_host.h"
#include "wgmma_pipeline.cuh"

namespace m4t {

namespace {

using namespace wg;

constexpr int kPanel = 256;  // weight rows per all-reduce panel of the fused kernel (one counter each)
constexpr int kCommWarps = 4;

struct GemmArgs {
  void* C;
  int M, N, K;
  int ldc;
  // fused MSE epilogue (EPI == 1): C receives dL/dy = grad_scale * (y - T),
  // loss_acc accumulates loss_scale * sum((y - T)^2); y itself is never stored
  const void* T;
  int ldt;
  float* loss_acc;
  float loss_scale, grad_scale;
  // fused mode ----------------------------------------------------------------
  const uint32_t* panel_flags;  // [N / kPanel] counters in local HBM (written through multicast)
  uint32_t panel_target;        // a panel is ready when its counter >= target (wrap-safe)
};

// the fused kernel's communication warps need registers: half-width tiles there
template <bool FUSED> constexpr int tile_n() { return FUSED ? 128 : 256; }

// Epilogues of the two-layer MLP (EPI 2..4; unused by EPI 0/1):
//   EPI 2  TN  z = acc + bias -> C,  h = gelu_tanh(z) -> h_out
//   EPI 3  TN  d = acc + bias - T:  C = grad_scale * d, loss as EPI 1, column-sum partials of C
//   EPI 4  NN  C = gscale * acc * gelu_tanh'(z), z read from T (bf16), column-sum partials of C
// Column sums are deterministic: a warp adds its 16 rows in registers (h pair, then lane bits 2-4) and
// lanes 0-3 store one fp32 row of colsum[ceil(M/16), N]; column_sum_kernel adds those rows in a fixed order.
struct MlpEpiArgs {
  const float* bias;    // [N] fp32
  void* h_out;          // EPI 2: bf16, same layout as C
  float* colsum;        // EPI 3, 4: [ceil(M/16), N] fp32, row-major
  const float* gscale;  // EPI 4: optional device scalar
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

// Epilogue of one consumer warpgroup's 64 x BN accumulators for EPI 2..4.  Column pairs are handled in
// groups of kGroup, small enough that the bias / target / z values and the column sums fit next to acc.
template <int EPI, int BN>
__device__ __forceinline__ void mlp_epilogue(const float (&acc)[BN / 2], const GemmArgs& g, const MlpEpiArgs& e,
                                             int m_blk, int n_blk, int wgi, float& loss_part) {
  constexpr int kGroup = 4;
  constexpr bool kBias = EPI != 4, kReadT = EPI != 2, kColsum = EPI != 2;
  const int lane = threadIdx.x & 31;
  const int row0 = m_blk * BM + wgi * 64 + frag_row(0);
  const bool row_ok[2] = {row0 < g.M, row0 + 8 < g.M};
  const float gs = (EPI == 4 && e.gscale != nullptr) ? *e.gscale : 1.f;
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
      if (kBias) bv[j] = col_ok ? *reinterpret_cast<const float2*>(e.bias + col) : make_float2(0.f, 0.f);
      if (kReadT) {
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
        if (kBias) {
          v0 += bv[j].x;
          v1 += bv[j].y;
        }
        if (!row_ok[h]) continue;
        const int64_t off = static_cast<int64_t>(row0 + 8 * h) * g.ldc + col;
        const float t0 = bf16_bits_to_float(static_cast<uint16_t>(tv[h][j] & 0xffffu));
        const float t1 = bf16_bits_to_float(static_cast<uint16_t>(tv[h][j] >> 16));
        if (EPI == 2) {
          *reinterpret_cast<uint32_t*>(static_cast<uint16_t*>(e.h_out) + off) = pack_bf16x2(gelu_tanh(v0), gelu_tanh(v1));
        } else if (EPI == 3) {
          const float d0 = v0 - t0, d1 = v1 - t1;
          loss_part = fmaf(d0, d0, loss_part);
          loss_part = fmaf(d1, d1, loss_part);
          v0 = d0 * g.grad_scale;
          v1 = d1 * g.grad_scale;
        } else {
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

template <bool FUSED, int EPI, bool B_MN>
__global__ void __launch_bounds__(kGemmThreads + (FUSED ? kCommWarps * 32 : 0), 1)
gemm_bf16_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                       const GemmArgs g, const CommArgs cm, const MlpEpiArgs e) {
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
  __syncthreads();

  // The MLP epilogues hold bias, target / z values and column sums next to the accumulators: the
  // producer warpgroup hands registers to the consumers (40 + 2 x 232 per thread fits the register file).
  constexpr bool kRealloc = EPI >= 2;
  if (warp < 4) {
    // =========================== TMA producer ===========================
    if constexpr (kRealloc) tc::setmaxnreg_dec<40>();
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
        for (int kb = 0; kb < k_blocks; ++kb)
          load_stage<false, B_MN, BN>(smem, pipe, stage, phase, &tmap_a, &tmap_b, m_blk * BM, n_blk * BN, kb * BK);
      }
    }
  } else if (warp < kGemmThreads / 32) {
    // ====================== consumers: wgmma + epilogue ======================
    if constexpr (kRealloc) tc::setmaxnreg_inc<232>();
    const int wgi = warp / 4 - 1;
    int stage = 0;
    uint32_t phase = 0;
    float acc[BN / 2];
    for (int t = first_tile; t < num_tiles; t += tile_stride) {
      const int n_blk = t / m_tiles;
      const int m_blk = t - n_blk * m_tiles;
      mma_tile<false, B_MN, BN>(acc, smem, pipe, stage, phase, k_blocks, wgi);
      float loss_part = 0.f;
      if constexpr (EPI >= 2) {
        mlp_epilogue<EPI, BN>(acc, g, e, m_blk, n_blk, wgi, loss_part);
      } else {
  #pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int row = m_blk * BM + wgi * 64 + frag_row(h);
          if (row >= g.M) continue;
          uint16_t* crow = static_cast<uint16_t*>(g.C) + static_cast<int64_t>(row) * g.ldc;
          const uint16_t* trow = EPI == 1 ? static_cast<const uint16_t*>(g.T) + static_cast<int64_t>(row) * g.ldt : nullptr;
          // N is a multiple of 8, so a column pair is either wholly inside or wholly outside
  #pragma unroll
          for (int j0 = 0; j0 < BN / 8; j0 += 8) {
            uint32_t tv[8];  // the targets of eight column pairs are requested before the first is used
            if (EPI == 1) {
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
              if (EPI == 1) {
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
      }
      if (EPI == 1 || EPI == 3) {
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

template <bool FUSED> constexpr int smem_bytes() { return Tile<tile_n<FUSED>()>::kSmemBytes; }

template <bool FUSED, int EPI, bool B_MN> void configure_once() {
  static std::once_flag once;
  std::call_once(once, [] {
    cudaError_t e = cudaFuncSetAttribute(gemm_bf16_wgmma_kernel<FUSED, EPI, B_MN>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes<FUSED>());
    M4T_CHECK(e == cudaSuccess, "cudaFuncSetAttribute(smem) failed: " << cudaGetErrorString(e));
  });
}

template <bool FUSED, int EPI, bool B_MN>
void launch(int grid, const CUtensorMap& ta, const CUtensorMap& tb, const GemmArgs& g, const CommArgs& cm,
            cudaStream_t stream, const char* what, const MlpEpiArgs& e = MlpEpiArgs{}) {
  configure_once<FUSED, EPI, B_MN>();
  gemm_bf16_wgmma_kernel<FUSED, EPI, B_MN>
      <<<grid, kGemmThreads + (FUSED ? kCommWarps * 32 : 0), smem_bytes<FUSED>(), stream>>>(ta, tb, g, cm, e);
  cudaError_t err = cudaGetLastError();
  M4T_CHECK(err == cudaSuccess, what << " launch failed: " << cudaGetErrorString(err));
  note_kernel_launch(what);
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
__global__ void __launch_bounds__(256) column_sum_kernel(const float* __restrict__ partial, int rows, int N,
                                                         float* __restrict__ out, const float* gscale) {
  __shared__ float part[8][33];
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

GemmArgs plain_args(void* C, int64_t M, int64_t N, int64_t K, int64_t ldc) {
  GemmArgs g{};
  g.C = C;
  g.M = static_cast<int>(M);
  g.N = static_cast<int>(N);
  g.K = static_cast<int>(K);
  g.ldc = static_cast<int>(ldc);
  return g;
}

int plain_grid(int64_t M, int64_t N, int sm_count) {
  constexpr int BN = tile_n<false>();
  const int tiles = static_cast<int>(((M + BM - 1) / BM) * ((N + BN - 1) / BN));
  return std::max(1, std::min(tiles, sm_count));
}

}  // namespace

bool gemm_bf16_tn_supported(int64_t M, int64_t N, int64_t K, const void* A, const void* B, const void* C, int64_t lda,
                            int64_t ldb, int64_t ldc) {
  auto al16 = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; };
  return M > 0 && N > 0 && K > 0 && (K % 8) == 0 && (N % 8) == 0 && (lda % 8) == 0 && (ldb % 8) == 0 && (ldc % 8) == 0 &&
         lda >= K && ldb >= K && ldc >= N && al16(A) && al16(B) && al16(C) && M < (1ll << 31) && N < (1ll << 31) &&
         K < (1ll << 31);
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
  constexpr int BN = tile_n<false>();
  const CUtensorMap ta = make_tmap(A, M, K, lda, BM);
  const CUtensorMap tb = make_tmap(B, N, K, ldb, BN);
  GemmArgs g{};
  g.C = C;
  g.M = static_cast<int>(M);
  g.N = static_cast<int>(N);
  g.K = static_cast<int>(K);
  g.ldc = static_cast<int>(ldc);
  const int tiles = static_cast<int>(((M + BM - 1) / BM) * ((N + BN - 1) / BN));
  const int grid = std::max(1, std::min(tiles, sm_count));
  if (mse) {
    set_mse(g, mse);
    launch<false, 1, false>(grid, ta, tb, g, CommArgs{}, stream, "gemm_mse_epilogue");
  } else {
    launch<false, 0, false>(grid, ta, tb, g, CommArgs{}, stream, "gemm_bf16_tn");
  }
}

bool gemm_bf16_nn_supported(int64_t M, int64_t N, int64_t K, const void* A, const void* B, const void* C, int64_t lda,
                            int64_t ldb, int64_t ldc) {
  auto al = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; };
  return M > 0 && N > 0 && K > 0 && N % 8 == 0 && K % 8 == 0 && al(A) && al(B) && al(C) && lda % 8 == 0 && ldb % 8 == 0 &&
         ldc % 8 == 0 && lda >= K && ldb >= N && ldc >= N && M < (1ll << 31) && N < (1ll << 31) && K < (1ll << 31);
}

// C[M,N] = A[M,K] * B[K,N], both row-major (the dgrad shape: gy @ W).
void launch_gemm_bf16_nn(const void* A, const void* B, void* C, int64_t M, int64_t N, int64_t K, int64_t lda,
                         int64_t ldb, int64_t ldc, int sm_count, cudaStream_t stream) {
  M4T_CHECK(gemm_bf16_nn_supported(M, N, K, A, B, C, lda, ldb, ldc), "unsupported GEMM shape/alignment for the wgmma NN path");
  constexpr int BN = tile_n<false>();
  const CUtensorMap ta = make_tmap(A, M, K, lda, BM);
  const CUtensorMap tb = make_tmap_bf16_sw128(B, K, N, ldb, 64, BK);  // boxes of {64 n, BK k-rows}
  GemmArgs g{};
  g.C = C;
  g.M = static_cast<int>(M);
  g.N = static_cast<int>(N);
  g.K = static_cast<int>(K);
  g.ldc = static_cast<int>(ldc);
  const int tiles = static_cast<int>(((M + BM - 1) / BM) * ((N + BN - 1) / BN));
  const int grid = std::max(1, std::min(tiles, sm_count));
  launch<false, 0, true>(grid, ta, tb, g, CommArgs{}, stream, "gemm_nn");
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
  GemmArgs g{};
  g.C = y;
  g.M = static_cast<int>(M);
  g.N = static_cast<int>(N);
  g.K = static_cast<int>(K);
  g.ldc = static_cast<int>(ldy);
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
    launch<true, 1, false>(grid, ta, tb, g, cm, stream, "fused_allreduce_gemm_mse");
  } else {
    launch<true, 0, false>(grid, ta, tb, g, cm, stream, "fused_allreduce_gemm");
  }
}

int64_t colsum_rows(int64_t M) { return (M + 15) / 16; }

void launch_gemm_bias_gelu(const void* A, const void* B, const float* bias, void* z, void* h, int64_t M, int64_t N,
                           int64_t K, int64_t lda, int64_t ldb, int64_t ldc, int sm_count, cudaStream_t stream) {
  M4T_CHECK(gemm_bf16_tn_supported(M, N, K, A, B, z, lda, ldb, ldc) && (reinterpret_cast<uintptr_t>(h) & 15u) == 0,
            "unsupported GEMM shape/alignment for the wgmma bias+GELU path");
  M4T_CHECK(epilogue_bias_ok(bias), "the bias needs an 8-byte-aligned base");
  MlpEpiArgs e{};
  e.bias = bias;
  e.h_out = h;
  launch<false, 2, false>(plain_grid(M, N, sm_count), make_tmap(A, M, K, lda, BM), make_tmap(B, N, K, ldb, tile_n<false>()),
                          plain_args(z, M, N, K, ldc), CommArgs{}, stream, "gemm_bias_gelu", e);
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
  launch<false, 3, false>(plain_grid(M, N, sm_count), make_tmap(A, M, K, lda, BM), make_tmap(B, N, K, ldb, tile_n<false>()),
                          g, CommArgs{}, stream, "gemm_bias_mse_colsum", e);
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
  launch<false, 4, true>(plain_grid(M, N, sm_count), make_tmap(A, M, K, lda, BM), make_tmap_bf16_sw128(B, K, N, ldb, 64, BK),
                         g, CommArgs{}, stream, "gemm_nn_gelu_bwd_colsum", e);
}

void launch_column_sum(const float* partial, int64_t rows, int64_t N, float* out, const float* gscale, cudaStream_t stream) {
  M4T_CHECK(rows > 0 && N > 0 && N < (1ll << 31) && rows < (1ll << 31), "column_sum: empty or oversized workspace");
  column_sum_kernel<<<static_cast<unsigned>((N + 31) / 32), 256, 0, stream>>>(partial, static_cast<int>(rows),
                                                                              static_cast<int>(N), out, gscale);
  cudaError_t err = cudaGetLastError();
  M4T_CHECK(err == cudaSuccess, "column_sum launch failed: " << cudaGetErrorString(err));
  note_kernel_launch("column_sum");
}

int fused_gemm_grid(const DeviceComm& dc) { return std::min(dc.sm_count, kMaxChannels) & ~1; }

}  // namespace m4t
