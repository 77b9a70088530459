// FP8 training kernels of the data-parallel linear layer (DESIGN §4.4):
//
//   quantize_fp8_amax   amax = max |v| over a bf16 matrix, as an atomicMax on the bit pattern of |v| (exact, order-
//                       independent; NaN and Inf sort above every finite value)
//   quantize_fp8_cast   q = fp8(v * s) row-major and/or transposed (through an smem tile), s = the power of two of
//                       the amax (computed by every thread from the device amax; the host never reads it)
//   gemm_fp8_*          C = A[M,K] * B[N,K]^T with both operands K-major fp8 (A E4M3 or E5M2, B E4M3), on the shared
//                       wgmma ring (wgmma_pipeline.cuh, 128 x 128 tiles, split accumulation), dequantized in the
//                       epilogue by acc * (1/s_a) * (1/s_b):
//                         plain  C = bf16(g * acc / (s_a s_b))
//                         MSE    y = acc / (s_x s_w), dy = bf16(grad_scale (y - t)), loss as the bf16 MSE epilogue,
//                                amax(|dy|) of the stored bf16 values
//                         SGD    W = bf16(W + alpha g acc / (s_a s_b)), in place
#include <cuda.h>
#include <cuda_fp8.h>

#include "kernels.h"
#include "tma_host.h"
#include "wgmma_pipeline.cuh"

namespace m4t {

namespace {

using namespace wg;

constexpr int BN8 = 128;  // tile width: the 64 + 64 registers of the split accumulation fit beside it
constexpr int BK8 = 128;  // fp8 values per 128-byte stage row

enum Fp8Epi : int { kPlain = 0, kMse = 1, kSgd = 2 };

struct Fp8Args {
  void* C;  // bf16 [M, N]: the output (plain, MSE: dy) or the weight updated in place (SGD)
  int M, N, K;
  int ldc;
  const float* a_scale_inv;  // device scalars 1/s_a, 1/s_b
  const float* b_scale_inv;
  const float* gscale;       // optional device scalar g (plain, SGD)
  float alpha;               // SGD: W += alpha * g * acc / (s_a s_b)
  // MSE
  const void* T;
  int ldt;
  float* loss_acc;
  float loss_scale, grad_scale;
  unsigned int* dy_amax;     // bits of max |dy| (fp32), atomicMax
};

// |bf16| as the bit pattern of the fp32 of the same value: non-negative floats order as their bits.
__device__ __forceinline__ unsigned int abs_bits(uint16_t b) { return static_cast<unsigned int>(b & 0x7fffu) << 16; }

template <int EPI, bool A_E5M2>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_fp8_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b, const Fp8Args g) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = aligned_smem(smem_raw);
  Pipe* pipe = pipe_of<BN8>(smem);
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int m_tiles = (g.M + BM - 1) / BM;
  const int n_tiles = (g.N + BN8 - 1) / BN8;
  const int num_tiles = m_tiles * n_tiles;
  const int k_blocks = (g.K + BK8 - 1) / BK8;

  if (warp == 0 && lane == 0) {
    tc::prefetch_tmap(&tmap_a);
    tc::prefetch_tmap(&tmap_b);
    init_pipe<BN8>(pipe);
  }
  __syncthreads();

  if (warp < 4) {
    if (warp == 0 && lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
        const int n_blk = t / m_tiles;
        const int m_blk = t - n_blk * m_tiles;
        for (int kb = 0; kb < k_blocks; ++kb)
          load_stage<false, false, BN8>(smem, pipe, stage, phase, &tmap_a, &tmap_b, m_blk * BM, n_blk * BN8, kb * BK8);
      }
    }
  } else {
    const int wgi = warp / 4 - 1;
    int stage = 0;
    uint32_t phase = 0;
    float acc[64];
    // acc * ia * ib: both factors are powers of two, so the dequantization rounds nothing (a NaN scale poisons all)
    const float ia = *g.a_scale_inv, ib = *g.b_scale_inv;
    const float gs = EPI == kMse ? 1.f : (g.gscale ? *g.gscale : 1.f) * (EPI == kSgd ? g.alpha : 1.f);
    unsigned int amax = 0u;
    for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
      const int n_blk = t / m_tiles;
      const int m_blk = t - n_blk * m_tiles;
      mma_tile_fp8<A_E5M2>(acc, smem, pipe, stage, phase, k_blocks, wgi);
      float loss_part = 0.f;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = m_blk * BM + wgi * 64 + frag_row(h);
        if (row >= g.M) continue;
        uint16_t* crow = static_cast<uint16_t*>(g.C) + static_cast<int64_t>(row) * g.ldc;
        const uint16_t* trow = EPI == kMse ? static_cast<const uint16_t*>(g.T) + static_cast<int64_t>(row) * g.ldt : nullptr;
#pragma unroll
        for (int j0 = 0; j0 < BN8 / 8; j0 += 8) {
          uint32_t prev[8];  // the targets / weights of eight column pairs are requested before the first is used
          if (EPI != kPlain) {
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              const int col = n_blk * BN8 + frag_col(j0 + j);
              const uint16_t* src = EPI == kMse ? trow + col : crow + col;
              prev[j] = col < g.N ? (EPI == kMse ? __ldcs(reinterpret_cast<const unsigned int*>(src))
                                                 : *reinterpret_cast<const uint32_t*>(src))
                                  : 0u;
            }
          }
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const int col = n_blk * BN8 + frag_col(j0 + j);
            if (col >= g.N) continue;  // N is a multiple of 8: a column pair is wholly in or out
            float v0 = acc[4 * (j0 + j) + 2 * h] * ia * ib, v1 = acc[4 * (j0 + j) + 2 * h + 1] * ia * ib;
            const float p0 = bf16_bits_to_float(static_cast<uint16_t>(prev[j] & 0xffffu));
            const float p1 = bf16_bits_to_float(static_cast<uint16_t>(prev[j] >> 16));
            if (EPI == kMse) {
              const float d0 = v0 - p0, d1 = v1 - p1;
              loss_part = fmaf(d0, d0, loss_part);
              loss_part = fmaf(d1, d1, loss_part);
              v0 = d0 * g.grad_scale;
              v1 = d1 * g.grad_scale;
            } else {
              // rounded on its own: the SGD add below must not contract with it into an fma
              v0 = __fmul_rn(v0, gs);
              v1 = __fmul_rn(v1, gs);
              if (EPI == kSgd) {
                v0 += p0;
                v1 += p1;
              }
            }
            const uint32_t o = pack_bf16x2(v0, v1);
            *reinterpret_cast<uint32_t*>(crow + col) = o;
            if (EPI == kMse) amax = max(amax, max(abs_bits(o & 0xffffu), abs_bits(o >> 16)));
          }
        }
      }
      if (EPI == kMse) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) loss_part += __shfl_xor_sync(0xffffffffu, loss_part, o);
        if (lane == 0) atomicAdd(g.loss_acc, loss_part * g.loss_scale);
      }
    }
    if (EPI == kMse) {
      amax = __reduce_max_sync(0xffffffffu, amax);
      if (lane == 0) atomicMax(g.dy_amax, amax);
    }
  }
  __syncthreads();
}

// ---- quantization ---------------------------------------------------------------------------------------------
constexpr int kQThreads = 256;
constexpr int kQTile = 64;  // cast: 64 x 64 elements per block

// s = the largest power of two with amax * s <= F (F = 0.875 * 2^fe: 448 = 0.875 * 2^9, 57344 = 0.875 * 2^16), its
// exponent clamped to [-126, 126] so that s and 1/s are normal; amax = 0 gives s = 1; a non-finite amax gives s = 1
// and 1/s = NaN, which poisons every product that reads the operand.
__device__ __forceinline__ void fp8_scale(float amax, int fe, float& s, float& inv) {
  if (!(amax <= 3.402823466e38f)) {
    s = 1.f;
    inv = __int_as_float(0x7fc00000);
    return;
  }
  int e = 0;
  if (amax > 0.f) {
    int ex;
    const float m = frexpf(amax, &ex);
    e = fe - ex - (m > 0.875f ? 1 : 0);
    e = max(-126, min(126, e));
  }
  s = __int_as_float((e + 127) << 23);
  inv = __int_as_float((127 - e) << 23);
}

// amax of a bf16 [rows, cols] matrix (leading dimension ld) into *amax_bits (zeroed by the caller).
__global__ void __launch_bounds__(kQThreads) quantize_fp8_amax_kernel(const uint16_t* __restrict__ x, int64_t rows,
                                                                      int64_t cols, int64_t ld, bool vec,
                                                                      unsigned int* amax_bits) {
  unsigned int m = 0u;
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  if (vec) {  // cols % 8 == 0, ld % 8 == 0, 16-byte-aligned base: one 16-byte load per 8 values
    const int64_t groups = cols / 8;
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < rows * groups; i += stride) {
      const int64_t r = i / groups, c = (i - r * groups) * 8;
      const uint4 v = __ldcs(reinterpret_cast<const uint4*>(x + r * ld + c));
      const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int k = 0; k < 4; ++k) m = max(m, max(abs_bits(w[k] & 0xffffu), abs_bits(w[k] >> 16)));
    }
  } else {
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < rows * cols; i += stride) {
      const int64_t r = i / cols, c = i - r * cols;
      m = max(m, abs_bits(x[r * ld + c]));
    }
  }
  __shared__ unsigned int part[kQThreads / 32];
  m = __reduce_max_sync(0xffffffffu, m);
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
#pragma unroll
    for (int k = 1; k < kQThreads / 32; ++k) m = max(m, part[k]);
    atomicMax(amax_bits, m);
  }
}

template <bool E5M2>
__device__ __forceinline__ uint16_t to_fp8x2(float lo, float hi) {
  return __nv_cvt_float2_to_fp8x2(make_float2(lo, hi), __NV_SATFINITE, E5M2 ? __NV_E5M2 : __NV_E4M3);
}

// Block (bx, by) casts x[64 by .. +64, 64 bx .. +64]: q row-major [rows, cols] and/or qt = q^T [cols, rows] (both
// contiguous).  Thread t handles columns 8 (t % 8) .. +8 of rows t / 8 and t / 8 + 32; the transposed copy goes
// through a byte tile in smem and leaves as 16-byte rows of qt.  Block (0, 0) also stores 1/s.
template <bool E5M2>
__global__ void __launch_bounds__(kQThreads) quantize_fp8_cast_kernel(const uint16_t* __restrict__ x, int64_t rows,
                                                                      int64_t cols, int64_t ld, bool vec,
                                                                      const unsigned int* amax_bits,
                                                                      uint8_t* __restrict__ q, uint8_t* __restrict__ qt,
                                                                      float* scale_inv) {
  __shared__ __align__(16) uint8_t tile[kQTile][kQTile + 16];
  float s, inv;
  fp8_scale(__uint_as_float(*amax_bits), E5M2 ? 16 : 9, s, inv);
  if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) *scale_inv = inv;
  const int64_t r0 = static_cast<int64_t>(blockIdx.y) * kQTile, c0 = static_cast<int64_t>(blockIdx.x) * kQTile;
  const int cg = (threadIdx.x % 8) * 8;
#pragma unroll
  for (int pass = 0; pass < 2; ++pass) {
    const int rr = threadIdx.x / 8 + 32 * pass;
    const int64_t r = r0 + rr, c = c0 + cg;
    float v[8];
    if (vec && r < rows && c + 8 <= cols) {
      const uint4 raw = __ldcs(reinterpret_cast<const uint4*>(x + r * ld + c));
      const uint32_t w[4] = {raw.x, raw.y, raw.z, raw.w};
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        v[2 * k] = bf16_bits_to_float(static_cast<uint16_t>(w[k] & 0xffffu));
        v[2 * k + 1] = bf16_bits_to_float(static_cast<uint16_t>(w[k] >> 16));
      }
    } else {
#pragma unroll
      for (int k = 0; k < 8; ++k) v[k] = (r < rows && c + k < cols) ? bf16_bits_to_float(x[r * ld + c + k]) : 0.f;
    }
    uint16_t p[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) p[k] = to_fp8x2<E5M2>(v[2 * k] * s, v[2 * k + 1] * s);
    if (q != nullptr && r < rows) {
      if (vec && c + 8 <= cols) {
        *reinterpret_cast<uint2*>(q + r * cols + c) =
            make_uint2(p[0] | (static_cast<uint32_t>(p[1]) << 16), p[2] | (static_cast<uint32_t>(p[3]) << 16));
      } else {
#pragma unroll
        for (int k = 0; k < 8; ++k)
          if (c + k < cols) q[r * cols + c + k] = static_cast<uint8_t>(p[k / 2] >> (8 * (k % 2)));
      }
    }
    if (qt != nullptr) {
#pragma unroll
      for (int k = 0; k < 8; ++k) tile[cg + k][rr] = static_cast<uint8_t>(p[k / 2] >> (8 * (k % 2)));
    }
  }
  if (qt == nullptr) return;
  __syncthreads();
  // qt rows c0 .. c0 + 63, bytes r0 .. r0 + 63 of each: four 16-byte pieces per row
  const int cr = threadIdx.x / 4, piece = (threadIdx.x % 4) * 16;
  const int64_t orow = c0 + cr, ocol = r0 + piece;
  if (orow >= cols) return;
  if (rows % 16 == 0 && ocol + 16 <= rows) {
    *reinterpret_cast<uint4*>(qt + orow * rows + ocol) = *reinterpret_cast<const uint4*>(&tile[cr][piece]);
  } else {
    for (int k = 0; k < 16 && ocol + k < rows; ++k) qt[orow * rows + ocol + k] = tile[cr][piece + k];
  }
}

// ---- host side ------------------------------------------------------------------------------------------------
template <int EPI, bool A_E5M2>
void launch_fp8(const Fp8Args& g, const void* A, const void* B, int64_t lda, int64_t ldb, int sm_count,
                cudaStream_t stream, const char* what) {
  const int64_t tiles = ((g.M + BM - 1) / BM) * ((g.N + BN8 - 1) / BN8);
  launch_kernel<gemm_fp8_kernel<EPI, A_E5M2>>(persistent_grid(tiles, sm_count), kGemmThreads, Tile<BN8>::kSmemBytes,
                                              stream, what, make_tmap_u8_sw128(A, g.M, g.K, lda, BM),
                                              make_tmap_u8_sw128(B, g.N, g.K, ldb, BN8), g);
}

template <int EPI>
void dispatch_fp8(const Fp8Args& g, bool a_e5m2, const void* A, const void* B, int64_t lda, int64_t ldb, int sm_count,
                  cudaStream_t stream, const char* what) {
  if (a_e5m2) launch_fp8<EPI, true>(g, A, B, lda, ldb, sm_count, stream, what);
  else launch_fp8<EPI, false>(g, A, B, lda, ldb, sm_count, stream, what);
}

Fp8Args fp8_args(void* C, int64_t M, int64_t N, int64_t K, int64_t ldc, const float* a_si, const float* b_si) {
  Fp8Args g{};
  g.C = C;
  g.M = static_cast<int>(M);
  g.N = static_cast<int>(N);
  g.K = static_cast<int>(K);
  g.ldc = static_cast<int>(ldc);
  g.a_scale_inv = a_si;
  g.b_scale_inv = b_si;
  return g;
}

}  // namespace

bool gemm_fp8_tn_supported(int64_t M, int64_t N, int64_t K, const void* A, const void* B, const void* C, int64_t lda,
                           int64_t ldb, int64_t ldc) {
  return M > 0 && N > 0 && K > 0 && K % 16 == 0 && N % 8 == 0 && lda % 16 == 0 && ldb % 16 == 0 && ldc % 8 == 0 &&
         lda >= K && ldb >= K && ldc >= N && aligned16(A) && aligned16(B) && aligned16(C) && M < (1ll << 31) &&
         N < (1ll << 31) && K < (1ll << 31) && ldc < (1ll << 31);
}

void launch_gemm_fp8_tn(const void* A, bool a_e5m2, const void* B, void* C, int64_t M, int64_t N, int64_t K, int64_t lda,
                        int64_t ldb, int64_t ldc, const float* a_scale_inv, const float* b_scale_inv, const float* gscale,
                        int sm_count, cudaStream_t stream) {
  M4T_CHECK(gemm_fp8_tn_supported(M, N, K, A, B, C, lda, ldb, ldc), "unsupported shape/alignment for gemm_fp8_tn");
  Fp8Args g = fp8_args(C, M, N, K, ldc, a_scale_inv, b_scale_inv);
  g.gscale = gscale;
  dispatch_fp8<kPlain>(g, a_e5m2, A, B, lda, ldb, sm_count, stream, "gemm_fp8_tn");
}

void launch_gemm_fp8_mse(const void* A, const void* B, void* dy, int64_t M, int64_t N, int64_t K, int64_t lda,
                         int64_t ldb, int64_t ldc, const float* a_scale_inv, const float* b_scale_inv,
                         const MseEpilogue& mse, unsigned int* dy_amax, int sm_count, cudaStream_t stream) {
  M4T_CHECK(gemm_fp8_tn_supported(M, N, K, A, B, dy, lda, ldb, ldc), "unsupported shape/alignment for gemm_fp8_mse");
  M4T_CHECK(epilogue_bf16_pairs_ok(mse.target, mse.ldt), "the MSE target needs a 4-byte-aligned base and an even row stride");
  Fp8Args g = fp8_args(dy, M, N, K, ldc, a_scale_inv, b_scale_inv);
  g.T = mse.target;
  g.ldt = static_cast<int>(mse.ldt);
  g.loss_acc = mse.loss_acc;
  g.loss_scale = mse.loss_scale;
  g.grad_scale = mse.grad_scale;
  g.dy_amax = dy_amax;
  dispatch_fp8<kMse>(g, false, A, B, lda, ldb, sm_count, stream, "gemm_fp8_mse");
}

void launch_gemm_fp8_sgd(const void* A, bool a_e5m2, const void* B, void* W, int64_t M, int64_t N, int64_t K,
                         int64_t lda, int64_t ldb, int64_t ldw, const float* a_scale_inv, const float* b_scale_inv,
                         float alpha, const float* gscale, int sm_count, cudaStream_t stream) {
  M4T_CHECK(gemm_fp8_tn_supported(M, N, K, A, B, W, lda, ldb, ldw), "unsupported shape/alignment for gemm_fp8_sgd");
  Fp8Args g = fp8_args(W, M, N, K, ldw, a_scale_inv, b_scale_inv);
  g.gscale = gscale;
  g.alpha = alpha;
  dispatch_fp8<kSgd>(g, a_e5m2, A, B, lda, ldb, sm_count, stream, "gemm_fp8_sgd");
}

bool quantize_fp8_vec_ok(const void* x, int64_t cols, int64_t ld) { return aligned16(x) && cols % 8 == 0 && ld % 8 == 0; }

void launch_quantize_fp8_amax(const void* x, int64_t rows, int64_t cols, int64_t ld, unsigned int* amax_bits,
                              int sm_count, cudaStream_t stream) {
  M4T_CHECK(rows > 0 && cols > 0 && ld >= cols, "quantize_fp8: empty matrix or bad leading dimension");
  const bool vec = quantize_fp8_vec_ok(x, cols, ld);
  const int64_t work = vec ? rows * (cols / 8) : rows * cols;
  const int blocks = static_cast<int>(std::max<int64_t>(1, std::min<int64_t>((work + kQThreads - 1) / kQThreads,
                                                                             static_cast<int64_t>(sm_count) * 8)));
  launch_kernel<quantize_fp8_amax_kernel>(blocks, kQThreads, 0, stream, "quantize_fp8_amax",
                                          static_cast<const uint16_t*>(x), rows, cols, ld, vec, amax_bits);
}

void launch_quantize_fp8_cast(const void* x, int64_t rows, int64_t cols, int64_t ld, bool e5m2,
                              const unsigned int* amax_bits, void* q, void* qt, float* scale_inv, cudaStream_t stream) {
  M4T_CHECK(rows > 0 && cols > 0 && ld >= cols, "quantize_fp8: empty matrix or bad leading dimension");
  M4T_CHECK(q == nullptr || cols % 8 != 0 || (reinterpret_cast<uintptr_t>(q) & 7u) == 0, "quantize_fp8: q misaligned");
  M4T_CHECK(qt == nullptr || aligned16(qt), "quantize_fp8: qt misaligned");
  const int64_t bx = (cols + kQTile - 1) / kQTile, by = (rows + kQTile - 1) / kQTile;
  M4T_CHECK(bx < (1ll << 31) && by < 65536, "quantize_fp8: matrix too large");
  const dim3 grid(static_cast<unsigned>(bx), static_cast<unsigned>(by));
  const bool vec = quantize_fp8_vec_ok(x, cols, ld);
  const auto* xb = static_cast<const uint16_t*>(x);
  auto* qb = static_cast<uint8_t*>(q);
  auto* qtb = static_cast<uint8_t*>(qt);
  if (e5m2)
    launch_kernel<quantize_fp8_cast_kernel<true>>(grid, kQThreads, 0, stream, "quantize_fp8_cast", xb, rows, cols, ld,
                                                  vec, amax_bits, qb, qtb, scale_inv);
  else
    launch_kernel<quantize_fp8_cast_kernel<false>>(grid, kQThreads, 0, stream, "quantize_fp8_cast", xb, rows, cols, ld,
                                                   vec, amax_bits, qb, qtb, scale_inv);
}

}  // namespace m4t
