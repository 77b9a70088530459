// Host-callable launchers of the sm_90a kernels.  Torch-free; the CUDA backend
// (runtime/cuda_backend.cpp) fills a DeviceComm once and passes it by value.
#pragma once
#include <string>
#include <utility>
#include <vector>
#include <cuda_runtime.h>

#include "../runtime/common.h"
#include "../runtime/plan.h"
#include "device_sync.cuh"

namespace m4t {

// Symmetric-heap layout (identical on every rank):
//   [0, kPadBytes)                       barrier flag pads + p2p flags
//   [p2p_off, p2p_off + p2p_bytes)       p2p FIFO slots
//   [stage_off, stage_off + 2*half)      staging halves (op parity)
constexpr int64_t kBarrierPadBytes = static_cast<int64_t>(kMaxChannels) * kMaxGpuPeers * 4;  // 32 KiB

struct DeviceComm {
  SyncCtx sync;
  char* heap[kMaxGpuPeers];  // unicast mappings of every rank's heap (heap[rank] is local)
  char* mc_heap;             // multicast mapping of the heap, or nullptr
  int64_t stage_off;         // byte offset of staging half 0
  int64_t half_bytes;        // bytes per staging half
  int sm_count;
};

// Number of kernels this library has launched in this process (bench.py's
// "gpu_launches" evidence).
unsigned long long kernel_launch_count();
void note_kernel_launch();
// Same, and additionally tallied under `name` (bench.py reports which code paths really ran).
void note_kernel_launch(const char* name);
std::vector<std::pair<std::string, unsigned long long>> kernel_launch_table();

enum class ArAlgo : int { AUTO = 0, ONESHOT = 1, TWOSHOT = 2, NVLS = 3, LOCAL = 4 };

// True if the (dtype, op) pair has an in-switch multimem.ld_reduce form we emit.
bool nvls_supported(DType dt, ReduceOp op);

// Bytes of staging (per half) an allreduce of n elements needs with `algo`.
int64_t allreduce_stage_bytes(int64_t n, DType dt, ArAlgo algo, int size);

// out = epilogue(reduce over ranks of in).  One launch.
// sym_in_off >= 0: `in` is this rank's instance of a symmetric tensor at that heap offset (the
// same on every rank); two-shot / NVLS kernels then read it in place instead of staging it.
void launch_allreduce(const DeviceComm& dc, const void* in, void* out, int64_t n, DType dt, ReduceOp op,
                      const Epilogue& epi, ArAlgo algo, int blocks, int64_t chunk_bytes, cudaStream_t stream,
                      int64_t sym_in_off = -1);

// World-size-1 / local form: out = epilogue(normalise(in)); also the copy kernel.
void launch_local_epilogue(const void* in, void* out, int64_t n, DType dt, ReduceOp op, const Epilogue& epi,
                           int sm_count, cudaStream_t stream);

// Broadcast root's private buffer in place (NVLS push when mc_heap, else peer pull).
void launch_bcast(const DeviceComm& dc, void* buf, int64_t n, DType dt, int root, int blocks,
                  cudaStream_t stream);
// Reduce to root in place, zero-fill non-roots.
void launch_reduce(const DeviceComm& dc, void* buf, int64_t n, DType dt, ReduceOp op, int root, int blocks,
                   cudaStream_t stream);

// Copies `bytes` of a private buffer into this rank's staging half (current parity).
void launch_stage_in(const DeviceComm& dc, const void* in, int64_t bytes, int sm_count, cudaStream_t stream);
// Barrier + strided box pulls from peers' staging (Gather/Allgather/Scatter/Alltoall).
void launch_slab_pull(const DeviceComm& dc, const PullPlan& plan, const void* in, void* out, DType dt,
                      int blocks, cudaStream_t stream);
// Experimental Allgather by multicast push (slab_push.cu); false = not eligible, nothing launched.
bool launch_allgather_push(const DeviceComm& dc, const PullPlan& plan, const void* in, void* out, DType dt, int blocks,
                           cudaStream_t stream);
// Barrier + reduce-scatter box (Allgather adjoint) with fused epilogue.
void launch_slab_reduce(const DeviceComm& dc, const ReducePlan& plan, const void* in, void* out, DType dt,
                        ReduceOp op, const Epilogue& epi, bool use_nvls, int blocks, cudaStream_t stream);
// Local strided box copy (world size 1).
void launch_slab_local(const PullPlan& plan, const void* in, void* out, DType dt, int sm_count,
                       cudaStream_t stream);

// ---- point-to-point FIFO (one directed pair) --------------------------------
// As seen from the launching side: `slots` is the sender's ring (local pointer
// on the sender, peer mapping on the receiver); head flags live in the
// RECEIVER's pad (sender writes them remotely), tail flags in the SENDER's pad.
struct P2pChannel {
  char* slots;
  uint32_t* head_flags;  // [nslots], value = chunk index + 1 once the slot holds that chunk
  uint32_t* tail_flags;  // [nslots], value = chunk index + 1 once that chunk has been consumed
  int64_t slot_bytes;
  int nslots;
};
// Forces both p2p kernels to be loaded (lazy module loading hazard, see p2p.cu).
void preload_p2p_kernels();
// Chunks a message of `bytes` occupies in the ring (>= 1: empty messages carry a flag).
int64_t p2p_num_chunks(int64_t bytes, int64_t slot_bytes);
// Sender: copies `bytes` from `src` into the ring, chunk by chunk, publishing head flags.
void launch_p2p_send(const SyncCtx& sync, const P2pChannel& ch, const void* src, int64_t bytes,
                     unsigned long long first_chunk, int blocks, cudaStream_t stream);
// Receiver: pulls chunks out of the sender's ring into `dst`, acknowledging tail flags.
void launch_p2p_recv(const SyncCtx& sync, const P2pChannel& ch, void* dst, int64_t bytes,
                     unsigned long long first_chunk, int blocks, cudaStream_t stream);
// Copy-engine variants for large messages: same ring / flags / chunk numbering, payload moved by
// cudaMemcpyAsync (no SM copies a byte), flags handled by one-warp kernels between the copies.
void launch_p2p_send_ce(const SyncCtx& sync, const P2pChannel& ch, const void* src, int64_t bytes,
                        unsigned long long first_chunk, cudaStream_t stream);
void launch_p2p_recv_ce(const SyncCtx& sync, const P2pChannel& ch, void* dst, int64_t bytes,
                        unsigned long long first_chunk, cudaStream_t stream);

// ---- wgmma GEMM + fused Allreduce->GEMM (gemm_wgmma.cu) ------------------------
bool gemm_bf16_tn_supported(int64_t M, int64_t N, int64_t K, const void* A, const void* B, const void* C, int64_t lda,
                            int64_t ldb, int64_t ldc);
// Optional fused MSE epilogue: instead of y the kernel stores dL/dy =
// grad_scale * (y - target) and adds loss_scale * sum((y - target)^2) to *loss_acc.
struct MseEpilogue {
  const void* target;
  int64_t ldt;
  float* loss_acc;
  float loss_scale, grad_scale;
};
// Operands the GEMM epilogues read with vector loads.  The MSE target and the GELU input z are read as bf16 pairs
// (4 bytes at an even column): they need a 4-byte-aligned base and an even leading dimension.  The bias is read as
// fp32 pairs: it needs an 8-byte-aligned base.  The launchers check both before launching.
bool epilogue_bf16_pairs_ok(const void* p, int64_t ld);
bool epilogue_bias_ok(const float* bias);
// C[M,N] = A[M,K] * B[N,K]^T, bf16 in / fp32 accumulate / bf16 out.
void launch_gemm_bf16_tn(const void* A, const void* B, void* C, int64_t M, int64_t N, int64_t K, int64_t lda,
                         int64_t ldb, int64_t ldc, int sm_count, cudaStream_t stream, const MseEpilogue* mse = nullptr);
// y = x @ (scale * sum_ranks W)^T in one kernel; W staged at heap offset w_off on every rank.
void launch_fused_allreduce_gemm(const DeviceComm& dc, const void* x, void* y, int64_t M, int64_t N, int64_t K,
                                 int64_t ldx, int64_t ldy, int64_t w_off, int64_t wavg_off, int64_t flags_off,
                                 uint32_t panel_target, float scale, cudaStream_t stream, const MseEpilogue* mse = nullptr);
int fused_gemm_grid(const DeviceComm& dc);

// ---- epilogues of the two-layer MLP (gemm_wgmma.cu) -----------------------------------
// Column sums come as fp32 partials [colsum_rows(M), N] (one row per 16 output rows, deterministic);
// launch_column_sum reduces them in a fixed order.
int64_t colsum_rows(int64_t M);
// z = A[M,K] * B[N,K]^T + bias, h = gelu_tanh(z) (from the fp32 z); z and h bf16 with leading dimension ldc.
void launch_gemm_bias_gelu(const void* A, const void* B, const float* bias, void* z, void* h, int64_t M, int64_t N,
                           int64_t K, int64_t lda, int64_t ldb, int64_t ldc, int sm_count, cudaStream_t stream);
// dy = grad_scale * (A * B^T + bias - target), loss as MseEpilogue, colsum = partial column sums of dy.
void launch_gemm_bias_mse_colsum(const void* A, const void* B, const float* bias, void* dy, float* colsum, int64_t M,
                                 int64_t N, int64_t K, int64_t lda, int64_t ldb, int64_t ldc, int sm_count,
                                 cudaStream_t stream, const MseEpilogue& mse);
// dz = gscale * (A[M,K] * B[K,N]) * gelu_tanh'(z)  (B row-major, read MN-major; z bf16 [M,N]),
// colsum = partial column sums of dz.
void launch_gemm_nn_gelu_bwd_colsum(const void* A, const void* B, const void* z, void* dz, float* colsum, int64_t M,
                                    int64_t N, int64_t K, int64_t lda, int64_t ldb, int64_t ldz, int64_t ldc,
                                    int sm_count, cudaStream_t stream, const float* gscale = nullptr);
// out[n] = gscale * sum_i partial[i, n], fp32, summed in a fixed order of i.
void launch_column_sum(const float* partial, int64_t rows, int64_t N, float* out, const float* gscale,
                       cudaStream_t stream);
// Softmax cross-entropy output layer, two kernels.  gemm_bias_xent: logits = bf16(A * B^T + bias) -> logits, and per
// row and 256-column tile the pair (max, sum exp(logit - max)) of the stored logits -> ms [xent_tiles(N), M].
int64_t xent_tiles(int64_t N);
void launch_gemm_bias_xent(const void* A, const void* B, const float* bias, void* logits, float2* ms, int64_t M,
                           int64_t N, int64_t K, int64_t lda, int64_t ldb, int64_t ldc, int sm_count, cudaStream_t stream);
// xent_finish, in place over the logits: dy = grad_scale * (softmax - onehot(labels)) (bf16), colsum = partial
// column sums of dy as launch_gemm_bias_mse_colsum writes them, *loss = loss_scale * sum_rows (lse - logit[label])
// in a fixed order.  A label equal to ignore_index gives a zero row and loss 0, one outside [0, N) a NaN row and loss.
// Workspaces: row_loss [M] fp32, done: one zeroed counter.
void launch_xent_finish(void* y, int64_t M, int64_t N, int64_t ldy, const float2* ms, const int64_t* labels,
                        int64_t ignore_index, float loss_scale, float grad_scale, float* row_loss, unsigned int* done,
                        float* loss, float* colsum, cudaStream_t stream);

// ---- weight gradient (wgrad_wgmma.cu) ------------------------------------------------
// G[N,K] = dY[Mb,N]^T * X[Mb,K]: both operands MN-major, no transposed copies.
bool wgrad_bf16_supported(int64_t Mb, int64_t N, int64_t K, const void* dy, const void* x, const void* g, int64_t ldy,
                          int64_t ldx, int64_t ldg);
// C[M,N] = A[M,K] * B[K,N], both row-major bf16 (dgrad: gy @ W): the wgmma kernel with an MN-major B operand.
bool gemm_bf16_nn_supported(int64_t M, int64_t N, int64_t K, const void* A, const void* B, const void* C, int64_t lda,
                            int64_t ldb, int64_t ldc);
void launch_gemm_bf16_nn(const void* A, const void* B, void* C, int64_t M, int64_t N, int64_t K, int64_t lda,
                         int64_t ldb, int64_t ldc, int sm_count, cudaStream_t stream);
void launch_wgrad_bf16(const void* dy, const void* x, void* g, int64_t Mb, int64_t N, int64_t K, int64_t ldy,
                       int64_t ldx, int64_t ldg, int sm_count, cudaStream_t stream, const float* gscale = nullptr,
                       float axpy = 0.0f);
// gscale: optional device scalar folded into the epilogue; axpy != 0: g <- g + axpy * gscale * (dy^T x)
// (the single-rank SGD step as the GEMM's own epilogue).
// acc[N,K] (contiguous fp32) <- fmaf(gscale, dy^T x, acc) elementwise: one rounding per call.  Gradient
// accumulation over micro-batches; the operand rules are wgrad_bf16_supported's with ldg = K.
void launch_wgrad_accumulate(const void* dy, const void* x, float* acc, int64_t Mb, int64_t N, int64_t K, int64_t ldy,
                             int64_t ldx, int sm_count, cudaStream_t stream, const float* gscale = nullptr);
// wgrad GEMM -> reduce-scatter through the switch -> W += scale * sum -> multicast of the new
// weights, ONE kernel.  W (bf16 [N,K] contiguous) lives at heap offset w_off on every rank and
// must be replicated (identical on all ranks), as it is under data-parallel SGD.
void set_wgrad_debug(int mask);  // timing experiments (see WgradComm::debug)
int64_t fused_wgrad_tiles(int64_t N, int64_t K);
int fused_wgrad_signals_per_unit();   // signals on a tile counter per work unit and rank
int fused_wgrad_max_unicast_ranks();  // largest world the peer-load (no multicast) mode supports
void launch_fused_wgrad_update(const DeviceComm& dc, const void* dy, const void* x, int64_t Mb, int64_t N, int64_t K,
                               int64_t ldy, int64_t ldx, int64_t w_off, int64_t stage_off, int64_t stage_stride,
                               int64_t cnt_off, int64_t done_off, int ksplit, uint32_t tile_target,
                               uint32_t done_target, float scale, int64_t wavg_off, cudaStream_t stream,
                               int64_t epoch_off = -1, const float* gscale = nullptr, bool use_multicast = true,
                               int64_t src_stride = 0);
// src_stride (peer-store mode): the staging area holds one copy per SOURCE rank, src_stride bytes apart.
// tile_target = signals per WORK UNIT summed over ranks (the kernel multiplies by the tile's number of units).
// epoch_off >= 0: tile_target / done_target are PER-CALL increments and the call index lives in the local
// device word at that heap offset (advanced by the kernel): no host-side step state, graph-capturable.
// wavg_off >= 0: additionally leaves (1/P) * sum_ranks W_new in the bf16 [N,K] buffer at that heap
// offset on every rank (the parameter all-reduce of the NEXT forward, run under this GEMM).

// ---- batched experts (gemm_wgmma.cu, wgrad_wgmma.cu; DESIGN §4.4) -------------------------------------------------
// E experts of identical shapes in ONE launch.  Every operand is contiguous and stacked along its leading dimension:
// A [E, M, K], B [E, N, K] (TN) or [E, K, N] (NN), C [E, M, N], bias [E, N] fp32, column-sum partials
// [E, M / 16, N].  M % 128 == 0 (a tile never spans two experts), N % 128 == K % 128 == 0, 16-byte-aligned bases.
bool batched_gemm_supported(int64_t E, int64_t M, int64_t N, int64_t K, const void* A, const void* B, const void* C);
// z_e = A_e B_e^T + bias_e, h_e = gelu_tanh(z_e), as launch_gemm_bias_gelu per expert.
void launch_gemm_bias_gelu_batched(const void* A, const void* B, const float* bias, void* z, void* h, int64_t E,
                                   int64_t M, int64_t N, int64_t K, int sm_count, cudaStream_t stream);
// y_e = bf16(A_e B_e^T + bias_e).
void launch_gemm_bias_batched(const void* A, const void* B, const float* bias, void* y, int64_t E, int64_t M, int64_t N,
                              int64_t K, int sm_count, cudaStream_t stream);
// dz_e = gscale * (A_e B_e) * gelu_tanh'(z_e) and its column-sum partials, as launch_gemm_nn_gelu_bwd_colsum.
void launch_gemm_nn_gelu_bwd_colsum_batched(const void* A, const void* B, const void* z, void* dz, float* colsum,
                                            int64_t E, int64_t M, int64_t N, int64_t K, int sm_count, cudaStream_t stream,
                                            const float* gscale = nullptr);
// C_e = A_e B_e, as launch_gemm_bf16_nn.
void launch_gemm_nn_batched(const void* A, const void* B, void* C, int64_t E, int64_t M, int64_t N, int64_t K,
                            int sm_count, cudaStream_t stream);
// out[e, n] = gscale * sum_i partial[e, i, n], in column_sum's order.
void launch_column_sum_batched(const float* partial, int64_t E, int64_t rows, int64_t N, float* out, const float* gscale,
                               cudaStream_t stream);
// G_e [N, K] = gscale * dY_e^T X_e with dY [E, Mb, N], X [E, Mb, K], G [E, N, K]; the rules of wgrad_bf16_supported.
bool wgrad_bf16_batched_supported(int64_t E, int64_t Mb, int64_t N, int64_t K, const void* dy, const void* x,
                                  const void* g);
// axpy != 0: the SGD step g_e <- bf16(g_e + axpy * gscale * dY_e^T X_e) in place of G (as launch_wgrad_bf16).
void launch_wgrad_bf16_batched(const void* dy, const void* x, void* g, int64_t E, int64_t Mb, int64_t N, int64_t K,
                               int sm_count, cudaStream_t stream, const float* gscale = nullptr, float axpy = 0.0f);
// acc [E, N, K] (fp32) <- fmaf(gscale, dY_e^T X_e, acc_e), as launch_wgrad_accumulate per expert.
void launch_wgrad_accumulate_batched(const void* dy, const void* x, float* acc, int64_t E, int64_t Mb, int64_t N,
                                     int64_t K, int sm_count, cudaStream_t stream, const float* gscale = nullptr);

// ---- grouped experts (gemm_wgmma.cu, wgrad_wgmma.cu; DESIGN §4.4) -------------------------------------------------
// E experts with row counts `counts` [E] (int32, read on the device only) share one [R, .] operand in the grouped
// layout: expert e's rows start at row 128 * sum_{j<e} ceil(counts[j] / 128).  Counts are clamped to [0, R]; rows of
// a group that would lie past R do not exist.  Weights are stacked as for the batched kernels: B [E, N, K] (TN) or
// [E, K, N] (NN), bias [E, N].  Outputs [R, N] are written whole: rows past a group's count and behind the last group
// are zero.  R % 128 == N % 128 == K % 128 == 0, 1 <= E <= 1024, 16-byte-aligned operands.
bool grouped_gemm_supported(int64_t E, int64_t R, int64_t N, int64_t K, const void* A, const void* B, const void* C,
                            const void* counts);
void launch_gemm_bias_gelu_grouped(const void* A, const void* B, const float* bias, void* z, void* h, const int* counts,
                                   int64_t E, int64_t R, int64_t N, int64_t K, int sm_count, cudaStream_t stream);
void launch_gemm_bias_grouped(const void* A, const void* B, const float* bias, void* y, const int* counts, int64_t E,
                              int64_t R, int64_t N, int64_t K, int sm_count, cudaStream_t stream);
// colsum: [R / 16, N] partials; the rows of group e's ceil(count / 16) partial rows are written, the others are not.
void launch_gemm_nn_gelu_bwd_colsum_grouped(const void* A, const void* B, const void* z, void* dz, float* colsum,
                                            const int* counts, int64_t E, int64_t R, int64_t N, int64_t K, int sm_count,
                                            cudaStream_t stream);
void launch_gemm_nn_grouped(const void* A, const void* B, void* C, const int* counts, int64_t E, int64_t R, int64_t N,
                            int64_t K, int sm_count, cudaStream_t stream);
// out [E, N] fp32: per group, the sum of its column-sum partial rows ([R / 16, N] fp32), or of its valid rows
// (bf16_rows: [R, N] bf16), in column_sum's fixed order.
void launch_column_sum_grouped(const void* in, bool bf16_rows, const int* counts, int64_t E, int64_t R, int64_t N,
                               float* out, cudaStream_t stream);
// G_e [N, K] = gscale * dY_e^T X_e over group e's rows of dY [R, N] and X [R, K]; G [E, N, K], zero for an empty group.
bool wgrad_bf16_grouped_supported(int64_t E, int64_t R, int64_t N, int64_t K, const void* dy, const void* x,
                                  const void* g, const void* counts);
// axpy != 0: the SGD step g_e <- bf16(g_e + axpy * gscale * G_e); an empty group's g_e is not written.
void launch_wgrad_bf16_grouped(const void* dy, const void* x, void* g, const int* counts, int64_t E, int64_t R,
                               int64_t N, int64_t K, int sm_count, cudaStream_t stream, const float* gscale = nullptr,
                               float axpy = 0.0f);
// acc [E, N, K] (fp32) <- fmaf(gscale, G_e, acc_e); an empty group's acc_e is not written.
void launch_wgrad_accumulate_grouped(const void* dy, const void* x, float* acc, const int* counts, int64_t E, int64_t R,
                                     int64_t N, int64_t K, int sm_count, cudaStream_t stream,
                                     const float* gscale = nullptr);

// ---- FP8 training of the linear layer (gemm_fp8.cu, DESIGN §4.4) ---------------------------------------------
// Per-tensor power-of-two scaling: amax of a bf16 [rows, cols] matrix (leading dimension ld) -> *amax_bits (the bit
// pattern of the fp32 amax; zeroed by the caller, atomicMax), then q = fp8(v * s) row-major [rows, cols] and/or
// qt = q^T [cols, rows] (either may be null; both contiguous), and *scale_inv = 1/s.
void launch_quantize_fp8_amax(const void* x, int64_t rows, int64_t cols, int64_t ld, unsigned int* amax_bits,
                              int sm_count, cudaStream_t stream);
void launch_quantize_fp8_cast(const void* x, int64_t rows, int64_t cols, int64_t ld, bool e5m2,
                              const unsigned int* amax_bits, void* q, void* qt, float* scale_inv, cudaStream_t stream);
// C[M,N] = A[M,K] * B[N,K]^T with both operands K-major fp8 (A E4M3, or E5M2 when a_e5m2; B E4M3), dequantized by the
// device scalars 1/s_a, 1/s_b.  K % 16, lda % 16, ldb % 16 == 0 and 16-byte-aligned bases (TMA), N % 8 == 0.
bool gemm_fp8_tn_supported(int64_t M, int64_t N, int64_t K, const void* A, const void* B, const void* C, int64_t lda,
                           int64_t ldb, int64_t ldc);
// C = bf16(gscale * acc / (s_a s_b)) (gscale optional)
void launch_gemm_fp8_tn(const void* A, bool a_e5m2, const void* B, void* C, int64_t M, int64_t N, int64_t K, int64_t lda,
                        int64_t ldb, int64_t ldc, const float* a_scale_inv, const float* b_scale_inv, const float* gscale,
                        int sm_count, cudaStream_t stream);
// A E4M3: dy = bf16(grad_scale (acc / (s_a s_b) - target)), the loss as MseEpilogue, *dy_amax = bits of max |dy|
// over the stored bf16 values (atomicMax; zeroed by the caller).
void launch_gemm_fp8_mse(const void* A, const void* B, void* dy, int64_t M, int64_t N, int64_t K, int64_t lda,
                         int64_t ldb, int64_t ldc, const float* a_scale_inv, const float* b_scale_inv,
                         const MseEpilogue& mse, unsigned int* dy_amax, int sm_count, cudaStream_t stream);
// W[M,N] (bf16, in place) = bf16(W + alpha * gscale * acc / (s_a s_b)).
void launch_gemm_fp8_sgd(const void* A, bool a_e5m2, const void* B, void* W, int64_t M, int64_t N, int64_t K,
                         int64_t lda, int64_t ldb, int64_t ldw, const float* a_scale_inv, const float* b_scale_inv,
                         float alpha, const float* gscale, int sm_count, cudaStream_t stream);

// Plain device copy into the heap (used to stage the weight for the fused kernel).
void launch_copy_bytes(void* dst, const void* src, int64_t bytes, int sm_count, cudaStream_t stream);

// Fills `n` bytes with zero (used for non-root results / backward recv buffers).
void launch_zero(void* p, int64_t bytes, int sm_count, cudaStream_t stream);

}  // namespace m4t
