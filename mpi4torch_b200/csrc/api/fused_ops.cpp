// Tensor-core ops exposed to Python: the wgmma GEMM and the fused
// Allreduce->GEMM linear forward (BASELINE.json config "4096x4096 linear layer:
// Allreduce(params)->GEMM fused").  The reference has no fused op and no GPU
// kernel at all (SURVEY 2.4); its equivalent is Allreduce + `/ size` + matmul
// as three library calls (reference examples/simple_linear_regression.py:29).
#include <c10/cuda/CUDAGuard.h>
#include <c10/cuda/CUDAStream.h>
#include <torch/library.h>
#include <torch/torch.h>

#include "../runtime/cuda_backend.h"
#include "../runtime/world.h"
#include "communicator.h"

namespace m4t {

namespace {

using torch::Tensor;

CudaBackend& backend() {
  World& w = World::instance();
  TORCH_CHECK(w.cuda_ready(), "mpi4torch_b200: the CUDA backend is not initialised");
  return *w.cuda();
}

cudaStream_t stream_of(const Tensor& t) { return c10::cuda::getCurrentCUDAStream(t.device().index()).stream(); }

int sm_count() { return backend().device_comm().sm_count; }

void check_2d_bf16(const Tensor& t, const char* name) {
  TORCH_CHECK(t.is_cuda() && t.dim() == 2 && t.scalar_type() == at::kBFloat16 && t.stride(1) == 1,
              "mpi4torch_b200: ", name, " must be a 2-d bf16 CUDA tensor with unit inner stride");
}

// An MSE target [M, N] the GEMM epilogues can read: bf16 with unit inner stride, read as pairs.
bool mse_target_ok(const Tensor& t, int64_t M, int64_t N) {
  return t.is_cuda() && t.dim() == 2 && t.scalar_type() == at::kBFloat16 && t.stride(1) == 1 && t.size(0) == M &&
         t.size(1) == N && epilogue_bf16_pairs_ok(t.data_ptr(), t.stride(0));
}

// The MSE epilogue against `target`, adding its loss into the fp32 scalar `loss`.
MseEpilogue mse_epilogue(const Tensor& target, const Tensor& loss, double loss_scale, double grad_scale) {
  return MseEpilogue{target.data_ptr(), target.stride(0), loss.data_ptr<float>(), static_cast<float>(loss_scale),
                     static_cast<float>(grad_scale)};
}

// y = x @ w^T on the wgmma path.
Tensor gemm_bf16_tn(const Tensor& x, const Tensor& w) {
  check_2d_bf16(x, "x");
  check_2d_bf16(w, "w");
  TORCH_CHECK(x.size(1) == w.size(1), "mpi4torch_b200: inner dimensions differ");
  c10::cuda::CUDAGuard guard(x.device());
  Tensor y = at::empty({x.size(0), w.size(0)}, x.options());
  if (y.numel() == 0) return y;
  std::lock_guard<std::recursive_mutex> g(World::instance().mutex());
  backend().gemm_bf16_tn(x.data_ptr(), w.data_ptr(), y.data_ptr(), x.size(0), w.size(0), x.size(1), x.stride(0),
                         w.stride(0), y.stride(0), stream_of(x));
  return y;
}

// y = a @ b with both operands row-major (dgrad: gy[M,N] @ W[N,K]); the weight is read in place through an
// MN-major wgmma operand, no transposed copy.
bool gemm_bf16_nn_ok(const Tensor& a, const Tensor& b) {
  if (!(a.is_cuda() && b.is_cuda() && a.dim() == 2 && b.dim() == 2 && a.scalar_type() == at::kBFloat16 &&
        b.scalar_type() == at::kBFloat16 && a.stride(1) == 1 && b.stride(1) == 1 && a.size(1) == b.size(0)))
    return false;
  return World::instance().cuda_ready() &&
         gemm_bf16_nn_supported(a.size(0), b.size(1), a.size(1), a.data_ptr(), b.data_ptr(), a.data_ptr(), a.stride(0),
                                b.stride(0), b.size(1));
}

Tensor gemm_bf16_nn(const Tensor& a, const Tensor& b) {
  check_2d_bf16(a, "a");
  check_2d_bf16(b, "b");
  TORCH_CHECK(a.size(1) == b.size(0), "mpi4torch_b200: inner dimensions differ");
  c10::cuda::CUDAGuard guard(a.device());
  Tensor y = at::empty({a.size(0), b.size(1)}, a.options());
  if (y.numel() == 0) return y;
  std::lock_guard<std::recursive_mutex> g(World::instance().mutex());
  launch_gemm_bf16_nn(a.data_ptr(), b.data_ptr(), y.data_ptr(), a.size(0), b.size(1), a.size(1), a.stride(0),
                      b.stride(0), y.stride(0), sm_count(), stream_of(a));
  return y;
}

// Also answers for the epilogue operands when given: an MSE target [M, N] (bf16) and a bias [N] (fp32).
bool gemm_bf16_tn_ok(const Tensor& x, const Tensor& w, const c10::optional<Tensor>& target,
                     const c10::optional<Tensor>& bias) {
  if (!(x.is_cuda() && w.is_cuda() && x.dim() == 2 && w.dim() == 2 && x.scalar_type() == at::kBFloat16 &&
        w.scalar_type() == at::kBFloat16 && x.stride(1) == 1 && w.stride(1) == 1 && x.size(1) == w.size(1)))
    return false;
  if (target.has_value() && !mse_target_ok(*target, x.size(0), w.size(0))) return false;
  if (bias.has_value() && !(bias->is_cuda() && bias->dim() == 1 && bias->scalar_type() == at::kFloat &&
                            bias->is_contiguous() && bias->size(0) == w.size(0) && epilogue_bias_ok(bias->data_ptr<float>())))
    return false;
  return World::instance().cuda_ready() &&
         gemm_bf16_tn_supported(x.size(0), w.size(0), x.size(1), x.data_ptr(), w.data_ptr(), x.data_ptr(), x.stride(0),
                                w.stride(0), w.size(0));
}

bool allreduce_linear_supported(const Tensor& x, const Tensor& w) {
  if (!World::instance().cuda_ready()) return false;
  if (!(x.is_cuda() && w.is_cuda() && x.dim() == 2 && w.dim() == 2 && x.scalar_type() == at::kBFloat16 &&
        w.scalar_type() == at::kBFloat16 && x.is_contiguous() && w.is_contiguous() && x.size(1) == w.size(1)))
    return false;
  return backend().fused_linear_available(w.size(0), w.size(1));
}

// (y, w_avg) with y = x @ (scale * sum_ranks w)^T, one kernel.  w_avg aliases
// symmetric-heap memory that stays valid until the call after next.
std::tuple<Tensor, Tensor> allreduce_linear_fused(const Tensor& x, const Tensor& w, double scale) {
  TORCH_CHECK(allreduce_linear_supported(x, w), "mpi4torch_b200: fused Allreduce->GEMM does not support these tensors");
  c10::cuda::CUDAGuard guard(x.device());
  Tensor y = at::empty({x.size(0), w.size(0)}, x.options());
  std::lock_guard<std::recursive_mutex> g(World::instance().mutex());
  const void* wavg = backend().fused_allreduce_linear(
      x.data_ptr(), w.data_ptr(), y.data_ptr(), x.size(0), w.size(0), x.size(1), x.stride(0), y.stride(0),
      static_cast<float>(scale), stream_of(x));
  Tensor w_avg = torch::from_blob(const_cast<void*>(wavg), {w.size(0), w.size(1)}, w.options());
  return {y, w_avg};
}

// Training forward of the data-parallel linear layer with everything fused:
//   W_avg = scale * sum_ranks W          (inside the GEMM kernel when NVLS is up)
//   y     = x @ W_avg^T                  (wgmma, never stored)
//   dy    = grad_scale * (y - target)    (GEMM epilogue)
//   loss  = loss_scale * sum((y-target)^2)  (GEMM epilogue, one atomic per warp per tile)
// Returns (dy, loss[1] fp32, W_avg).
std::tuple<Tensor, Tensor, Tensor> linear_mse_forward(const Tensor& x, const Tensor& w, const Tensor& target, double scale,
                                                      double loss_scale, double grad_scale, bool allow_fused) {
  check_2d_bf16(x, "x");
  check_2d_bf16(w, "w");
  check_2d_bf16(target, "target");
  TORCH_CHECK(x.size(1) == w.size(1) && target.size(0) == x.size(0) && target.size(1) == w.size(0),
              "mpi4torch_b200: linear_mse_forward shape mismatch");
  // checked here as well as in the GEMM launchers: with more than one rank a weight average is launched first
  TORCH_CHECK(epilogue_bf16_pairs_ok(target.data_ptr(), target.stride(0)),
              "mpi4torch_b200: the MSE target needs a 4-byte-aligned base and an even row stride");
  c10::cuda::CUDAGuard guard(x.device());
  cudaStream_t stream = stream_of(x);
  Tensor dy = at::empty({x.size(0), w.size(0)}, x.options());
  Tensor loss = at::zeros({1}, x.options().dtype(at::kFloat));
  const MseEpilogue mse = mse_epilogue(target, loss, loss_scale, grad_scale);
  std::lock_guard<std::recursive_mutex> g(World::instance().mutex());
  CudaBackend& be = backend();
  Tensor w_avg;
  if (allow_fused && be.size() > 1 && x.is_contiguous() && w.is_contiguous() && be.fused_linear_available(w.size(0), w.size(1))) {
    const void* wavg = be.fused_allreduce_linear(x.data_ptr(), w.data_ptr(), dy.data_ptr(), x.size(0), w.size(0), x.size(1),
                                                 x.stride(0), dy.stride(0), static_cast<float>(scale), stream, &mse);
    w_avg = torch::from_blob(const_cast<void*>(wavg), {w.size(0), w.size(1)}, w.options());
  } else {
    if (be.size() > 1) {
      w_avg = at::empty_like(w, at::MemoryFormat::Contiguous);
      Tensor wc = w.contiguous();
      Epilogue epi;
      epi.scale = scale;
      epi.has_scale = true;
      be.allreduce(wc.data_ptr(), w_avg.data_ptr(), wc.numel(), DType::BF16, ReduceOp::SUM, epi, stream);
    } else {
      w_avg = w;
    }
    be.gemm_bf16_tn(x.data_ptr(), w_avg.data_ptr(), dy.data_ptr(), x.size(0), w_avg.size(0), x.size(1), x.stride(0),
                    w_avg.stride(0), dy.stride(0), stream, &mse);
  }
  return {dy, loss, w_avg};
}

// Tensor backed by the symmetric heap's persistent arena (same offset on every
// rank when all ranks allocate in the same order).  Kernels that need peer- or
// switch-visible inputs use such tensors in place instead of staging them.
Tensor symmetric_empty(c10::IntArrayRef shape, c10::ScalarType dtype) {
  std::lock_guard<std::recursive_mutex> g(World::instance().mutex());
  CudaBackend& be = backend();
  int64_t numel = 1;
  for (int64_t d : shape) numel *= d;
  const int64_t bytes = numel * static_cast<int64_t>(c10::elementSize(dtype));
  auto opts = at::TensorOptions().dtype(dtype).device(c10::Device(c10::kCUDA, static_cast<c10::DeviceIndex>(be.device())));
  if (be.size() <= 1) return at::empty(shape, opts);  // no peers: ordinary memory is as good
  const int64_t off = be.symm_alloc(bytes);
  return torch::from_blob(be.symm_ptr(off), shape, opts);
}

// param <- param + scale * Allreduce(grad): the gradient all-reduce with the
// optimizer update as its epilogue, in place.
void allreduce_axpy_(Tensor param, const Tensor& grad, double scale, int64_t max_blocks) {
  auto comm = c10::make_intrusive<Communicator>();
  comm->raw_allreduce_axpy_(param, grad, scale, max_blocks);
}

const float* grad_scale_ptr(const c10::optional<Tensor>& gs, const Tensor& like) {
  if (!gs.has_value() || !gs->defined()) return nullptr;
  TORCH_CHECK(gs->is_cuda() && gs->device() == like.device() && gs->scalar_type() == at::kFloat && gs->numel() == 1,
              "mpi4torch_b200: grad_scale must be a one-element fp32 tensor on the same device");
  return gs->data_ptr<float>();
}

// G = grad_scale * dy^T @ x on the wgmma path with MN-major operands (no transposed copies).
// grad_scale is a device scalar (the upstream gradient of the loss as autograd delivers it).
Tensor wgrad_bf16(const Tensor& dy, const Tensor& x, const c10::optional<Tensor>& grad_scale) {
  check_2d_bf16(dy, "dy");
  check_2d_bf16(x, "x");
  TORCH_CHECK(dy.size(0) == x.size(0), "mpi4torch_b200: batch dimensions differ");
  c10::cuda::CUDAGuard guard(x.device());
  Tensor gw = at::empty({dy.size(1), x.size(1)}, x.options());
  std::lock_guard<std::recursive_mutex> g(World::instance().mutex());
  launch_wgrad_bf16(dy.data_ptr(), x.data_ptr(), gw.data_ptr(), dy.size(0), dy.size(1), x.size(1), dy.stride(0),
                    x.stride(0), gw.stride(0), sm_count(), stream_of(x), grad_scale_ptr(grad_scale, x));
  return gw;
}

// w += scale * grad_scale * dy^T @ x: the single-rank SGD step as the wgrad GEMM's own epilogue
// (no gradient tensor, one kernel).  Not a collective.
void wgrad_sgd_(Tensor w, const Tensor& dy, const Tensor& x, double scale, const c10::optional<Tensor>& grad_scale) {
  check_2d_bf16(dy, "dy");
  check_2d_bf16(x, "x");
  check_2d_bf16(w, "w");
  TORCH_CHECK(dy.size(0) == x.size(0) && w.size(0) == dy.size(1) && w.size(1) == x.size(1),
              "mpi4torch_b200: wgrad_sgd_ shape mismatch");
  TORCH_CHECK(scale != 0.0, "mpi4torch_b200: wgrad_sgd_ needs a non-zero scale");
  c10::cuda::CUDAGuard guard(x.device());
  std::lock_guard<std::recursive_mutex> g(World::instance().mutex());
  launch_wgrad_bf16(dy.data_ptr(), x.data_ptr(), w.data_ptr(), dy.size(0), dy.size(1), x.size(1), dy.stride(0),
                    x.stride(0), w.stride(0), sm_count(), stream_of(x), grad_scale_ptr(grad_scale, x),
                    static_cast<float>(scale));
}

bool wgrad_bf16_ok(const Tensor& dy, const Tensor& x) {
  if (!(dy.is_cuda() && x.is_cuda() && dy.dim() == 2 && x.dim() == 2 && dy.scalar_type() == at::kBFloat16 &&
        x.scalar_type() == at::kBFloat16 && dy.stride(1) == 1 && x.stride(1) == 1 && dy.size(0) == x.size(0)))
    return false;
  return World::instance().cuda_ready() &&
         wgrad_bf16_supported(dy.size(0), dy.size(1), x.size(1), dy.data_ptr(), x.data_ptr(), x.data_ptr(), dy.stride(0),
                              x.stride(0), x.size(1));
}

// The rules of wgrad_bf16_supported, and acc a contiguous, 16-byte-aligned fp32 [N, K] tensor on x's device.
bool wgrad_accumulate_ok(const Tensor& acc, const Tensor& dy, const Tensor& x) {
  if (!wgrad_bf16_ok(dy, x)) return false;
  if (!(acc.is_cuda() && acc.device() == x.device() && dy.device() == x.device() && acc.dim() == 2 &&
        acc.scalar_type() == at::kFloat && acc.is_contiguous() && acc.size(0) == dy.size(1) && acc.size(1) == x.size(1)))
    return false;
  return wgrad_bf16_supported(dy.size(0), dy.size(1), x.size(1), dy.data_ptr(), x.data_ptr(), acc.data_ptr<float>(),
                              dy.stride(0), x.stride(0), x.size(1));
}

// acc += grad_scale * dy^T @ x, accumulated in fp32 by the wgrad kernel's epilogue with one fmaf per element
// (gradient accumulation over micro-batches).  Not a collective.
void wgrad_accumulate_(Tensor acc, const Tensor& dy, const Tensor& x, const c10::optional<Tensor>& grad_scale) {
  TORCH_CHECK(wgrad_accumulate_ok(acc, dy, x),
              "mpi4torch_b200: wgrad_accumulate_ needs bf16 dy [B, N] and x [B, K] with unit inner strides, N % 128 == "
              "K % 128 == B % 64 == 0, 16-byte-aligned operands, and acc a contiguous 16-byte-aligned fp32 [N, K] "
              "tensor on the same device");
  c10::cuda::CUDAGuard guard(x.device());
  std::lock_guard<std::recursive_mutex> g(World::instance().mutex());
  launch_wgrad_accumulate(dy.data_ptr(), x.data_ptr(), acc.data_ptr<float>(), dy.size(0), dy.size(1), x.size(1),
                          dy.stride(0), x.stride(0), sm_count(), stream_of(x), grad_scale_ptr(grad_scale, x));
}

bool wgrad_allreduce_sgd_supported(const Tensor& w, const Tensor& dy, const Tensor& x) {
  if (!World::instance().cuda_ready() || !wgrad_bf16_ok(dy, x)) return false;
  if (!(w.is_cuda() && w.dim() == 2 && w.scalar_type() == at::kBFloat16 && w.is_contiguous() &&
        w.size(0) == dy.size(1) && w.size(1) == x.size(1)))
    return false;
  return backend().fused_wgrad_available(w.data_ptr(), dy.size(0), w.size(0), w.size(1));
}

// w += scale * sum_ranks(dy^T @ x): backward GEMM, gradient all-reduce and SGD step in one kernel.
// Collective; `w` must be a replicated symmetric_empty() tensor (M4T_FUSED_WGRAD=0 disables the kernel).
void wgrad_allreduce_sgd_(Tensor w, const Tensor& dy, const Tensor& x, double scale,
                          const c10::optional<Tensor>& grad_scale) {
  TORCH_CHECK(wgrad_allreduce_sgd_supported(w, dy, x), "mpi4torch_b200: fused wgrad->Allreduce->SGD does not support these tensors");
  c10::cuda::CUDAGuard guard(x.device());
  std::lock_guard<std::recursive_mutex> g(World::instance().mutex());
  backend().fused_wgrad_update(w.data_ptr(), dy.data_ptr(), x.data_ptr(), dy.size(0), w.size(0), w.size(1), dy.stride(0),
                               x.stride(0), static_cast<float>(scale), stream_of(x), false, grad_scale_ptr(grad_scale, x));
}

// Same kernel, and additionally the parameter all-reduce of the NEXT forward: returns
// W_avg = (1/size) * sum_ranks w_new (symmetric-heap memory, valid until the next call).
Tensor wgrad_allreduce_sgd_prefetch_(Tensor w, const Tensor& dy, const Tensor& x, double scale,
                                     const c10::optional<Tensor>& grad_scale) {
  TORCH_CHECK(wgrad_allreduce_sgd_supported(w, dy, x), "mpi4torch_b200: fused wgrad->Allreduce->SGD does not support these tensors");
  c10::cuda::CUDAGuard guard(x.device());
  std::lock_guard<std::recursive_mutex> g(World::instance().mutex());
  const void* wavg = backend().fused_wgrad_update(w.data_ptr(), dy.data_ptr(), x.data_ptr(), dy.size(0), w.size(0), w.size(1),
                                                  dy.stride(0), x.stride(0), static_cast<float>(scale), stream_of(x),
                                                  true, grad_scale_ptr(grad_scale, x));
  return torch::from_blob(const_cast<void*>(wavg), {w.size(0), w.size(1)}, w.options().requires_grad(false));
}

// Forward + fused MSE epilogue against weights that are ALREADY averaged (no collective):
// (dL/dy, loss[1]).  Pairs with wgrad_allreduce_sgd_prefetch_.
std::tuple<Tensor, Tensor> linear_mse_forward_local(const Tensor& x, const Tensor& w_avg, const Tensor& target,
                                                    double loss_scale, double grad_scale) {
  check_2d_bf16(x, "x");
  check_2d_bf16(w_avg, "w_avg");
  check_2d_bf16(target, "target");
  TORCH_CHECK(x.size(1) == w_avg.size(1) && target.size(0) == x.size(0) && target.size(1) == w_avg.size(0),
              "mpi4torch_b200: linear_mse_forward_local shape mismatch");
  c10::cuda::CUDAGuard guard(x.device());
  cudaStream_t stream = stream_of(x);
  Tensor dy = at::empty({x.size(0), w_avg.size(0)}, x.options());
  Tensor loss = at::zeros({1}, x.options().dtype(at::kFloat));
  const MseEpilogue mse = mse_epilogue(target, loss, loss_scale, grad_scale);
  std::lock_guard<std::recursive_mutex> g(World::instance().mutex());
  backend().gemm_bf16_tn(x.data_ptr(), w_avg.data_ptr(), dy.data_ptr(), x.size(0), w_avg.size(0), x.size(1), x.stride(0),
                         w_avg.stride(0), dy.stride(0), stream, &mse);
  return {dy, loss};
}

// ---- two-layer MLP (Linear -> GELU(tanh) -> Linear, MSE) ------------------------------------------
void check_bias(const Tensor& b, const Tensor& w) {
  TORCH_CHECK(b.is_cuda() && b.device() == w.device() && b.dim() == 1 && b.scalar_type() == at::kFloat &&
                  b.is_contiguous() && b.size(0) == w.size(0),
              "mpi4torch_b200: the bias must be a contiguous fp32 CUDA vector of the weight's output size");
}

Tensor colsum_workspace(int64_t M, int64_t N, const Tensor& like) {
  return at::empty({colsum_rows(M), N}, like.options().dtype(at::kFloat));
}

// (h, z) with z = x @ w^T + b and h = gelu_tanh(z), both bf16; h is computed from the fp32 z.
std::tuple<Tensor, Tensor> linear_bias_gelu_forward(const Tensor& x, const Tensor& w, const Tensor& b) {
  check_2d_bf16(x, "x");
  check_2d_bf16(w, "w");
  check_bias(b, w);
  TORCH_CHECK(x.size(1) == w.size(1), "mpi4torch_b200: inner dimensions differ");
  c10::cuda::CUDAGuard guard(x.device());
  Tensor z = at::empty({x.size(0), w.size(0)}, x.options());
  Tensor h = at::empty_like(z);
  if (z.numel() == 0) return {h, z};
  std::lock_guard<std::recursive_mutex> g(World::instance().mutex());
  launch_gemm_bias_gelu(x.data_ptr(), w.data_ptr(), b.data_ptr<float>(), z.data_ptr(), h.data_ptr(), x.size(0), w.size(0),
                        x.size(1), x.stride(0), w.stride(0), z.stride(0), sm_count(), stream_of(x));
  return {h, z};
}

// Forward of the output layer with the MSE epilogue, against already averaged parameters:
//   dy = grad_scale * (x @ w^T + b - target)  (bf16),  loss[1] = loss_scale * sum((x @ w^T + b - target)^2),
//   partials = fp32 column-sum partials of dy (reduce them with column_sum).
std::tuple<Tensor, Tensor, Tensor> linear_bias_mse_forward_local(const Tensor& x, const Tensor& w, const Tensor& b,
                                                                 const Tensor& target, double loss_scale,
                                                                 double grad_scale) {
  check_2d_bf16(x, "x");
  check_2d_bf16(w, "w");
  check_2d_bf16(target, "target");
  check_bias(b, w);
  TORCH_CHECK(x.size(1) == w.size(1) && target.size(0) == x.size(0) && target.size(1) == w.size(0),
              "mpi4torch_b200: linear_bias_mse_forward_local shape mismatch");
  TORCH_CHECK(x.size(0) > 0, "mpi4torch_b200: linear_bias_mse_forward_local needs a non-empty batch");
  c10::cuda::CUDAGuard guard(x.device());
  Tensor dy = at::empty({x.size(0), w.size(0)}, x.options());
  Tensor loss = at::zeros({1}, x.options().dtype(at::kFloat));
  Tensor part = colsum_workspace(x.size(0), w.size(0), x);
  const MseEpilogue mse = mse_epilogue(target, loss, loss_scale, grad_scale);
  std::lock_guard<std::recursive_mutex> g(World::instance().mutex());
  launch_gemm_bias_mse_colsum(x.data_ptr(), w.data_ptr(), b.data_ptr<float>(), dy.data_ptr(), part.data_ptr<float>(),
                              x.size(0), w.size(0), x.size(1), x.stride(0), w.stride(0), dy.stride(0),
                              sm_count(), stream_of(x),
                              mse);
  return {dy, loss, part};
}

// Forward of the output layer with the softmax cross-entropy loss, against already averaged parameters:
//   logits = bf16(x @ w^T + b),  lse[r] = log sum_c exp(logits[r, c]),
//   dy = grad_scale * (softmax(logits) - onehot(labels))  (bf16, written over the logits),
//   loss[1] = loss_scale * sum_r (lse[r] - logits[r, labels[r]]), summed in a fixed order,
//   partials = fp32 column-sum partials of dy, as linear_bias_mse_forward_local returns them.
// A row labelled ignore_index gets a zero dy row and adds nothing to the loss; any other label outside [0, C) makes
// its dy row and the loss NaN (it is never used as an index).
std::tuple<Tensor, Tensor, Tensor> linear_bias_xent_forward_local(const Tensor& x, const Tensor& w, const Tensor& b,
                                                                  const Tensor& labels, double loss_scale,
                                                                  double grad_scale, int64_t ignore_index) {
  check_2d_bf16(x, "x");
  check_2d_bf16(w, "w");
  check_bias(b, w);
  TORCH_CHECK(labels.is_cuda() && labels.device() == x.device() && labels.dim() == 1 &&
                  labels.scalar_type() == at::kLong && labels.is_contiguous() && labels.size(0) == x.size(0),
              "mpi4torch_b200: labels must be a contiguous 1-d int64 CUDA tensor with one label per row of x");
  TORCH_CHECK(x.size(1) == w.size(1), "mpi4torch_b200: linear_bias_xent_forward_local shape mismatch");
  TORCH_CHECK(x.size(0) > 0, "mpi4torch_b200: linear_bias_xent_forward_local needs a non-empty batch");
  c10::cuda::CUDAGuard guard(x.device());
  const int64_t M = x.size(0), C = w.size(0);
  Tensor dy = at::empty({M, C}, x.options());
  Tensor loss = at::empty({1}, x.options().dtype(at::kFloat));
  Tensor part = colsum_workspace(M, C, x);
  Tensor ms = at::empty({xent_tiles(C), M, 2}, x.options().dtype(at::kFloat));
  Tensor row_loss = at::empty({M}, x.options().dtype(at::kFloat));
  Tensor done = at::zeros({1}, x.options().dtype(at::kInt));
  cudaStream_t stream = stream_of(x);
  std::lock_guard<std::recursive_mutex> g(World::instance().mutex());
  float2* ms_ptr = reinterpret_cast<float2*>(ms.data_ptr<float>());
  launch_gemm_bias_xent(x.data_ptr(), w.data_ptr(), b.data_ptr<float>(), dy.data_ptr(), ms_ptr, M, C, x.size(1),
                        x.stride(0), w.stride(0), dy.stride(0), sm_count(), stream);
  launch_xent_finish(dy.data_ptr(), M, C, dy.stride(0), ms_ptr, labels.data_ptr<int64_t>(), ignore_index,
                     static_cast<float>(loss_scale), static_cast<float>(grad_scale), row_loss.data_ptr<float>(),
                     reinterpret_cast<unsigned int*>(done.data_ptr<int>()), loss.data_ptr<float>(), part.data_ptr<float>(),
                     stream);
  return {dy, loss, part};
}

// (dz, partials): dz = grad_scale * (dy @ w) * gelu_tanh'(z) in bf16 (w read in place as in gemm_bf16_nn), and the
// fp32 column-sum partials of dz.
std::tuple<Tensor, Tensor> gemm_nn_gelu_backward(const Tensor& dy, const Tensor& w, const Tensor& z,
                                                 const c10::optional<Tensor>& grad_scale) {
  check_2d_bf16(dy, "dy");
  check_2d_bf16(w, "w");
  check_2d_bf16(z, "z");
  TORCH_CHECK(dy.size(1) == w.size(0) && z.size(0) == dy.size(0) && z.size(1) == w.size(1),
              "mpi4torch_b200: gemm_nn_gelu_backward shape mismatch");
  TORCH_CHECK(dy.size(0) > 0, "mpi4torch_b200: gemm_nn_gelu_backward needs a non-empty batch");
  c10::cuda::CUDAGuard guard(dy.device());
  Tensor dz = at::empty({dy.size(0), w.size(1)}, dy.options());
  Tensor part = colsum_workspace(dy.size(0), w.size(1), dy);
  std::lock_guard<std::recursive_mutex> g(World::instance().mutex());
  launch_gemm_nn_gelu_bwd_colsum(dy.data_ptr(), w.data_ptr(), z.data_ptr(), dz.data_ptr(), part.data_ptr<float>(), dy.size(0),
                                 w.size(1), dy.size(1), dy.stride(0), w.stride(0), z.stride(0), dz.stride(0),
                                 sm_count(), stream_of(dy), grad_scale_ptr(grad_scale, dy));
  return {dz, part};
}

// out[n] = grad_scale * sum_i partials[i, n] (fp32), in a fixed order of i: bit-identical on every call.
Tensor column_sum(const Tensor& partials, const c10::optional<Tensor>& grad_scale) {
  TORCH_CHECK(partials.is_cuda() && partials.dim() == 2 && partials.scalar_type() == at::kFloat && partials.is_contiguous() &&
                  partials.size(0) > 0,
              "mpi4torch_b200: column_sum needs a non-empty contiguous 2-d fp32 CUDA tensor");
  c10::cuda::CUDAGuard guard(partials.device());
  Tensor out = at::empty({partials.size(1)}, partials.options());
  if (out.numel() == 0) return out;
  launch_column_sum(partials.data_ptr<float>(), partials.size(0), partials.size(1), out.data_ptr<float>(),
                    grad_scale_ptr(grad_scale, partials), stream_of(partials));
  return out;
}

// ---- batched experts (E experts of one shape per launch) ---------------------------------------------------------
// Operands are contiguous bf16 CUDA tensors stacked along dim 0 on one device; see batched_gemm_supported.
bool bf16_3d(const Tensor& t) {
  return t.is_cuda() && t.dim() == 3 && t.scalar_type() == at::kBFloat16 && t.is_contiguous();
}

bool same_device(std::initializer_list<const Tensor*> ts) {
  for (const Tensor* t : ts)
    if (t->device() != (*ts.begin())->device()) return false;
  return true;
}

// x [E, M, K] @ w [E, N, K]^T, and the bias [E, N] (contiguous fp32, 8-byte aligned) when given.
bool batched_gemm_tn_ok(const Tensor& x, const Tensor& w, const c10::optional<Tensor>& bias) {
  if (!(bf16_3d(x) && bf16_3d(w) && same_device({&x, &w}) && x.size(0) == w.size(0) && x.size(2) == w.size(2)))
    return false;
  if (bias.has_value() && !(bias->is_cuda() && bias->device() == x.device() && bias->dim() == 2 &&
                            bias->scalar_type() == at::kFloat && bias->is_contiguous() && bias->size(0) == w.size(0) &&
                            bias->size(1) == w.size(1) && epilogue_bias_ok(bias->data_ptr<float>())))
    return false;
  return World::instance().cuda_ready() &&
         batched_gemm_supported(x.size(0), x.size(1), w.size(1), x.size(2), x.data_ptr(), w.data_ptr(), x.data_ptr());
}

// a [E, M, K] @ b [E, K, N].
bool batched_gemm_nn_ok(const Tensor& a, const Tensor& b) {
  if (!(bf16_3d(a) && bf16_3d(b) && same_device({&a, &b}) && a.size(0) == b.size(0) && a.size(2) == b.size(1)))
    return false;
  return World::instance().cuda_ready() &&
         batched_gemm_supported(a.size(0), a.size(1), b.size(2), a.size(2), a.data_ptr(), b.data_ptr(), a.data_ptr());
}

// dy [E, M, N]^T @ x [E, M, K] per expert.
bool batched_wgrad_bf16_ok(const Tensor& dy, const Tensor& x) {
  if (!(bf16_3d(dy) && bf16_3d(x) && same_device({&dy, &x}) && dy.size(0) == x.size(0) && dy.size(1) == x.size(1)))
    return false;
  return World::instance().cuda_ready() && wgrad_bf16_batched_supported(dy.size(0), dy.size(1), dy.size(2), x.size(2),
                                                                         dy.data_ptr(), x.data_ptr(), x.data_ptr());
}

// (h, z) per expert: z_e = x_e @ w_e^T + b_e, h_e = gelu_tanh(z_e), as linear_bias_gelu_forward, in one launch.
std::tuple<Tensor, Tensor> batched_linear_bias_gelu_forward(const Tensor& x, const Tensor& w, const Tensor& b) {
  TORCH_CHECK(batched_gemm_tn_ok(x, w, b),
              "mpi4torch_b200: batched_linear_bias_gelu_forward needs contiguous bf16 x [E, M, K], w [E, N, K] and fp32 "
              "b [E, N] on one CUDA device, M % 128 == N % 128 == K % 128 == 0, and aligned bases");
  c10::cuda::CUDAGuard guard(x.device());
  Tensor z = at::empty({x.size(0), x.size(1), w.size(1)}, x.options());
  Tensor h = at::empty_like(z);
  std::lock_guard<std::recursive_mutex> g(World::instance().mutex());
  launch_gemm_bias_gelu_batched(x.data_ptr(), w.data_ptr(), b.data_ptr<float>(), z.data_ptr(), h.data_ptr(), x.size(0),
                                x.size(1), w.size(1), x.size(2), sm_count(), stream_of(x));
  return {h, z};
}

// y_e = bf16(x_e @ w_e^T + b_e), one launch.
Tensor batched_linear_bias_forward(const Tensor& x, const Tensor& w, const Tensor& b) {
  TORCH_CHECK(batched_gemm_tn_ok(x, w, b),
              "mpi4torch_b200: batched_linear_bias_forward needs contiguous bf16 x [E, M, K], w [E, N, K] and fp32 "
              "b [E, N] on one CUDA device, M % 128 == N % 128 == K % 128 == 0, and aligned bases");
  c10::cuda::CUDAGuard guard(x.device());
  Tensor y = at::empty({x.size(0), x.size(1), w.size(1)}, x.options());
  std::lock_guard<std::recursive_mutex> g(World::instance().mutex());
  launch_gemm_bias_batched(x.data_ptr(), w.data_ptr(), b.data_ptr<float>(), y.data_ptr(), x.size(0), x.size(1), w.size(1),
                           x.size(2), sm_count(), stream_of(x));
  return y;
}

// (dz, partials) per expert: dz_e = grad_scale * (dy_e @ w_e) * gelu_tanh'(z_e) (w [E, K, N] read in place), and the
// column-sum partials of dz as [E, M / 16, N] (reduce them with batched_column_sum).
std::tuple<Tensor, Tensor> batched_gemm_nn_gelu_backward(const Tensor& dy, const Tensor& w, const Tensor& z,
                                                         const c10::optional<Tensor>& grad_scale) {
  TORCH_CHECK(batched_gemm_nn_ok(dy, w) && bf16_3d(z) && z.device() == dy.device() && z.size(0) == dy.size(0) &&
                  z.size(1) == dy.size(1) && z.size(2) == w.size(2),
              "mpi4torch_b200: batched_gemm_nn_gelu_backward needs contiguous bf16 dy [E, M, K], w [E, K, N] and "
              "z [E, M, N] on one CUDA device, M % 128 == N % 128 == K % 128 == 0, and aligned bases");
  c10::cuda::CUDAGuard guard(dy.device());
  const int64_t E = dy.size(0), M = dy.size(1), N = w.size(2);
  Tensor dz = at::empty({E, M, N}, dy.options());
  Tensor part = at::empty({E, colsum_rows(M), N}, dy.options().dtype(at::kFloat));
  std::lock_guard<std::recursive_mutex> g(World::instance().mutex());
  launch_gemm_nn_gelu_bwd_colsum_batched(dy.data_ptr(), w.data_ptr(), z.data_ptr(), dz.data_ptr(), part.data_ptr<float>(),
                                         E, M, N, dy.size(2), sm_count(), stream_of(dy), grad_scale_ptr(grad_scale, dy));
  return {dz, part};
}

// c_e = a_e @ b_e with b [E, K, N] read in place, one launch.
Tensor batched_gemm_nn(const Tensor& a, const Tensor& b) {
  TORCH_CHECK(batched_gemm_nn_ok(a, b),
              "mpi4torch_b200: batched_gemm_nn needs contiguous bf16 a [E, M, K] and b [E, K, N] on one CUDA device, "
              "M % 128 == N % 128 == K % 128 == 0, and 16-byte-aligned bases");
  c10::cuda::CUDAGuard guard(a.device());
  Tensor c = at::empty({a.size(0), a.size(1), b.size(2)}, a.options());
  std::lock_guard<std::recursive_mutex> g(World::instance().mutex());
  launch_gemm_nn_batched(a.data_ptr(), b.data_ptr(), c.data_ptr(), a.size(0), a.size(1), b.size(2), a.size(2), sm_count(),
                         stream_of(a));
  return c;
}

// G_e = grad_scale * dy_e^T @ x_e -> [E, N, K], one launch.
Tensor batched_wgrad_bf16(const Tensor& dy, const Tensor& x, const c10::optional<Tensor>& grad_scale) {
  TORCH_CHECK(batched_wgrad_bf16_ok(dy, x),
              "mpi4torch_b200: batched_wgrad_bf16 needs contiguous bf16 dy [E, M, N] and x [E, M, K] on one CUDA device, "
              "N % 128 == K % 128 == M % 64 == 0, and 16-byte-aligned bases");
  c10::cuda::CUDAGuard guard(x.device());
  Tensor gw = at::empty({dy.size(0), dy.size(2), x.size(2)}, x.options());
  std::lock_guard<std::recursive_mutex> g(World::instance().mutex());
  launch_wgrad_bf16_batched(dy.data_ptr(), x.data_ptr(), gw.data_ptr(), dy.size(0), dy.size(1), dy.size(2), x.size(2),
                            sm_count(), stream_of(x), grad_scale_ptr(grad_scale, x));
  return gw;
}

// out[e, n] = grad_scale * sum_i partials[e, i, n] (fp32), in column_sum's fixed order, one launch.
Tensor batched_column_sum(const Tensor& partials, const c10::optional<Tensor>& grad_scale) {
  TORCH_CHECK(partials.is_cuda() && partials.dim() == 3 && partials.scalar_type() == at::kFloat &&
                  partials.is_contiguous() && partials.size(0) > 0 && partials.size(1) > 0,
              "mpi4torch_b200: batched_column_sum needs a non-empty contiguous 3-d fp32 CUDA tensor");
  c10::cuda::CUDAGuard guard(partials.device());
  Tensor out = at::empty({partials.size(0), partials.size(2)}, partials.options());
  if (out.numel() == 0) return out;
  launch_column_sum_batched(partials.data_ptr<float>(), partials.size(0), partials.size(1), partials.size(2),
                            out.data_ptr<float>(), grad_scale_ptr(grad_scale, partials), stream_of(partials));
  return out;
}

// ---- grouped experts (E experts with device-resident row counts, one launch per op) ------------------------------
// x [R, K] holds expert e's rows at row 128 * sum_{j<e} ceil(counts[j] / 128) (ops.expert_group_starts); counts [E] is
// contiguous int32 on x's device and is never read on the host.  Weights and biases are stacked as for the batched ops.
bool bf16_2d(const Tensor& t) {
  return t.is_cuda() && t.dim() == 2 && t.scalar_type() == at::kBFloat16 && t.is_contiguous();
}

// The kernels read the counts as int32 words: a 4-byte-aligned base.
bool counts_ok(const Tensor& counts, const Tensor& like) {
  return counts.is_cuda() && counts.device() == like.device() && counts.dim() == 1 && counts.scalar_type() == at::kInt &&
         counts.is_contiguous() && counts.numel() > 0 && (reinterpret_cast<uintptr_t>(counts.data_ptr()) & 3u) == 0;
}

// x [R, K] @ w [E, N, K]^T by groups, and the bias [E, N] (contiguous fp32, 8-byte aligned) when given.
bool grouped_gemm_tn_ok(const Tensor& x, const Tensor& w, const Tensor& counts, const c10::optional<Tensor>& bias) {
  if (!(bf16_2d(x) && bf16_3d(w) && same_device({&x, &w}) && counts_ok(counts, x) && counts.size(0) == w.size(0) &&
        x.size(1) == w.size(2)))
    return false;
  if (bias.has_value() && !(bias->is_cuda() && bias->device() == x.device() && bias->dim() == 2 &&
                            bias->scalar_type() == at::kFloat && bias->is_contiguous() && bias->size(0) == w.size(0) &&
                            bias->size(1) == w.size(1) && epilogue_bias_ok(bias->data_ptr<float>())))
    return false;
  return World::instance().cuda_ready() && grouped_gemm_supported(w.size(0), x.size(0), w.size(1), x.size(1), x.data_ptr(),
                                                                  w.data_ptr(), x.data_ptr(), counts.data_ptr());
}

// a [R, K] @ b [E, K, N] by groups.
bool grouped_gemm_nn_ok(const Tensor& a, const Tensor& b, const Tensor& counts) {
  if (!(bf16_2d(a) && bf16_3d(b) && same_device({&a, &b}) && counts_ok(counts, a) && counts.size(0) == b.size(0) &&
        a.size(1) == b.size(1)))
    return false;
  return World::instance().cuda_ready() && grouped_gemm_supported(b.size(0), a.size(0), b.size(2), a.size(1), a.data_ptr(),
                                                                  b.data_ptr(), a.data_ptr(), counts.data_ptr());
}

// dy [R, N]^T @ x [R, K] over each group's rows.
bool grouped_wgrad_bf16_ok(const Tensor& dy, const Tensor& x, const Tensor& counts) {
  if (!(bf16_2d(dy) && bf16_2d(x) && same_device({&dy, &x}) && counts_ok(counts, x) && dy.size(0) == x.size(0)))
    return false;
  return World::instance().cuda_ready() && wgrad_bf16_grouped_supported(counts.size(0), dy.size(0), dy.size(1), x.size(1),
                                                                        dy.data_ptr(), x.data_ptr(), x.data_ptr(),
                                                                        counts.data_ptr());
}

const char* kGroupedRules = " on one CUDA device with contiguous int32 counts [E], 1 <= E <= 1024, R % 128 == N % 128 == "
                            "K % 128 == 0, and aligned bases";

// (h, z) [R, N]: z = x_e @ w_e^T + b_e on group e's rows, h = gelu_tanh(z); other rows zero.  One launch.
std::tuple<Tensor, Tensor> grouped_linear_bias_gelu_forward(const Tensor& x, const Tensor& w, const Tensor& b,
                                                            const Tensor& counts) {
  TORCH_CHECK(grouped_gemm_tn_ok(x, w, counts, b),
              "mpi4torch_b200: grouped_linear_bias_gelu_forward needs contiguous bf16 x [R, K], w [E, N, K] and fp32 "
              "b [E, N]", kGroupedRules);
  c10::cuda::CUDAGuard guard(x.device());
  Tensor z = at::empty({x.size(0), w.size(1)}, x.options());
  Tensor h = at::empty_like(z);
  std::lock_guard<std::recursive_mutex> g(World::instance().mutex());
  launch_gemm_bias_gelu_grouped(x.data_ptr(), w.data_ptr(), b.data_ptr<float>(), z.data_ptr(), h.data_ptr(),
                                counts.data_ptr<int>(), w.size(0), x.size(0), w.size(1), x.size(1), sm_count(), stream_of(x));
  return {h, z};
}

// y [R, N] = bf16(x_e @ w_e^T + b_e) on group e's rows, other rows zero.  One launch.
Tensor grouped_linear_bias_forward(const Tensor& x, const Tensor& w, const Tensor& b, const Tensor& counts) {
  TORCH_CHECK(grouped_gemm_tn_ok(x, w, counts, b),
              "mpi4torch_b200: grouped_linear_bias_forward needs contiguous bf16 x [R, K], w [E, N, K] and fp32 b [E, N]",
              kGroupedRules);
  c10::cuda::CUDAGuard guard(x.device());
  Tensor y = at::empty({x.size(0), w.size(1)}, x.options());
  std::lock_guard<std::recursive_mutex> g(World::instance().mutex());
  launch_gemm_bias_grouped(x.data_ptr(), w.data_ptr(), b.data_ptr<float>(), y.data_ptr(), counts.data_ptr<int>(),
                           w.size(0), x.size(0), w.size(1), x.size(1), sm_count(), stream_of(x));
  return y;
}

// (dz [R, N], partials [R / 16, N]): dz = (dy_e @ w_e) * gelu_tanh'(z) on group e's rows (w [E, K, N] read in place),
// other rows zero; the partial rows of each group's ceil(count / 16) row blocks (reduce with grouped_column_sum).
std::tuple<Tensor, Tensor> grouped_gemm_nn_gelu_backward(const Tensor& dy, const Tensor& w, const Tensor& z,
                                                         const Tensor& counts) {
  TORCH_CHECK(grouped_gemm_nn_ok(dy, w, counts) && bf16_2d(z) && z.device() == dy.device() && z.size(0) == dy.size(0) &&
                  z.size(1) == w.size(2),
              "mpi4torch_b200: grouped_gemm_nn_gelu_backward needs contiguous bf16 dy [R, K], w [E, K, N] and z [R, N]",
              kGroupedRules);
  c10::cuda::CUDAGuard guard(dy.device());
  const int64_t R = dy.size(0), N = w.size(2);
  Tensor dz = at::empty({R, N}, dy.options());
  Tensor part = at::empty({colsum_rows(R), N}, dy.options().dtype(at::kFloat));
  std::lock_guard<std::recursive_mutex> g(World::instance().mutex());
  launch_gemm_nn_gelu_bwd_colsum_grouped(dy.data_ptr(), w.data_ptr(), z.data_ptr(), dz.data_ptr(), part.data_ptr<float>(),
                                         counts.data_ptr<int>(), w.size(0), R, N, dy.size(1), sm_count(), stream_of(dy));
  return {dz, part};
}

// c [R, N] = a_e @ b_e on group e's rows (b [E, K, N] read in place), other rows zero.  One launch.
Tensor grouped_gemm_nn(const Tensor& a, const Tensor& b, const Tensor& counts) {
  TORCH_CHECK(grouped_gemm_nn_ok(a, b, counts),
              "mpi4torch_b200: grouped_gemm_nn needs contiguous bf16 a [R, K] and b [E, K, N]", kGroupedRules);
  c10::cuda::CUDAGuard guard(a.device());
  Tensor c = at::empty({a.size(0), b.size(2)}, a.options());
  std::lock_guard<std::recursive_mutex> g(World::instance().mutex());
  launch_gemm_nn_grouped(a.data_ptr(), b.data_ptr(), c.data_ptr(), counts.data_ptr<int>(), b.size(0), a.size(0), b.size(2),
                         a.size(1), sm_count(), stream_of(a));
  return c;
}

// G [E, N, K]: G_e = grad_scale * dy_e^T @ x_e over group e's rows; zero for an empty group.  One launch.
Tensor grouped_wgrad_bf16(const Tensor& dy, const Tensor& x, const Tensor& counts, const c10::optional<Tensor>& grad_scale) {
  TORCH_CHECK(grouped_wgrad_bf16_ok(dy, x, counts),
              "mpi4torch_b200: grouped_wgrad_bf16 needs contiguous bf16 dy [R, N] and x [R, K]", kGroupedRules);
  c10::cuda::CUDAGuard guard(x.device());
  Tensor gw = at::empty({counts.size(0), dy.size(1), x.size(1)}, x.options());
  std::lock_guard<std::recursive_mutex> g(World::instance().mutex());
  launch_wgrad_bf16_grouped(dy.data_ptr(), x.data_ptr(), gw.data_ptr(), counts.data_ptr<int>(), counts.size(0), dy.size(0),
                            dy.size(1), x.size(1), sm_count(), stream_of(x), grad_scale_ptr(grad_scale, x));
  return gw;
}

// out [E, N] fp32: per group, the sum of its column-sum partial rows (partials [R / 16, N] fp32, R = rows of the
// grouped tensor) or, for a bf16 [R, N] input, of its valid rows.  Fixed order, no atomics.  One launch.
Tensor grouped_column_sum(const Tensor& in, const Tensor& counts) {
  const bool bf16_rows = in.scalar_type() == at::kBFloat16;
  const int64_t rows = in.dim() == 2 ? (bf16_rows ? 1 : 16) * in.size(0) : 0;  // R
  TORCH_CHECK(in.is_cuda() && in.dim() == 2 && in.is_contiguous() && (bf16_rows || in.scalar_type() == at::kFloat) &&
                  counts_ok(counts, in) && counts.size(0) <= 1024 && rows > 0 && rows % 128 == 0 && in.size(1) > 0,
              "mpi4torch_b200: grouped_column_sum needs bf16 rows [R, N] or fp32 partials [R / 16, N] (contiguous, "
              "R % 128 == 0) and contiguous int32 counts [E <= 1024] on the same CUDA device");
  c10::cuda::CUDAGuard guard(in.device());
  Tensor out = at::empty({counts.size(0), in.size(1)}, in.options().dtype(at::kFloat));
  launch_column_sum_grouped(in.data_ptr(), bf16_rows, counts.data_ptr<int>(), counts.size(0), rows, in.size(1),
                            out.data_ptr<float>(), stream_of(in));
  return out;
}

// ---- expert weight updates inside the expert wgrads (in-backward SGD, fp32 micro-batch accumulation) --------------
// The weight or buffer is written in place, tile by tile, by the one CTA that computes the tile, and the wgrad never
// reads it: the update is safe unless it shares memory with dy or x, which the predicates reject.
bool disjoint(const Tensor& a, const Tensor& b) {
  const auto* pa = static_cast<const char*>(a.data_ptr());
  const auto* pb = static_cast<const char*>(b.data_ptr());
  return pa + a.nbytes() <= pb || pb + b.nbytes() <= pa;
}

// `out` [E, N, K] contiguous, of dtype `dt`, on the operands' device, 16-byte aligned, disjoint from dy and x.
bool expert_out_ok(const Tensor& out, at::ScalarType dt, int64_t E, const Tensor& dy, const Tensor& x, int64_t N,
                   int64_t K) {
  return out.is_cuda() && out.device() == x.device() && out.dim() == 3 && out.scalar_type() == dt &&
         out.is_contiguous() && out.size(0) == E && out.size(1) == N && out.size(2) == K && (reinterpret_cast<uintptr_t>(out.data_ptr()) & 15u) == 0 &&
         disjoint(out, dy) && disjoint(out, x);
}

// w [E, N, K] bf16 (or buf fp32) updated from dy [E, M, N] and x [E, M, K].
bool batched_wgrad_update_ok(const Tensor& out, at::ScalarType dt, const Tensor& dy, const Tensor& x) {
  return batched_wgrad_bf16_ok(dy, x) && expert_out_ok(out, dt, dy.size(0), dy, x, dy.size(2), x.size(2));
}

bool batched_wgrad_sgd_ok(const Tensor& w, const Tensor& dy, const Tensor& x) {
  return batched_wgrad_update_ok(w, at::kBFloat16, dy, x);
}

bool batched_wgrad_accumulate_ok(const Tensor& buf, const Tensor& dy, const Tensor& x) {
  return batched_wgrad_update_ok(buf, at::kFloat, dy, x);
}

// w [E, N, K] bf16 (or buf fp32) updated from dy [R, N] and x [R, K] by groups of counts [E].
bool grouped_wgrad_update_ok(const Tensor& out, at::ScalarType dt, const Tensor& dy, const Tensor& x,
                             const Tensor& counts) {
  return grouped_wgrad_bf16_ok(dy, x, counts) && expert_out_ok(out, dt, counts.size(0), dy, x, dy.size(1), x.size(1)) &&
         disjoint(out, counts);
}

bool grouped_wgrad_sgd_ok(const Tensor& w, const Tensor& dy, const Tensor& x, const Tensor& counts) {
  return grouped_wgrad_update_ok(w, at::kBFloat16, dy, x, counts);
}

bool grouped_wgrad_accumulate_ok(const Tensor& buf, const Tensor& dy, const Tensor& x, const Tensor& counts) {
  return grouped_wgrad_update_ok(buf, at::kFloat, dy, x, counts);
}

const char* kUpdateRules = ", the batched_wgrad_bf16 (or grouped_wgrad_bf16) operand rules, and the updated tensor "
                           "contiguous and 16-byte aligned on the same device, sharing no memory with dy, x or counts";

// w_e <- bf16(w_e + scale * grad_scale * dy_e^T @ x_e): the SGD step of every expert as the batched wgrad's epilogue.
void batched_wgrad_sgd_(Tensor w, const Tensor& dy, const Tensor& x, double scale, const c10::optional<Tensor>& grad_scale) {
  TORCH_CHECK(batched_wgrad_sgd_ok(w, dy, x), "mpi4torch_b200: batched_wgrad_sgd_ needs bf16 w [E, N, K], dy [E, M, N] "
              "and x [E, M, K]", kUpdateRules);
  TORCH_CHECK(scale != 0.0, "mpi4torch_b200: batched_wgrad_sgd_ needs a non-zero scale");
  c10::cuda::CUDAGuard guard(x.device());
  std::lock_guard<std::recursive_mutex> g(World::instance().mutex());
  launch_wgrad_bf16_batched(dy.data_ptr(), x.data_ptr(), w.data_ptr(), dy.size(0), dy.size(1), dy.size(2), x.size(2),
                            sm_count(), stream_of(x), grad_scale_ptr(grad_scale, x), static_cast<float>(scale));
}

// buf_e <- fmaf(grad_scale, dy_e^T @ x_e, buf_e) in fp32, every expert in one launch.
void batched_wgrad_accumulate_(Tensor buf, const Tensor& dy, const Tensor& x, const c10::optional<Tensor>& grad_scale) {
  TORCH_CHECK(batched_wgrad_accumulate_ok(buf, dy, x), "mpi4torch_b200: batched_wgrad_accumulate_ needs fp32 buf "
              "[E, N, K], bf16 dy [E, M, N] and x [E, M, K]", kUpdateRules);
  c10::cuda::CUDAGuard guard(x.device());
  std::lock_guard<std::recursive_mutex> g(World::instance().mutex());
  launch_wgrad_accumulate_batched(dy.data_ptr(), x.data_ptr(), buf.data_ptr<float>(), dy.size(0), dy.size(1), dy.size(2),
                                  x.size(2), sm_count(), stream_of(x), grad_scale_ptr(grad_scale, x));
}

// w_e <- bf16(w_e + scale * grad_scale * G_e) over group e's rows; an empty group's w_e is not written.
void grouped_wgrad_sgd_(Tensor w, const Tensor& dy, const Tensor& x, const Tensor& counts, double scale,
                        const c10::optional<Tensor>& grad_scale) {
  TORCH_CHECK(grouped_wgrad_sgd_ok(w, dy, x, counts), "mpi4torch_b200: grouped_wgrad_sgd_ needs bf16 w [E, N, K], "
              "dy [R, N] and x [R, K], int32 counts [E]", kUpdateRules);
  TORCH_CHECK(scale != 0.0, "mpi4torch_b200: grouped_wgrad_sgd_ needs a non-zero scale");
  c10::cuda::CUDAGuard guard(x.device());
  std::lock_guard<std::recursive_mutex> g(World::instance().mutex());
  launch_wgrad_bf16_grouped(dy.data_ptr(), x.data_ptr(), w.data_ptr(), counts.data_ptr<int>(), counts.size(0), dy.size(0),
                            dy.size(1), x.size(1), sm_count(), stream_of(x), grad_scale_ptr(grad_scale, x),
                            static_cast<float>(scale));
}

// buf_e <- fmaf(grad_scale, G_e, buf_e) in fp32 over group e's rows; an empty group's buf_e is not written.
void grouped_wgrad_accumulate_(Tensor buf, const Tensor& dy, const Tensor& x, const Tensor& counts,
                               const c10::optional<Tensor>& grad_scale) {
  TORCH_CHECK(grouped_wgrad_accumulate_ok(buf, dy, x, counts), "mpi4torch_b200: grouped_wgrad_accumulate_ needs fp32 "
              "buf [E, N, K], bf16 dy [R, N] and x [R, K], int32 counts [E]", kUpdateRules);
  c10::cuda::CUDAGuard guard(x.device());
  std::lock_guard<std::recursive_mutex> g(World::instance().mutex());
  launch_wgrad_accumulate_grouped(dy.data_ptr(), x.data_ptr(), buf.data_ptr<float>(), counts.data_ptr<int>(),
                                  counts.size(0), dy.size(0), dy.size(1), x.size(1), sm_count(), stream_of(x),
                                  grad_scale_ptr(grad_scale, x));
}

// ---- FP8 linear layer (gemm_fp8.cu) ------------------------------------------------------------------------------
bool fp8_e5m2(c10::string_view fmt) {
  TORCH_CHECK(fmt == "e4m3" || fmt == "e5m2", "mpi4torch_b200: the fp8 format must be 'e4m3' or 'e5m2'");
  return fmt == "e5m2";
}

bool is_fp8(const Tensor& t) { return t.scalar_type() == at::kFloat8_e4m3fn || t.scalar_type() == at::kFloat8_e5m2; }

bool scalar_ok(const Tensor& s, const Tensor& like) {
  return s.is_cuda() && s.device() == like.device() && s.scalar_type() == at::kFloat && s.numel() == 1;
}

// (q, qt, scale_inv): q = fp8(x * s) [rows, cols] when rowwise, qt = its transpose [cols, rows] when transposed (each
// contiguous, or None), scale_inv = 1/s as a device fp32 [1].  s is the power of two of amax (DESIGN §4.4): of max|x|,
// computed here, or of a given device amax (fp32 [1]).
std::tuple<Tensor, Tensor, Tensor> quantize_fp8(const Tensor& x, c10::string_view fmt, bool rowwise, bool transposed,
                                                const c10::optional<Tensor>& amax) {
  const bool e5m2 = fp8_e5m2(fmt);
  TORCH_CHECK(x.is_cuda() && x.dim() == 2 && x.scalar_type() == at::kBFloat16 && x.stride(1) == 1 && x.numel() > 0,
              "mpi4torch_b200: quantize_fp8 needs a non-empty 2-d bf16 CUDA tensor with unit inner stride");
  TORCH_CHECK(rowwise || transposed, "mpi4torch_b200: quantize_fp8 needs rowwise or transposed");
  const bool given = amax.has_value() && amax->defined();
  TORCH_CHECK(!given || (scalar_ok(*amax, x) && amax->is_contiguous()),
              "mpi4torch_b200: amax must be a one-element fp32 tensor on x's device");
  c10::cuda::CUDAGuard guard(x.device());
  cudaStream_t stream = stream_of(x);
  const auto dt = e5m2 ? at::kFloat8_e5m2 : at::kFloat8_e4m3fn;
  const int64_t R = x.size(0), C = x.size(1);
  Tensor q = rowwise ? at::empty({R, C}, x.options().dtype(dt)) : Tensor();
  Tensor qt = transposed ? at::empty({C, R}, x.options().dtype(dt)) : Tensor();
  Tensor si = at::empty({1}, x.options().dtype(at::kFloat));
  std::lock_guard<std::recursive_mutex> g(World::instance().mutex());
  Tensor am = given ? *amax : at::zeros({1}, x.options().dtype(at::kFloat));
  auto* bits = reinterpret_cast<unsigned int*>(am.data_ptr<float>());
  if (!given) launch_quantize_fp8_amax(x.data_ptr(), R, C, x.stride(0), bits, sm_count(), stream);
  launch_quantize_fp8_cast(x.data_ptr(), R, C, x.stride(0), e5m2, bits, rowwise ? q.data_ptr() : nullptr,
                           transposed ? qt.data_ptr() : nullptr, si.data_ptr<float>(), stream);
  return {q, qt, si};
}

// The operand rules of the fp8 GEMMs: a [M, K] fp8 (E4M3 or E5M2), b [N, K] E4M3, unit inner strides, K, the row
// strides and the bases 16-byte aligned, N % 8 == 0, both scale_inv one-element fp32 on the same device; and the MSE
// target [M, N] (bf16 pairs) or the SGD weight [M, N] (bf16, 16-byte-aligned, row stride % 8) when given.
bool gemm_fp8_tn_ok(const Tensor& a, const Tensor& b, const Tensor& a_si, const Tensor& b_si,
                    const c10::optional<Tensor>& target, const c10::optional<Tensor>& w) {
  if (!(a.is_cuda() && b.is_cuda() && a.device() == b.device() && a.dim() == 2 && b.dim() == 2 && is_fp8(a) &&
        b.scalar_type() == at::kFloat8_e4m3fn && a.stride(1) == 1 && b.stride(1) == 1 && a.size(1) == b.size(1) &&
        scalar_ok(a_si, a) && scalar_ok(b_si, a)))
    return false;
  if (target.has_value() && target->defined() &&
      !(target->device() == a.device() && mse_target_ok(*target, a.size(0), b.size(0))))
    return false;
  const void* c = a.data_ptr();
  int64_t ldc = b.size(0);
  if (w.has_value() && w->defined()) {
    if (!(w->is_cuda() && w->device() == a.device() && w->dim() == 2 && w->scalar_type() == at::kBFloat16 &&
          w->stride(1) == 1 && w->size(0) == a.size(0) && w->size(1) == b.size(0)))
      return false;
    c = w->data_ptr();
    ldc = w->stride(0);
  }
  return World::instance().cuda_ready() &&
         gemm_fp8_tn_supported(a.size(0), b.size(0), a.size(1), a.data_ptr(), b.data_ptr(), c, a.stride(0), b.stride(0),
                               ldc);
}

// C = bf16(grad_scale * a @ b^T * a_scale_inv * b_scale_inv).
Tensor gemm_fp8_tn(const Tensor& a, const Tensor& b, const Tensor& a_si, const Tensor& b_si,
                   const c10::optional<Tensor>& grad_scale) {
  TORCH_CHECK(gemm_fp8_tn_ok(a, b, a_si, b_si, c10::nullopt, c10::nullopt),
              "mpi4torch_b200: gemm_fp8_tn needs a [M, K] fp8 and b [N, K] float8_e4m3fn CUDA tensors with unit inner "
              "strides, K and the row strides multiples of 16, 16-byte-aligned bases, N % 8 == 0, and one-element fp32 "
              "scale_inv tensors on the same device");
  c10::cuda::CUDAGuard guard(a.device());
  Tensor c = at::empty({a.size(0), b.size(0)}, a.options().dtype(at::kBFloat16));
  std::lock_guard<std::recursive_mutex> g(World::instance().mutex());
  launch_gemm_fp8_tn(a.data_ptr(), a.scalar_type() == at::kFloat8_e5m2, b.data_ptr(), c.data_ptr(), a.size(0), b.size(0),
                     a.size(1), a.stride(0), b.stride(0), c.stride(0), a_si.data_ptr<float>(), b_si.data_ptr<float>(),
                     grad_scale_ptr(grad_scale, a), sm_count(), stream_of(a));
  return c;
}

// Forward of the fp8 linear layer with the MSE epilogue, against an already averaged weight: (dy, loss[1], dy_amax[1])
// with y = xq @ wq^T / (s_x s_w), dy = bf16(grad_scale (y - target)), loss = loss_scale * sum((y - target)^2) and
// dy_amax = max |dy| over the stored bf16 values (fp32), ready for quantize_fp8(dy, "e5m2", amax=dy_amax).
std::tuple<Tensor, Tensor, Tensor> linear_mse_forward_fp8_local(const Tensor& xq, const Tensor& wq, const Tensor& x_si,
                                                                const Tensor& w_si, const Tensor& target,
                                                                double loss_scale, double grad_scale) {
  TORCH_CHECK(xq.scalar_type() == at::kFloat8_e4m3fn && gemm_fp8_tn_ok(xq, wq, x_si, w_si, target, c10::nullopt),
              "mpi4torch_b200: linear_mse_forward_fp8_local needs float8_e4m3fn xq [B, K] and wq [N, K] under the "
              "gemm_fp8_tn operand rules, and a bf16 target [B, N] with unit inner stride, a 4-byte-aligned base and an "
              "even row stride");
  c10::cuda::CUDAGuard guard(xq.device());
  Tensor dy = at::empty({xq.size(0), wq.size(0)}, xq.options().dtype(at::kBFloat16));
  Tensor loss = at::zeros({1}, xq.options().dtype(at::kFloat));
  Tensor amax = at::zeros({1}, xq.options().dtype(at::kFloat));
  const MseEpilogue mse = mse_epilogue(target, loss, loss_scale, grad_scale);
  std::lock_guard<std::recursive_mutex> g(World::instance().mutex());
  launch_gemm_fp8_mse(xq.data_ptr(), wq.data_ptr(), dy.data_ptr(), xq.size(0), wq.size(0), xq.size(1), xq.stride(0),
                      wq.stride(0), dy.stride(0), x_si.data_ptr<float>(), w_si.data_ptr<float>(), mse,
                      reinterpret_cast<unsigned int*>(amax.data_ptr<float>()), sm_count(), stream_of(xq));
  return {dy, loss, amax};
}

// w += scale * grad_scale * a @ b^T * a_scale_inv * b_scale_inv, the single-rank SGD step as the fp8 GEMM's epilogue.
void gemm_fp8_tn_sgd_(Tensor w, const Tensor& a, const Tensor& b, const Tensor& a_si, const Tensor& b_si, double scale,
                      const c10::optional<Tensor>& grad_scale) {
  TORCH_CHECK(gemm_fp8_tn_ok(a, b, a_si, b_si, c10::nullopt, w),
              "mpi4torch_b200: gemm_fp8_tn_sgd_ needs the gemm_fp8_tn operand rules and w a bf16 [M, N] CUDA tensor with "
              "unit inner stride, a 16-byte-aligned base and a row stride that is a multiple of 8");
  TORCH_CHECK(scale != 0.0, "mpi4torch_b200: gemm_fp8_tn_sgd_ needs a non-zero scale");
  c10::cuda::CUDAGuard guard(a.device());
  std::lock_guard<std::recursive_mutex> g(World::instance().mutex());
  launch_gemm_fp8_sgd(a.data_ptr(), a.scalar_type() == at::kFloat8_e5m2, b.data_ptr(), w.data_ptr(), a.size(0), b.size(0),
                      a.size(1), a.stride(0), b.stride(0), w.stride(0), a_si.data_ptr<float>(), b_si.data_ptr<float>(),
                      static_cast<float>(scale), grad_scale_ptr(grad_scale, a), sm_count(), stream_of(a));
}

}  // namespace

TORCH_LIBRARY_FRAGMENT(mpi4torch_b200, m) {
  m.def("quantize_fp8(Tensor x, str fmt, bool rowwise, bool transposed, Tensor? amax=None) -> (Tensor, Tensor, Tensor)",
        &quantize_fp8);
  m.def("gemm_fp8_tn_supported(Tensor a, Tensor b, Tensor a_scale_inv, Tensor b_scale_inv, Tensor? target=None, "
        "Tensor? w=None) -> bool",
        &gemm_fp8_tn_ok);
  m.def("gemm_fp8_tn(Tensor a, Tensor b, Tensor a_scale_inv, Tensor b_scale_inv, Tensor? grad_scale=None) -> Tensor",
        &gemm_fp8_tn);
  m.def("linear_mse_forward_fp8_local(Tensor xq, Tensor wq, Tensor x_scale_inv, Tensor w_scale_inv, Tensor target, "
        "float loss_scale, float grad_scale) -> (Tensor, Tensor, Tensor)",
        &linear_mse_forward_fp8_local);
  m.def("gemm_fp8_tn_sgd_(Tensor(a!) w, Tensor a, Tensor b, Tensor a_scale_inv, Tensor b_scale_inv, float scale, "
        "Tensor? grad_scale=None) -> ()",
        &gemm_fp8_tn_sgd_);
  m.def("batched_gemm_tn_supported(Tensor x, Tensor w, Tensor? bias=None) -> bool", &batched_gemm_tn_ok);
  m.def("batched_gemm_nn_supported(Tensor a, Tensor b) -> bool", &batched_gemm_nn_ok);
  m.def("batched_wgrad_bf16_supported(Tensor dy, Tensor x) -> bool", &batched_wgrad_bf16_ok);
  m.def("batched_linear_bias_gelu_forward(Tensor x, Tensor w, Tensor b) -> (Tensor, Tensor)",
        &batched_linear_bias_gelu_forward);
  m.def("batched_linear_bias_forward(Tensor x, Tensor w, Tensor b) -> Tensor", &batched_linear_bias_forward);
  m.def("batched_gemm_nn_gelu_backward(Tensor dy, Tensor w, Tensor z, Tensor? grad_scale=None) -> (Tensor, Tensor)",
        &batched_gemm_nn_gelu_backward);
  m.def("batched_gemm_nn(Tensor a, Tensor b) -> Tensor", &batched_gemm_nn);
  m.def("batched_wgrad_bf16(Tensor dy, Tensor x, Tensor? grad_scale=None) -> Tensor", &batched_wgrad_bf16);
  m.def("batched_column_sum(Tensor partials, Tensor? grad_scale=None) -> Tensor", &batched_column_sum);
  m.def("grouped_gemm_tn_supported(Tensor x, Tensor w, Tensor counts, Tensor? bias=None) -> bool", &grouped_gemm_tn_ok);
  m.def("grouped_gemm_nn_supported(Tensor a, Tensor b, Tensor counts) -> bool", &grouped_gemm_nn_ok);
  m.def("grouped_wgrad_bf16_supported(Tensor dy, Tensor x, Tensor counts) -> bool", &grouped_wgrad_bf16_ok);
  m.def("grouped_linear_bias_gelu_forward(Tensor x, Tensor w, Tensor b, Tensor counts) -> (Tensor, Tensor)",
        &grouped_linear_bias_gelu_forward);
  m.def("grouped_linear_bias_forward(Tensor x, Tensor w, Tensor b, Tensor counts) -> Tensor", &grouped_linear_bias_forward);
  m.def("grouped_gemm_nn_gelu_backward(Tensor dy, Tensor w, Tensor z, Tensor counts) -> (Tensor, Tensor)",
        &grouped_gemm_nn_gelu_backward);
  m.def("grouped_gemm_nn(Tensor a, Tensor b, Tensor counts) -> Tensor", &grouped_gemm_nn);
  m.def("grouped_wgrad_bf16(Tensor dy, Tensor x, Tensor counts, Tensor? grad_scale=None) -> Tensor", &grouped_wgrad_bf16);
  m.def("grouped_column_sum(Tensor partials, Tensor counts) -> Tensor", &grouped_column_sum);
  m.def("batched_wgrad_sgd_supported(Tensor w, Tensor dy, Tensor x) -> bool", &batched_wgrad_sgd_ok);
  m.def("batched_wgrad_accumulate_supported(Tensor buf, Tensor dy, Tensor x) -> bool", &batched_wgrad_accumulate_ok);
  m.def("grouped_wgrad_sgd_supported(Tensor w, Tensor dy, Tensor x, Tensor counts) -> bool", &grouped_wgrad_sgd_ok);
  m.def("grouped_wgrad_accumulate_supported(Tensor buf, Tensor dy, Tensor x, Tensor counts) -> bool",
        &grouped_wgrad_accumulate_ok);
  m.def("batched_wgrad_sgd_(Tensor(a!) w, Tensor dy, Tensor x, float scale, Tensor? grad_scale=None) -> ()",
        &batched_wgrad_sgd_);
  m.def("batched_wgrad_accumulate_(Tensor(a!) buf, Tensor dy, Tensor x, Tensor? grad_scale=None) -> ()",
        &batched_wgrad_accumulate_);
  m.def("grouped_wgrad_sgd_(Tensor(a!) w, Tensor dy, Tensor x, Tensor counts, float scale, Tensor? grad_scale=None) -> ()",
        &grouped_wgrad_sgd_);
  m.def("grouped_wgrad_accumulate_(Tensor(a!) buf, Tensor dy, Tensor x, Tensor counts, Tensor? grad_scale=None) -> ()",
        &grouped_wgrad_accumulate_);
  m.def("linear_bias_gelu_forward(Tensor x, Tensor w, Tensor b) -> (Tensor, Tensor)", &linear_bias_gelu_forward);
  m.def("linear_bias_mse_forward_local(Tensor x, Tensor w, Tensor b, Tensor target, float loss_scale, float grad_scale) "
        "-> (Tensor, Tensor, Tensor)",
        &linear_bias_mse_forward_local);
  m.def("linear_bias_xent_forward_local(Tensor x, Tensor w, Tensor b, Tensor labels, float loss_scale, float grad_scale, "
        "int ignore_index=-100) -> (Tensor, Tensor, Tensor)",
        &linear_bias_xent_forward_local);
  m.def("gemm_nn_gelu_backward(Tensor dy, Tensor w, Tensor z, Tensor? grad_scale=None) -> (Tensor, Tensor)",
        &gemm_nn_gelu_backward);
  m.def("column_sum(Tensor partials, Tensor? grad_scale=None) -> Tensor", &column_sum);
  m.def("wgrad_allreduce_sgd_prefetch_(Tensor(a!) w, Tensor dy, Tensor x, float scale, Tensor? grad_scale=None) -> Tensor",
        &wgrad_allreduce_sgd_prefetch_);
  m.def("wgrad_sgd_(Tensor(a!) w, Tensor dy, Tensor x, float scale, Tensor? grad_scale=None) -> ()", &wgrad_sgd_);
  m.def("linear_mse_forward_local(Tensor x, Tensor w_avg, Tensor target, float loss_scale, float grad_scale) -> (Tensor, Tensor)",
        &linear_mse_forward_local);
  m.def("wgrad_bf16(Tensor dy, Tensor x, Tensor? grad_scale=None) -> Tensor", &wgrad_bf16);
  m.def("wgrad_bf16_supported(Tensor dy, Tensor x) -> bool", &wgrad_bf16_ok);
  m.def("wgrad_accumulate_(Tensor(a!) acc, Tensor dy, Tensor x, Tensor? grad_scale=None) -> ()", &wgrad_accumulate_);
  m.def("wgrad_accumulate_supported(Tensor acc, Tensor dy, Tensor x) -> bool", &wgrad_accumulate_ok);
  m.def("wgrad_allreduce_sgd_supported(Tensor w, Tensor dy, Tensor x) -> bool", &wgrad_allreduce_sgd_supported);
  m.def("wgrad_allreduce_sgd_(Tensor(a!) w, Tensor dy, Tensor x, float scale, Tensor? grad_scale=None) -> ()",
        &wgrad_allreduce_sgd_);
  m.def("linear_mse_forward(Tensor x, Tensor w, Tensor target, float scale, float loss_scale, float grad_scale, "
        "bool allow_fused) -> (Tensor, Tensor, Tensor)",
        &linear_mse_forward);
  m.def("allreduce_axpy_(Tensor(a!) param, Tensor grad, float scale, int max_blocks=0) -> ()", &allreduce_axpy_);
  m.def("symmetric_empty(int[] shape, ScalarType dtype) -> Tensor", &symmetric_empty);
  m.def("gemm_bf16_tn(Tensor x, Tensor w) -> Tensor", &gemm_bf16_tn);
  m.def("gemm_bf16_nn(Tensor a, Tensor b) -> Tensor", &gemm_bf16_nn);
  m.def("gemm_bf16_nn_supported(Tensor a, Tensor b) -> bool", &gemm_bf16_nn_ok);
  m.def("gemm_bf16_tn_supported(Tensor x, Tensor w, Tensor? target=None, Tensor? bias=None) -> bool", &gemm_bf16_tn_ok);
  m.def("allreduce_linear_supported(Tensor x, Tensor w) -> bool", &allreduce_linear_supported);
  m.def("allreduce_linear_fused(Tensor x, Tensor w, float scale) -> (Tensor, Tensor)", &allreduce_linear_fused);
}

}  // namespace m4t
