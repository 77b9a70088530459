// Virtual ranks: P ranks of the multi-GPU collective kernels simulated on ONE device, for tests.
//
// The unicast forms of the all-reduce kernels (allreduce.cu) and of the fused wgrad -> reduce-scatter -> SGD kernel
// (wgrad_wgmma.cu, peer-store mode) only see their peers through plain device pointers: heap[p] and sync.pads[p].
// So P ranks can be P launches of the unchanged launchers in one process, each with its own zeroed heap, counters
// and done word, on its own stream.  The NVLS / multicast paths need an NVSwitch and are not reachable here
// (mc_heap = nullptr).  The process's World and symmetric heap are not touched.
//
// Residency: the rank kernels spin on each other's flags, so every rank's whole grid must be resident at once.
// Each rank gets sm_count = (SMs / P) & ~1 and at most that many CTAs; a CTA of any of these kernels fits on one SM
// (the 1024-thread pipelined all-reduce and the persistent wgrad kernel take one SM each), so the P grids fit.
// Module loading: the calls are launched one after the other, all ranks of a call back to back.  Under lazy module
// loading the first launch of a kernel may wait for the device to drain; in this order it only ever waits for earlier
// calls whose ranks have all been launched, never for a rank that has not been launched yet.  (Bringing up COMM_WORLD
// asks for CUDA_MODULE_LOADING=EAGER as well.)
#include <c10/cuda/CUDAGuard.h>
#include <c10/cuda/CUDAStream.h>
#include <ATen/cuda/CUDAContext.h>
#include <ATen/cuda/CUDAEvent.h>
#include <torch/extension.h>

#include <cstring>
#include <optional>
#include <string>
#include <vector>

#include "../kernels/kernels.h"

namespace m4t {

namespace {

constexpr int kMinRanks = 2;
constexpr int kMaxRanks = 8;
// Barrier pads of every rank: pad A at offset 0 (kMaxChannels x kMaxGpuPeers u32 = 32 KiB), pad B of the pipelined
// all-reduce at +64 KiB.
constexpr int64_t kPadRegionBytes = 128 << 10;
constexpr int64_t kHalfBytes = 16 << 20;  // staging half of the all-reduce kernels (two of them, by op parity)
constexpr unsigned long long kTimeoutNs = 5ull * 1000000000ull;

int64_t round_up(int64_t v, int64_t a) { return (v + a - 1) / a * a; }

DType dtype_of(const at::Tensor& t) {
  switch (t.scalar_type()) {
    case at::kByte: return DType::U8;
    case at::kChar: return DType::I8;
    case at::kShort: return DType::I16;
    case at::kInt: return DType::I32;
    case at::kLong: return DType::I64;
    case at::kFloat: return DType::F32;
    case at::kDouble: return DType::F64;
    case at::kBFloat16: return DType::BF16;
    case at::kHalf: return DType::F16;
    case at::kBool: return DType::BOOL;
    default: break;
  }
  M4T_CHECK(false, "virtual ranks: unsupported dtype " << c10::toString(t.scalar_type()));
  return DType::U8;
}

// One host-mapped error word shared by all virtual ranks (as every real rank has one).
int* error_word(int** dev) {
  static int* host = nullptr;
  static int* device = nullptr;
  if (!host) {
    C10_CUDA_CHECK(cudaHostAlloc(reinterpret_cast<void**>(&host), sizeof(int), cudaHostAllocMapped));
    C10_CUDA_CHECK(cudaHostGetDevicePointer(reinterpret_cast<void**>(&device), host, 0));
  }
  *dev = device;
  return host;
}

// P zeroed heaps of `heap_bytes`, per-rank counters / done words, the shared error word and one stream per rank.
struct VirtualRanks {
  int P;
  c10::Device device;
  std::vector<at::Tensor> heaps;
  at::Tensor words;  // per rank: counters[2] (u64) at 32 * p, done_ctr (u32) at 32 * p + 16
  std::vector<DeviceComm> dc;
  std::vector<c10::cuda::CUDAStream> streams;
  int* h_err = nullptr;

  VirtualRanks(int P_, c10::Device dev, int64_t heap_bytes, int64_t stage_off, int64_t half_bytes)
      : P(P_), device(dev) {
    M4T_CHECK(P >= kMinRanks && P <= kMaxRanks, "virtual ranks: P must be in [" << kMinRanks << ", " << kMaxRanks
                                                                                << "], got " << P);
    M4T_CHECK(dev.is_cuda(), "virtual ranks: tensors must be CUDA tensors");
    const auto opts = at::TensorOptions().dtype(at::kByte).device(dev);
    for (int p = 0; p < P; ++p) heaps.push_back(at::zeros({heap_bytes}, opts));
    words = at::zeros({32 * P}, opts);
    int* d_err = nullptr;
    h_err = error_word(&d_err);
    *reinterpret_cast<volatile int*>(h_err) = 0;
    const int sms = at::cuda::getDeviceProperties(dev.index())->multiProcessorCount;
    dc.resize(P);
    for (int r = 0; r < P; ++r) {
      DeviceComm& d = dc[r];
      std::memset(&d, 0, sizeof(d));
      for (int p = 0; p < P; ++p) {
        d.heap[p] = static_cast<char*>(heaps[p].data_ptr());
        d.sync.pads[p] = reinterpret_cast<uint32_t*>(heaps[p].data_ptr());
      }
      d.mc_heap = nullptr;
      char* w = static_cast<char*>(words.data_ptr()) + 32 * r;
      d.sync.counters = reinterpret_cast<unsigned long long*>(w);
      d.sync.done_ctr = reinterpret_cast<unsigned int*>(w + 16);
      d.sync.err_flag = d_err;
      d.sync.timeout_ns = kTimeoutNs;
      d.sync.rank = r;
      d.sync.size = P;
      d.stage_off = stage_off;
      d.half_bytes = half_bytes;
      d.sm_count = (sms / P) & ~1;
    }
    // the heaps are zeroed on the current stream; every rank stream starts after that
    at::cuda::CUDAEvent ready;
    ready.record(c10::cuda::getCurrentCUDAStream(dev.index()));
    for (int p = 0; p < P; ++p) {
      streams.push_back(c10::cuda::getStreamFromPool(false, dev.index()));
      ready.block(streams.back());
    }
  }

  int sm_count() const { return dc[0].sm_count; }
  char* heap(int p) const { return static_cast<char*>(heaps[p].data_ptr()); }

  // Waits for every rank, then reports a device-side timeout.
  void finish() {
    for (auto& s : streams) C10_CUDA_CHECK(cudaStreamSynchronize(s.stream()));
    const int err = *reinterpret_cast<volatile int*>(h_err);
    *reinterpret_cast<volatile int*>(h_err) = 0;
    M4T_CHECK(err == 0, "virtual ranks: a device-side wait timed out (code " << err << ")");
  }
};

void check_rank_list(const std::vector<at::Tensor>& ts, int P, const char* what) {
  M4T_CHECK(static_cast<int>(ts.size()) == P, "virtual ranks: " << what << " has " << ts.size() << " tensors for "
                                                                  << P << " ranks");
  for (const auto& t : ts) {
    M4T_CHECK(t.is_cuda() && t.device() == ts[0].device(), "virtual ranks: " << what << " must be on one CUDA device");
    M4T_CHECK(t.is_contiguous(), "virtual ranks: " << what << " must be contiguous (a view at any offset is fine)");
    M4T_CHECK(t.scalar_type() == ts[0].scalar_type() && t.numel() == ts[0].numel(),
              "virtual ranks: " << what << " must have one dtype and size on every rank");
  }
}

// Call c reduces ins[c][p] over the ranks p into outs[c][p] with the epilogue (scales[c], accs[c][p]); an empty
// accs[c] means no accumulate operand, and accs[c][p] may be outs[c][p] (in place).  All calls of all ranks are
// launched back to back with no host synchronisation, so consecutive calls exercise the staging parity and the
// device-resident flag counters.
void vr_allreduce(const std::vector<std::vector<at::Tensor>>& ins, const std::vector<std::vector<at::Tensor>>& outs,
                  int64_t op, const std::string& algo, int64_t blocks, int64_t chunk_bytes,
                  const std::vector<std::optional<double>>& scales, const std::vector<std::vector<at::Tensor>>& accs) {
  M4T_CHECK(!ins.empty() && outs.size() == ins.size() && scales.size() == ins.size() && accs.size() == ins.size(),
            "virtual ranks: ins, outs, scales and accs need one entry per call");
  M4T_CHECK(algo == "oneshot" || algo == "twoshot", "virtual ranks: algo must be 'oneshot' or 'twoshot'");
  const ArAlgo a = algo == "oneshot" ? ArAlgo::ONESHOT : ArAlgo::TWOSHOT;
  M4T_CHECK(op >= 0 && op < static_cast<int64_t>(ReduceOp::kCount), "virtual ranks: unknown op " << op);
  const int P = static_cast<int>(ins[0].size());
  M4T_CHECK(P >= kMinRanks && P <= kMaxRanks, "virtual ranks: P must be in [2, 8], got " << P);
  for (size_t c = 0; c < ins.size(); ++c) {
    check_rank_list(ins[c], P, "ins");
    check_rank_list(outs[c], P, "outs");
    M4T_CHECK(ins[c][0].numel() > 0 && outs[c][0].numel() == ins[c][0].numel() &&
                  outs[c][0].scalar_type() == ins[c][0].scalar_type() && outs[c][0].device() == ins[0][0].device() &&
                  ins[c][0].device() == ins[0][0].device(),
              "virtual ranks: call " << c << " needs non-empty inputs and outputs of one dtype, size and device");
    if (!accs[c].empty()) {
      check_rank_list(accs[c], P, "accs");
      M4T_CHECK(accs[c][0].numel() == ins[c][0].numel() && accs[c][0].scalar_type() == ins[c][0].scalar_type() &&
                    accs[c][0].device() == ins[0][0].device(),
                "virtual ranks: the accumulate operand of call " << c << " must match the output");
    }
  }
  const c10::Device dev = ins[0][0].device();
  c10::cuda::CUDAGuard guard(dev);
  VirtualRanks vr(P, dev, kPadRegionBytes + 2 * kHalfBytes, kPadRegionBytes, kHalfBytes);
  M4T_CHECK(blocks >= 1 && blocks <= vr.sm_count(),
            "virtual ranks: blocks must be in [1, " << vr.sm_count() << "] so that all " << P << " grids are resident");
  for (size_t c = 0; c < ins.size(); ++c) {
    const DType dt = dtype_of(ins[c][0]);
    Epilogue epi;
    if (scales[c]) {
      epi.has_scale = true;
      epi.scale = *scales[c];
    }
    for (int p = 0; p < P; ++p) {
      epi.accumulate = accs[c].empty() ? nullptr : accs[c][p].data_ptr();
      launch_allreduce(vr.dc[p], ins[c][p].data_ptr(), outs[c][p].data_ptr(), ins[c][p].numel(), dt,
                       static_cast<ReduceOp>(op), epi, a, static_cast<int>(blocks), chunk_bytes, vr.streams[p].stream());
    }
  }
  vr.finish();
}

// Peer-store mode of the fused wgrad -> reduce-scatter -> SGD kernel at P = 2 or 3.  weights[p] (bf16 [N, K]) is
// copied into rank p's heap; call c then runs W <- W + scale * sum_p gscale * dys[c][p]^T xs[c][p] on every rank.
// Returns every rank's final weights, the W_avg of the last call (prefetch), the device epoch words and the tile
// counters, all as fresh tensors.
py::dict vr_fused_wgrad_sgd(const std::vector<at::Tensor>& weights, const std::vector<std::vector<at::Tensor>>& dys,
                            const std::vector<std::vector<at::Tensor>>& xs, double scale,
                            const std::optional<at::Tensor>& gscale, int64_t ksplit, bool prefetch) {
  const int P = static_cast<int>(weights.size());
  M4T_CHECK(P >= 2 && P <= fused_wgrad_max_unicast_ranks(),
            "virtual ranks: the peer-store fused wgrad runs at 2 to " << fused_wgrad_max_unicast_ranks() << " ranks");
  check_rank_list(weights, P, "weights");
  M4T_CHECK(weights[0].dim() == 2 && weights[0].scalar_type() == at::kBFloat16, "virtual ranks: weights are bf16 [N, K]");
  const int64_t N = weights[0].size(0), K = weights[0].size(1);
  M4T_CHECK(!dys.empty() && xs.size() == dys.size(), "virtual ranks: dys and xs need one entry per call");
  for (size_t c = 0; c < dys.size(); ++c) {
    check_rank_list(dys[c], P, "dys");
    check_rank_list(xs[c], P, "xs");
    M4T_CHECK(dys[c][0].dim() == 2 && xs[c][0].dim() == 2 && dys[c][0].size(1) == N && xs[c][0].size(1) == K &&
                  dys[c][0].size(0) == dys[0][0].size(0) && xs[c][0].size(0) == dys[0][0].size(0),
              "virtual ranks: call " << c << " needs dy [Mb, N] and x [Mb, K] with the Mb of call 0");
  }
  if (gscale) {
    M4T_CHECK(gscale->is_cuda() && gscale->numel() == 1 && gscale->scalar_type() == at::kFloat,
              "virtual ranks: gscale is an fp32 device scalar");
  }
  const int64_t Mb = dys[0][0].size(0);
  const int64_t wbytes = N * K * 2;
  // heap layout: pads | W | W_avg | staging [P sources][ksplit][N, K] | tile counters | done | epoch
  const int64_t w_off = kPadRegionBytes;
  const int64_t wavg_off = round_up(w_off + wbytes, 256);
  const int64_t stage_off = round_up(wavg_off + wbytes, 256);
  const int64_t src_stride = ksplit * wbytes;
  const int64_t cnt_off = round_up(stage_off + P * src_stride, 256);
  const int64_t done_off = round_up(cnt_off + fused_wgrad_tiles(N, K) * 4, 256);
  const int64_t epoch_off = done_off + 16;
  const c10::Device dev = weights[0].device();
  c10::cuda::CUDAGuard guard(dev);
  VirtualRanks vr(P, dev, epoch_off + 16, 0, 0);
  for (int p = 0; p < P; ++p)
    C10_CUDA_CHECK(cudaMemcpyAsync(vr.heap(p) + w_off, weights[p].data_ptr(), wbytes, cudaMemcpyDeviceToDevice,
                                   vr.streams[p].stream()));
  const uint32_t tile_target = static_cast<uint32_t>(fused_wgrad_signals_per_unit() * P);
  const uint32_t done_target = static_cast<uint32_t>(P * fused_gemm_grid(vr.dc[0]));
  const float* gs = gscale ? gscale->data_ptr<float>() : nullptr;
  for (size_t c = 0; c < dys.size(); ++c)
    for (int p = 0; p < P; ++p)
      launch_fused_wgrad_update(vr.dc[p], dys[c][p].data_ptr(), xs[c][p].data_ptr(), Mb, N, K, dys[c][p].stride(0),
                                xs[c][p].stride(0), w_off, stage_off, wbytes, cnt_off, done_off, static_cast<int>(ksplit),
                                tile_target, done_target, static_cast<float>(scale), prefetch ? wavg_off : -1,
                                vr.streams[p].stream(), epoch_off, gs, /*use_multicast=*/false, src_stride);
  vr.finish();
  py::list w_out, wavg_out, epochs, counters;
  for (int p = 0; p < P; ++p) {
    const at::Tensor h = vr.heaps[p];
    w_out.append(h.narrow(0, w_off, wbytes).view(at::kBFloat16).view({N, K}).clone());
    if (prefetch) wavg_out.append(h.narrow(0, wavg_off, wbytes).view(at::kBFloat16).view({N, K}).clone());
    epochs.append(h.narrow(0, epoch_off, 4).view(at::kInt).item<int>());
    counters.append(h.narrow(0, cnt_off, fused_wgrad_tiles(N, K) * 4).view(at::kInt).clone());
  }
  py::dict out;
  out["weights"] = w_out;
  out["wavg"] = prefetch ? py::object(wavg_out) : py::none();
  out["epochs"] = epochs;
  out["counters"] = counters;
  out["grid"] = fused_gemm_grid(vr.dc[0]);
  return out;
}

}  // namespace

void register_virtual_ranks(py::module& m) {
  m.def("vr_allreduce", &vr_allreduce, py::arg("ins"), py::arg("outs"), py::arg("op"), py::arg("algo"),
        py::arg("blocks"), py::arg("chunk_bytes"), py::arg("scales"), py::arg("accs"),
        "Test entry: the unicast all-reduce kernels at P virtual ranks on one device (ins[call][rank]).");
  m.def("vr_fused_wgrad_sgd", &vr_fused_wgrad_sgd, py::arg("weights"), py::arg("dys"), py::arg("xs"), py::arg("scale"),
        py::arg("gscale"), py::arg("ksplit"), py::arg("prefetch"),
        "Test entry: the peer-store fused wgrad -> reduce-scatter -> SGD kernel at P virtual ranks on one device.");
  m.def("vr_sm_count", [](int64_t P) {
    const int sms = at::cuda::getCurrentDeviceProperties()->multiProcessorCount;
    return (sms / static_cast<int>(P)) & ~1;
  }, "SMs per virtual rank at P ranks: the largest grid a rank may launch.");
}

}  // namespace m4t
