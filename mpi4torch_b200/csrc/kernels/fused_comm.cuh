// Communication role of the fused Allreduce->GEMM kernels: all-reduce the weight
// panel by panel through the NVSwitch (multimem.ld_reduce -> x scale ->
// multimem.st into every rank's W_avg -> multimem.red on the panel counter) so
// that the tensor-core warps of the same kernel can consume finished panels.
// Used by the fused kernel of gemm_wgmma.cu.
#pragma once
#include "device_sync.cuh"
#include "vec_ops.cuh"

namespace m4t {

struct CommArgs {
  SyncCtx sync;
  char* mc_heap;        // multicast mapping of the symmetric heap
  char* my_heap;
  int64_t w_off;        // byte offset of the weight inside every rank's heap
  int64_t wavg_off;     // byte offset of the W_avg buffer inside every rank's heap
  int64_t flags_off;    // byte offset of the panel counters
  float scale;
  int do_barrier;       // 1: cross-rank barrier before the first multimem.ld_reduce
  int debug_skip;       // M4T_FUSED_DEBUG bit0: publish panels without moving data (timing experiments only)
};

// Executed by kCommWarps warps (threads [first_thread, first_thread + kCommWarps*32)).
// Panel = kPanelRows rows of the [N, K] weight; rank r owns rows
// [r*kPanelRows/P, (r+1)*kPanelRows/P) of every panel.
template <int kCommWarps, int kPanelRows>
__device__ __forceinline__ void comm_allreduce_panels(const CommArgs& cm, int first_thread, int n_panels, int K) {
  constexpr int BN = kPanelRows;
  const int n_tiles = n_panels;
  const int lane = threadIdx.x & 31;
    const SyncCtx& c = cm.sync;
    const int P = c.size, r = c.rank;
    const int ct = threadIdx.x - first_thread;  // 0 .. kCommWarps*32-1
    constexpr int kCommThreads = kCommWarps * 32;
    unsigned long long fb = 0;
    if (cm.do_barrier) {
      // every rank's weight (in its heap) is final before anyone reduces it
      fb = read_flag_base(c);
      asm volatile("bar.sync 1, %0;" ::"n"(kCommThreads));
      if (ct < P && ct != r) {
        const uint32_t v = static_cast<uint32_t>(fb + 1ull);
        st_release_sys_u32(c.pads[ct] + blockIdx.x * kMaxGpuPeers + r, v);
        wait_flag_ge(c.pads[r] + blockIdx.x * kMaxGpuPeers + ct, v, c);
      }
      asm volatile("bar.sync 1, %0;" ::"n"(kCommThreads));
    }
    const int64_t row_bytes = static_cast<int64_t>(K) * 2;
    const int rows_per_rank = BN / P;                      // host guarantees divisibility
    const int64_t slice_vecs = rows_per_rank * row_bytes / 16;
    DevEpilogue e;
    e.scale_f = cm.scale;
    e.scale_d = cm.scale;
    e.has_scale = 1;
    e.acc = nullptr;
    uint32_t* mc_flags = reinterpret_cast<uint32_t*>(cm.mc_heap + cm.flags_off);
    // One WARP per panel, round robin: four panels are in flight per CTA, so the
    // switch round trips (ld_reduce -> st -> release) of consecutive panels
    // overlap instead of forming one serial chain.  This CTA's share of a panel
    // slice is the contiguous vector range [lo, hi).
    constexpr int kCU = 8;  // independent multimem.ld_reduce requests in flight per lane
    const int cw = ct >> 5;
    const int64_t per_cta = (slice_vecs + gridDim.x - 1) / gridDim.x;
    const int64_t lo = min(slice_vecs, static_cast<int64_t>(blockIdx.x) * per_cta);
    const int64_t hi = min(slice_vecs, lo + per_cta);
    for (int p = cw; p < n_tiles; p += kCommWarps) {
      const int64_t base = (static_cast<int64_t>(p) * BN + static_cast<int64_t>(r) * rows_per_rank) * row_bytes;
      for (int64_t v0 = (cm.debug_skip & 1) ? hi : lo + lane; v0 < hi; v0 += 32 * kCU) {
        Vec16 x[kCU];
#pragma unroll
        for (int u = 0; u < kCU; ++u) {
          const int64_t v = v0 + u * 32;
          if (v < hi) x[u] = multimem_ld_reduce_vec<NvlsKind::ADD_BF16>(cm.mc_heap + cm.w_off + base + v * 16);
        }
#pragma unroll
        for (int u = 0; u < kCU; ++u) {
          const int64_t v = v0 + u * 32;
          if (v >= hi) continue;
          float a[8];
          VecOf<DType::BF16>::unpack(x[u], a);
          apply_scale<DType::BF16>(a, e);
          multimem_st_vec(cm.mc_heap + cm.wavg_off + base + v * 16, VecOf<DType::BF16>::pack(a));
        }
      }
      // publish: this CTA's share of panel p is in every rank's W_avg
      __syncwarp();
      if (lane == 0) {
        __threadfence_system();
        asm volatile("multimem.red.release.sys.global.add.u32 [%0], %1;" ::"l"(mc_flags + p), "r"(1u) : "memory");
      }
    }
    asm volatile("bar.sync 1, %0;" ::"n"(kCommThreads));
    if (cm.do_barrier && ct == 0) {
      // advance the communicator's flag/op counters exactly like finish_op()
      __threadfence();
      const unsigned int prev = atomicAdd(c.done_ctr, 1u);
      if (prev == gridDim.x - 1) {
        *c.done_ctr = 0;
        __threadfence();
        atomicAdd(c.counters + 0, 1ull);
        atomicAdd(c.counters + 1, 1ull);
      }
    }
}

}  // namespace m4t
