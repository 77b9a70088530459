#include <map>
#include <mutex>
#include <string>
// Allreduce over NVLink 4 / NVSwitch: one launch per collective, forward AND
// backward (the adjoint of Allreduce(SUM) is Allreduce(SUM), reference
// csrc/extension.cpp:265-272), with the adjacent elementwise work fused in:
//   out = accumulate + scale * reduce_ranks(in)        (cast in the store)
//
// Three algorithms, all built from per-block pipelines that meet the
// same-index block of every peer on signal-pad flags (device_sync.cuh):
//   ONESHOT  push my vector into slot[rank] of every peer's staging half
//            (one multimem.st when NVLS is mapped, else P peer stores), one
//            barrier, reduce the P slots locally in rank order.  Latency path.
//   TWOSHOT  stage -> barrier -> reduce my shard from all peers' staging over
//            NVLink loads -> barrier -> pull every owner's reduced shard.
//            Generic: every dtype x op.
//   NVLS     stage -> barrier -> multimem.ld_reduce my shard (the switch adds)
//            -> multimem.st the result to every rank -> barrier -> local
//            copy-out with the epilogue.  Bandwidth path.
// Reduction order is rank 0..P-1 (or the switch's fixed tree), and every shard
// is reduced exactly once by its owner, so all ranks obtain identical bits -
// required for lock-step optimisers (reference doc/examples.rst:46-65).
#include <algorithm>
#include <atomic>

#include "kernels.h"
#include "vec_ops.cuh"

namespace m4t {

namespace {

constexpr int kThreads = 512;

struct ArArgs {
  SyncCtx sync;
  char* heap[kMaxGpuPeers];
  char* mc_heap;
  const void* in;
  void* out;
  DevEpilogue epi;
  int64_t stage_off;
  int64_t half_bytes;
  int64_t n;           // elements
  int64_t nvec;        // 16-byte vectors covering n
  int64_t chunk_vecs;  // vectors per chunk (all shards together)
  int64_t slot_bytes;  // ONESHOT: bytes per rank slot
  int aligned;         // in/out/acc 16-byte aligned
  int skip_mask;       // debug only (M4T_AR_DEBUG_SKIP): bit0 skip phase A, bit1 B, bit2 C
  int64_t sym_in_off;  // >= 0: the input already lives at this heap offset on every rank (zero copy:
                       // phase A is skipped and peers / the switch read the tensor in place)
};

template <DType DT, ReduceOp OP>
__global__ void __launch_bounds__(kThreads) allreduce_oneshot_kernel(const ArArgs a) {
  using V = VecOf<DT>;
  const SyncCtx& c = a.sync;
  const unsigned long long fb = read_flag_base(c);
  const int par = static_cast<int>(read_op_count(c) & 1ull);
  const int64_t half = a.stage_off + static_cast<int64_t>(par) * a.half_bytes;
  const int P = c.size, r = c.rank;
  const int64_t stride = static_cast<int64_t>(gridDim.x) * kThreads;
  const int64_t first = static_cast<int64_t>(blockIdx.x) * kThreads + threadIdx.x;
  const bool al = a.aligned != 0;

  // push my contribution into slot[r] on every rank
  for (int64_t i = first; i < a.nvec; i += stride) {
    const Vec16 v = load_private<DT>(a.in, i, a.n, al);
    const int64_t off = half + static_cast<int64_t>(r) * a.slot_bytes + i * 16;
    if (a.mc_heap && P >= 4) {
      multimem_st_vec(a.mc_heap + off, v);  // one store, the switch replicates
    } else {
#pragma unroll 1
      for (int p = 0; p < P; ++p) st_vec(a.heap[p] + off, v);
    }
  }
  block_barrier_all(c, fb, 0);
  // reduce the P slots that landed in my own HBM
  const char* mine = a.heap[r] + half;
  for (int64_t i = first; i < a.nvec; i += stride) {
    typename V::A acc[V::N];
    init_from<DT, OP>(acc, ld_vec_sys(mine + i * 16));
#pragma unroll 1
    for (int p = 1; p < P; ++p)
      combine_into<DT, OP>(acc, ld_vec_sys(mine + static_cast<int64_t>(p) * a.slot_bytes + i * 16));
    apply_scale<DT>(acc, a.epi);
    apply_accumulate<DT>(acc, a.epi, i, a.n, al);
    store_private<DT>(a.out, i, a.n, al, V::pack(acc));
  }
  finish_op(c, 1);
}

// TWOSHOT (NK == NONE) and NVLS (NK != NONE) share the chunked three-phase pipeline.
// Every phase keeps kUnroll independent 16-byte requests in flight per thread:
// the NVLink round trip is ~2 us, so memory-level parallelism, not the
// instruction count, sets the bandwidth.
constexpr int kUnroll = 4;

template <DType DT, ReduceOp OP, NvlsKind NK>
__global__ void __launch_bounds__(kThreads) allreduce_twoshot_kernel(const ArArgs a) {
  using V = VecOf<DT>;
  const SyncCtx& c = a.sync;
  const unsigned long long fb = read_flag_base(c);
  const int par = static_cast<int>(read_op_count(c) & 1ull);
  const int P = c.size, r = c.rank;
  const bool al = a.aligned != 0;
  // staging half: [ in copy : nvec*16 ][ reduced out : nvec*16 ]
  const int64_t stage_in = a.stage_off + static_cast<int64_t>(par) * a.half_bytes;
  const bool zero_copy = a.sym_in_off >= 0;
  const int64_t in_off = zero_copy ? a.sym_in_off : stage_in;
  const int64_t out_off = stage_in + ((a.nvec * 16 + 127) / 128) * 128;
  char* my_in = a.heap[r] + in_off;
  char* my_out = a.heap[r] + out_off;
  const int64_t gstride = static_cast<int64_t>(gridDim.x) * kThreads;
  const int64_t first = static_cast<int64_t>(blockIdx.x) * kThreads + threadIdx.x;

  int bar = 0;
  for (int64_t base = 0; base < a.nvec; base += a.chunk_vecs) {
    const int64_t cc = min(a.chunk_vecs, a.nvec - base);
    const int64_t L = (cc + P - 1) / P;  // shard length inside this chunk
    // items of this thread in the all-shard phases (A, C): (w, q) pairs, q fastest
    const int64_t nw = first < L ? (L - first + gstride - 1) / gstride : 0;
    const int64_t nitems = nw * P;
    // ---- phase A: stage my part of every shard (block b owns pattern b of each shard)
    for (int64_t j0 = ((a.skip_mask & 1) || zero_copy) ? nitems : 0; j0 < nitems; j0 += kUnroll) {
      Vec16 v[kUnroll];
      int64_t idx[kUnroll];
#pragma unroll
      for (int u = 0; u < kUnroll; ++u) {
        const int64_t j = j0 + u;
        const int64_t i = (j % P) * L + first + (j / P) * gstride;
        idx[u] = (j < nitems && i < cc) ? i : -1;
        if (idx[u] >= 0) v[u] = load_private<DT>(a.in, base + idx[u], a.n, al);
      }
#pragma unroll
      for (int u = 0; u < kUnroll; ++u)
        if (idx[u] >= 0) st_vec(my_in + (base + idx[u]) * 16, v[u]);
    }
    block_barrier_all(c, fb, bar++);
    // ---- phase B: reduce shard r
    for (int64_t w0 = (a.skip_mask & 2) ? nw : 0; w0 < nw; w0 += kUnroll) {
      int64_t off[kUnroll];
#pragma unroll
      for (int u = 0; u < kUnroll; ++u) {
        const int64_t i = static_cast<int64_t>(r) * L + first + (w0 + u) * gstride;
        off[u] = (w0 + u < nw && i < cc) ? (base + i) * 16 : -1;
      }
      if constexpr (NK != NvlsKind::NONE) {
        Vec16 v[kUnroll];
#pragma unroll
        for (int u = 0; u < kUnroll; ++u)
          if (off[u] >= 0) v[u] = multimem_ld_reduce_vec<NK>(a.mc_heap + in_off + off[u]);
#pragma unroll
        for (int u = 0; u < kUnroll; ++u) {
          if (off[u] < 0) continue;
          if (a.epi.has_scale) {
            typename V::A acc[V::N];
            V::unpack(v[u], acc);
            apply_scale<DT>(acc, a.epi);
            v[u] = V::pack(acc);
          }
          multimem_st_vec(a.mc_heap + out_off + off[u], v[u]);
        }
      } else {
        typename V::A acc[kUnroll][V::N];
#pragma unroll
        for (int u = 0; u < kUnroll; ++u)
          if (off[u] >= 0) init_from<DT, OP>(acc[u], ld_vec_sys(a.heap[0] + in_off + off[u]));
#pragma unroll 1
        for (int p = 1; p < P; ++p) {
          Vec16 v[kUnroll];
#pragma unroll
          for (int u = 0; u < kUnroll; ++u)
            if (off[u] >= 0) v[u] = ld_vec_sys(a.heap[p] + in_off + off[u]);
#pragma unroll
          for (int u = 0; u < kUnroll; ++u)
            if (off[u] >= 0) combine_into<DT, OP>(acc[u], v[u]);
        }
#pragma unroll
        for (int u = 0; u < kUnroll; ++u) {
          if (off[u] < 0) continue;
          apply_scale<DT>(acc[u], a.epi);
          st_vec(my_out + off[u], V::pack(acc[u]));
        }
      }
    }
    block_barrier_all(c, fb, bar++);
    // ---- phase C: collect all shards (NVLS: already in my HBM; TWOSHOT: pull from owners)
    for (int64_t j0 = (a.skip_mask & 4) ? nitems : 0; j0 < nitems; j0 += kUnroll) {
      Vec16 v[kUnroll];
      int64_t idx[kUnroll];
#pragma unroll
      for (int u = 0; u < kUnroll; ++u) {
        const int64_t j = j0 + u;
        const int q = static_cast<int>(j % P);
        const int64_t i = static_cast<int64_t>(q) * L + first + (j / P) * gstride;
        idx[u] = (j < nitems && i < cc) ? i : -1;
        if (idx[u] >= 0) {
          const char* src = (NK != NvlsKind::NONE) ? my_out : (a.heap[q] + out_off);
          v[u] = ld_vec_sys(src + (base + idx[u]) * 16);
        }
      }
      // the accumulate operand is requested for the whole batch before any of it is used, so
      // its HBM latency is paid once per batch instead of once per vector
      Vec16 av[kUnroll];
      if (a.epi.acc) {
#pragma unroll
        for (int u = 0; u < kUnroll; ++u)
          if (idx[u] >= 0) av[u] = load_private<DT>(a.epi.acc, base + idx[u], a.n, al);
      }
#pragma unroll
      for (int u = 0; u < kUnroll; ++u) {
        if (idx[u] < 0) continue;
        if (a.epi.acc) {
          typename V::A acc[V::N];
          V::unpack(v[u], acc);
          add_vec<DT>(acc, av[u]);
          v[u] = V::pack(acc);
        }
        store_private<DT>(a.out, base + idx[u], a.n, al, v[u]);
      }
    }
  }
  finish_op(c, static_cast<unsigned int>(bar));
}

// ---------------------------------------------------------------------------
// Pipelined two-shot / NVLS allreduce.  One CTA = two 512-thread roles:
//   L (local)  : A(c) stage chunk c into my heap; C(c-1) copy reduced chunk c-1
//                out of my heap with the epilogue.            HBM-bound.
//   N (network): B(c) multimem.ld_reduce + multimem.st (or P peer loads +
//                store, then peers pull in C).                NVLink-bound.
// The roles are decoupled by chunk-indexed flags in two pads (A-done, B-done),
// exchanged with the same-index CTA of every peer, so the NVLink phase of chunk
// c overlaps the HBM phases of chunks c+1 / c-1 instead of alternating with
// them.  Flags are monotone (flag_base + chunk + 1): no resets, no grid sync.
// ---------------------------------------------------------------------------
constexpr int kRoleThreads = 512;
constexpr int kPipeUnroll = 4;

__device__ __forceinline__ void role_sync(int id) { asm volatile("bar.sync %0, %1;" ::"r"(id), "n"(kRoleThreads) : "memory"); }

template <DType DT, ReduceOp OP, NvlsKind NK>
__global__ void __launch_bounds__(2 * kRoleThreads, 1) allreduce_pipelined_kernel(const ArArgs a) {
  using V = VecOf<DT>;
  const SyncCtx& c = a.sync;
  const unsigned long long fb = read_flag_base(c);
  const int par = static_cast<int>(read_op_count(c) & 1ull);
  const int P = c.size, r = c.rank;
  const bool al = a.aligned != 0;
  const int64_t in_off = a.stage_off + static_cast<int64_t>(par) * a.half_bytes;
  const int64_t out_off = in_off + ((a.nvec * 16 + 127) / 128) * 128;
  char* my_in = a.heap[r] + in_off;
  char* my_out = a.heap[r] + out_off;
  const bool is_net = threadIdx.x >= kRoleThreads;
  const int t = threadIdx.x - (is_net ? kRoleThreads : 0);
  const int64_t gstride = static_cast<int64_t>(gridDim.x) * kRoleThreads;
  const int64_t first = static_cast<int64_t>(blockIdx.x) * kRoleThreads + t;
  const int64_t nchunks = (a.nvec + a.chunk_vecs - 1) / a.chunk_vecs;
  // flag slots of this CTA's channel: pad A at heap offset 0, pad B at kPadBOffset
  const int64_t slot = static_cast<int64_t>(blockIdx.x) * kMaxGpuPeers;
  constexpr int64_t kPadBOffset = 64 * 1024;

  auto flag_a = [&](int owner, int src) { return c.pads[owner] + slot + src; };
  auto flag_b = [&](int owner, int src) {
    return reinterpret_cast<uint32_t*>(reinterpret_cast<char*>(c.pads[owner]) + kPadBOffset) + slot + src;
  };

  if (!is_net) {
    // ============================ role L ============================
    for (int64_t ck = 0; ck <= nchunks; ++ck) {
      if (ck < nchunks) {
        // ---- A(ck): stage my pattern of every shard
        const int64_t base = ck * a.chunk_vecs;
        const int64_t cc = min(a.chunk_vecs, a.nvec - base);
        const int64_t L = (cc + P - 1) / P;
        const int64_t nw = first < L ? (L - first + gstride - 1) / gstride : 0;
        const int64_t nitems = nw * P;
        for (int64_t j0 = 0; j0 < nitems; j0 += kPipeUnroll) {
          Vec16 v[kPipeUnroll];
          int64_t idx[kPipeUnroll];
#pragma unroll
          for (int u = 0; u < kPipeUnroll; ++u) {
            const int64_t j = j0 + u;
            const int64_t i = (j % P) * L + first + (j / P) * gstride;
            idx[u] = (j < nitems && i < cc) ? i : -1;
            if (idx[u] >= 0) v[u] = load_private<DT>(a.in, base + idx[u], a.n, al);
          }
#pragma unroll
          for (int u = 0; u < kPipeUnroll; ++u)
            if (idx[u] >= 0) st_vec(my_in + (base + idx[u]) * 16, v[u]);
        }
        role_sync(1);
        if (t < P) st_release_sys_u32(flag_a(t, r), static_cast<uint32_t>(fb + ck + 1));
      }
      if (ck > 0) {
        // ---- C(ck-1): reduced chunk is in my heap (NVLS) or at its owners (two-shot)
        const int64_t cprev = ck - 1;
        if (t < P) wait_flag_ge(flag_b(r, t), static_cast<uint32_t>(fb + cprev + 1), c);
        role_sync(1);
        const int64_t base = cprev * a.chunk_vecs;
        const int64_t cc = min(a.chunk_vecs, a.nvec - base);
        const int64_t L = (cc + P - 1) / P;
        const int64_t nw = first < L ? (L - first + gstride - 1) / gstride : 0;
        const int64_t nitems = nw * P;
        for (int64_t j0 = 0; j0 < nitems; j0 += kPipeUnroll) {
          Vec16 v[kPipeUnroll];
          int64_t idx[kPipeUnroll];
#pragma unroll
          for (int u = 0; u < kPipeUnroll; ++u) {
            const int64_t j = j0 + u;
            const int q = static_cast<int>(j % P);
            const int64_t i = static_cast<int64_t>(q) * L + first + (j / P) * gstride;
            idx[u] = (j < nitems && i < cc) ? i : -1;
            if (idx[u] >= 0) {
              const char* src = (NK != NvlsKind::NONE) ? my_out : (a.heap[q] + out_off);
              v[u] = ld_vec_sys(src + (base + idx[u]) * 16);
            }
          }
#pragma unroll
          for (int u = 0; u < kPipeUnroll; ++u) {
            if (idx[u] < 0) continue;
            if (a.epi.acc) {
              typename V::A acc[V::N];
              V::unpack(v[u], acc);
              apply_accumulate<DT>(acc, a.epi, base + idx[u], a.n, al);
              v[u] = V::pack(acc);
            }
            store_private<DT>(a.out, base + idx[u], a.n, al, v[u]);
          }
        }
      }
    }
  } else {
    // ============================ role N ============================
    for (int64_t ck = 0; ck < nchunks; ++ck) {
      if (t < P) wait_flag_ge(flag_a(r, t), static_cast<uint32_t>(fb + ck + 1), c);
      role_sync(2);
      const int64_t base = ck * a.chunk_vecs;
      const int64_t cc = min(a.chunk_vecs, a.nvec - base);
      const int64_t L = (cc + P - 1) / P;
      const int64_t nw = first < L ? (L - first + gstride - 1) / gstride : 0;
      for (int64_t w0 = 0; w0 < nw; w0 += kPipeUnroll) {
        int64_t off[kPipeUnroll];
#pragma unroll
        for (int u = 0; u < kPipeUnroll; ++u) {
          const int64_t i = static_cast<int64_t>(r) * L + first + (w0 + u) * gstride;
          off[u] = (w0 + u < nw && i < cc) ? (base + i) * 16 : -1;
        }
        if constexpr (NK != NvlsKind::NONE) {
          Vec16 v[kPipeUnroll];
#pragma unroll
          for (int u = 0; u < kPipeUnroll; ++u)
            if (off[u] >= 0) v[u] = multimem_ld_reduce_vec<NK>(a.mc_heap + in_off + off[u]);
#pragma unroll
          for (int u = 0; u < kPipeUnroll; ++u) {
            if (off[u] < 0) continue;
            if (a.epi.has_scale) {
              typename V::A acc[V::N];
              V::unpack(v[u], acc);
              apply_scale<DT>(acc, a.epi);
              v[u] = V::pack(acc);
            }
            multimem_st_vec(a.mc_heap + out_off + off[u], v[u]);
          }
        } else {
#pragma unroll
          for (int u = 0; u < kPipeUnroll; ++u) {
            if (off[u] < 0) continue;
            typename V::A acc[V::N];
            init_from<DT, OP>(acc, ld_vec_sys(a.heap[0] + in_off + off[u]));
#pragma unroll 1
            for (int p = 1; p < P; ++p) combine_into<DT, OP>(acc, ld_vec_sys(a.heap[p] + in_off + off[u]));
            apply_scale<DT>(acc, a.epi);
            st_vec(my_out + off[u], V::pack(acc));
          }
        }
      }
      role_sync(2);
      if (t < P) st_release_sys_u32(flag_b(t, r), static_cast<uint32_t>(fb + ck + 1));
    }
  }
  finish_op(c, static_cast<unsigned int>(nchunks));
}

template <DType DT, ReduceOp OP>
__global__ void __launch_bounds__(kThreads) local_epilogue_kernel(const void* in, void* out, int64_t n,
                                                                   int64_t nvec, DevEpilogue epi, int aligned) {
  using V = VecOf<DT>;
  const bool al = aligned != 0;
  const int64_t stride = static_cast<int64_t>(gridDim.x) * kThreads;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * kThreads + threadIdx.x; i < nvec; i += stride) {
    typename V::A acc[V::N];
    init_from<DT, OP>(acc, load_private<DT>(in, i, n, al));
    apply_scale<DT>(acc, epi);
    apply_accumulate<DT>(acc, epi, i, n, al);
    store_private<DT>(out, i, n, al, V::pack(acc));
  }
}

bool is_aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

template <DType DT, ReduceOp OP> struct LaunchOneshot {
  static void run(const ArArgs& a, int blocks, cudaStream_t s) {
    allreduce_oneshot_kernel<DT, OP><<<blocks, kThreads, 0, s>>>(a);
  }
};
template <DType DT, ReduceOp OP> struct LaunchTwoshot {
  static void run(const ArArgs& a, int blocks, cudaStream_t s) {
    allreduce_twoshot_kernel<DT, OP, NvlsKind::NONE><<<blocks, kThreads, 0, s>>>(a);
  }
};
template <DType DT, ReduceOp OP> struct LaunchLocal {
  static void run(const void* in, void* out, int64_t n, int64_t nvec, const DevEpilogue& e, int aligned,
                  int blocks, cudaStream_t s) {
    local_epilogue_kernel<DT, OP><<<blocks, kThreads, 0, s>>>(in, out, n, nvec, e, aligned);
  }
};

NvlsKind nvls_kind(DType dt, ReduceOp op) {
  if (op == ReduceOp::SUM) {
    if (dt == DType::F32) return NvlsKind::ADD_F32;
    if (dt == DType::BF16) return NvlsKind::ADD_BF16;
    if (dt == DType::F16) return NvlsKind::ADD_F16;
  } else if (op == ReduceOp::MAX) {
    if (dt == DType::BF16) return NvlsKind::MAX_BF16;
    if (dt == DType::F16) return NvlsKind::MAX_F16;
  } else if (op == ReduceOp::MIN) {
    if (dt == DType::BF16) return NvlsKind::MIN_BF16;
    if (dt == DType::F16) return NvlsKind::MIN_F16;
  }
  return NvlsKind::NONE;
}

template <DType DT, ReduceOp OP> struct LaunchPipelinedTwoshot {
  static void run(const ArArgs& a, int blocks, cudaStream_t s) {
    allreduce_pipelined_kernel<DT, OP, NvlsKind::NONE><<<blocks, 2 * kRoleThreads, 0, s>>>(a);
  }
};

void launch_nvls_pipelined(NvlsKind k, const ArArgs& a, int blocks, cudaStream_t s) {
  switch (k) {
    case NvlsKind::ADD_F32:
      allreduce_pipelined_kernel<DType::F32, ReduceOp::SUM, NvlsKind::ADD_F32><<<blocks, 2 * kRoleThreads, 0, s>>>(a);
      break;
    case NvlsKind::ADD_BF16:
      allreduce_pipelined_kernel<DType::BF16, ReduceOp::SUM, NvlsKind::ADD_BF16><<<blocks, 2 * kRoleThreads, 0, s>>>(a);
      break;
    case NvlsKind::ADD_F16:
      allreduce_pipelined_kernel<DType::F16, ReduceOp::SUM, NvlsKind::ADD_F16><<<blocks, 2 * kRoleThreads, 0, s>>>(a);
      break;
    case NvlsKind::MAX_BF16:
      allreduce_pipelined_kernel<DType::BF16, ReduceOp::MAX, NvlsKind::MAX_BF16><<<blocks, 2 * kRoleThreads, 0, s>>>(a);
      break;
    case NvlsKind::MIN_BF16:
      allreduce_pipelined_kernel<DType::BF16, ReduceOp::MIN, NvlsKind::MIN_BF16><<<blocks, 2 * kRoleThreads, 0, s>>>(a);
      break;
    case NvlsKind::MAX_F16:
      allreduce_pipelined_kernel<DType::F16, ReduceOp::MAX, NvlsKind::MAX_F16><<<blocks, 2 * kRoleThreads, 0, s>>>(a);
      break;
    case NvlsKind::MIN_F16:
      allreduce_pipelined_kernel<DType::F16, ReduceOp::MIN, NvlsKind::MIN_F16><<<blocks, 2 * kRoleThreads, 0, s>>>(a);
      break;
    default:
      M4T_CHECK(false, "no NVLS kernel for this dtype/op");
  }
}

void launch_nvls(NvlsKind k, const ArArgs& a, int blocks, cudaStream_t s) {
  switch (k) {
    case NvlsKind::ADD_F32:
      allreduce_twoshot_kernel<DType::F32, ReduceOp::SUM, NvlsKind::ADD_F32><<<blocks, kThreads, 0, s>>>(a);
      break;
    case NvlsKind::ADD_BF16:
      allreduce_twoshot_kernel<DType::BF16, ReduceOp::SUM, NvlsKind::ADD_BF16><<<blocks, kThreads, 0, s>>>(a);
      break;
    case NvlsKind::ADD_F16:
      allreduce_twoshot_kernel<DType::F16, ReduceOp::SUM, NvlsKind::ADD_F16><<<blocks, kThreads, 0, s>>>(a);
      break;
    case NvlsKind::MAX_BF16:
      allreduce_twoshot_kernel<DType::BF16, ReduceOp::MAX, NvlsKind::MAX_BF16><<<blocks, kThreads, 0, s>>>(a);
      break;
    case NvlsKind::MIN_BF16:
      allreduce_twoshot_kernel<DType::BF16, ReduceOp::MIN, NvlsKind::MIN_BF16><<<blocks, kThreads, 0, s>>>(a);
      break;
    case NvlsKind::MAX_F16:
      allreduce_twoshot_kernel<DType::F16, ReduceOp::MAX, NvlsKind::MAX_F16><<<blocks, kThreads, 0, s>>>(a);
      break;
    case NvlsKind::MIN_F16:
      allreduce_twoshot_kernel<DType::F16, ReduceOp::MIN, NvlsKind::MIN_F16><<<blocks, kThreads, 0, s>>>(a);
      break;
    default:
      M4T_CHECK(false, "no NVLS kernel for this dtype/op");
  }
}

void check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  M4T_CHECK(e == cudaSuccess, what << " launch failed: " << cudaGetErrorString(e));
  note_kernel_launch();
}

}  // namespace

namespace {
std::atomic<unsigned long long> g_kernel_launches{0};
}
unsigned long long kernel_launch_count() { return g_kernel_launches.load(std::memory_order_relaxed); }
void note_kernel_launch() { g_kernel_launches.fetch_add(1, std::memory_order_relaxed); }

namespace {
std::mutex g_table_mu;
std::map<std::string, unsigned long long>& launch_table() {
  static std::map<std::string, unsigned long long> t;
  return t;
}
}  // namespace

void note_kernel_launch(const char* name) {
  g_kernel_launches.fetch_add(1, std::memory_order_relaxed);
  std::lock_guard<std::mutex> g(g_table_mu);
  launch_table()[name] += 1;
}

std::vector<std::pair<std::string, unsigned long long>> kernel_launch_table() {
  std::lock_guard<std::mutex> g(g_table_mu);
  return {launch_table().begin(), launch_table().end()};
}

bool nvls_supported(DType dt, ReduceOp op) { return nvls_kind(dt, op) != NvlsKind::NONE; }

int64_t allreduce_stage_bytes(int64_t n, DType dt, ArAlgo algo, int size) {
  const int64_t nvec = (n * dtype_size(dt) + 15) / 16;
  const int64_t span = ((nvec * 16 + 127) / 128) * 128;
  if (algo == ArAlgo::ONESHOT) return span * size;
  return 2 * span;
}

void launch_local_epilogue(const void* in, void* out, int64_t n, DType dt, ReduceOp op, const Epilogue& epi,
                           int sm_count, cudaStream_t stream) {
  if (n == 0) return;
  const int64_t nvec = (n * dtype_size(dt) + 15) / 16;
  const DevEpilogue de = make_dev_epilogue(epi);
  const int aligned = is_aligned16(in) && is_aligned16(out) && (!epi.accumulate || is_aligned16(epi.accumulate));
  const int blocks = static_cast<int>(std::min<int64_t>((nvec + kThreads - 1) / kThreads, 4LL * sm_count));
  M4T_DISPATCH_DTYPE_OP(dt, op, LaunchLocal, in, out, n, nvec, de, aligned, blocks, stream);
  check_launch("local_epilogue");
}

void launch_allreduce(const DeviceComm& dc, const void* in, void* out, int64_t n, DType dt, ReduceOp op,
                      const Epilogue& epi, ArAlgo algo, int blocks, int64_t chunk_bytes, cudaStream_t stream,
                      int64_t sym_in_off) {
  check_op_dtype(op, dt);
  M4T_CHECK(algo == ArAlgo::ONESHOT || algo == ArAlgo::TWOSHOT || algo == ArAlgo::NVLS,
            "launch_allreduce needs a concrete algorithm");
  ArArgs a;
  a.sync = dc.sync;
  for (int p = 0; p < kMaxGpuPeers; ++p) a.heap[p] = dc.heap[p];
  a.mc_heap = dc.mc_heap;
  a.in = in;
  a.out = out;
  a.epi = make_dev_epilogue(epi);
  a.stage_off = dc.stage_off;
  a.half_bytes = dc.half_bytes;
  a.n = n;
  a.nvec = (n * dtype_size(dt) + 15) / 16;
  a.slot_bytes = ((a.nvec * 16 + 127) / 128) * 128;
  a.aligned = is_aligned16(in) && is_aligned16(out) && (!epi.accumulate || is_aligned16(epi.accumulate));
  static const int skip_mask = static_cast<int>(env_i64("M4T_AR_DEBUG_SKIP", 0));  // read once (timing experiments)
  a.skip_mask = skip_mask;
  a.sym_in_off = -1;
  M4T_CHECK(allreduce_stage_bytes(n, dt, algo, dc.sync.size) <= dc.half_bytes,
            "allreduce of " << n << " elements does not fit the staging half (" << dc.half_bytes << " B)");
  blocks = std::max(1, std::min(blocks, kMaxChannels));
  const int P = dc.sync.size;
  if (algo == ArAlgo::ONESHOT) {
    blocks = static_cast<int>(std::min<int64_t>(blocks, std::max<int64_t>(1, (a.nvec + kThreads - 1) / kThreads)));
    a.chunk_vecs = a.nvec;
    M4T_DISPATCH_DTYPE_OP(dt, op, LaunchOneshot, a, blocks, stream);
    check_launch("allreduce_oneshot");
    return;
  }
  // chunk = all P shards of one pipeline step; keep it a multiple of P vectors
  int64_t cv = std::max<int64_t>(chunk_bytes / 16, P);
  cv = (cv + P - 1) / P * P;
  a.chunk_vecs = std::max<int64_t>(1, std::min(cv, std::max<int64_t>(a.nvec, 1)));
  const int64_t shard = (a.chunk_vecs + P - 1) / P;
  blocks = static_cast<int>(std::min<int64_t>(blocks, std::max<int64_t>(1, (shard + kThreads - 1) / kThreads)));
  // Pipelined role-split kernels: one 1024-thread CTA per SM, >= 2 chunks to overlap.
  static const bool pipe_enabled = env_i64("M4T_AR_PIPE", 1) != 0;  // read once
  const bool pipelined = pipe_enabled && a.nvec > a.chunk_vecs;
  if (pipelined) blocks = std::min(blocks, dc.sm_count);
  // zero copy: single-chunk kernels only (the chunk loop of the two-shot kernel indexes one buffer)
  if (!pipelined && a.nvec <= a.chunk_vecs && sym_in_off >= 0 && (sym_in_off & 15) == 0) a.sym_in_off = sym_in_off;
  if (algo == ArAlgo::NVLS) {
    M4T_CHECK(dc.mc_heap != nullptr, "NVLS allreduce requested but no multicast mapping exists");
    if (pipelined) launch_nvls_pipelined(nvls_kind(dt, op), a, blocks, stream);
    else launch_nvls(nvls_kind(dt, op), a, blocks, stream);
    check_launch("allreduce_nvls");
  } else {
    if (pipelined) {
      M4T_DISPATCH_DTYPE_OP(dt, op, LaunchPipelinedTwoshot, a, blocks, stream);
    } else {
      M4T_DISPATCH_DTYPE_OP(dt, op, LaunchTwoshot, a, blocks, stream);
    }
    check_launch("allreduce_twoshot");
  }
}

}  // namespace m4t
