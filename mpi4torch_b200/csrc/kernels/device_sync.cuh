// Device-side cross-GPU synchronisation over the symmetric signal pad, and the
// NVLS (NVSwitch multicast) load-reduce / store wrappers.
//
// Replaces the host-blocking MPI progress engine of the reference (every call
// in csrc/extension.cpp blocks the host thread inside MPI, e.g. :297-300):
// here a collective is one stream-ordered kernel and ranks meet on flags that
// live in each other's HBM, written with st.release.sys over NVLink and polled
// locally with ld.acquire.sys.
//
// Flag protocol: every launch that contains barriers reads two
// device-resident counters of the communicator (identical on all ranks because
// all ranks launch the same collective sequence in one serialised order):
//   counters[0] = flag_base : flag values consumed so far,
//   counters[1] = op_count  : collectives launched so far (staging parity).
// Barrier k of a launch uses the value v = flag_base + k + 1.  Block b uses
// flag channel b: it writes v to pads[peer][b][rank] and waits until
// pads[rank][b][peer] >= v (wrap-safe signed compare).  Values are monotone per
// channel, so no reset traffic is needed and a block that skips values
// (smaller grid) is harmless.  The last block to finish advances flag_base by
// the launch's barrier count and op_count by one - all on the device, so the
// kernels are CUDA-graph capturable.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace m4t {

constexpr int kMaxGpuPeers = 16;       // one NVLink domain (8 on HGX H100)
constexpr int kMaxChannels = 512;      // barrier channels == max grid of barrier kernels
constexpr int kErrTimeout = 1;

struct SyncCtx {
  uint32_t* pads[kMaxGpuPeers];  // pads[p]: peer p's barrier flag array [kMaxChannels][kMaxGpuPeers]
  unsigned long long* counters;  // local device memory: [0] flag_base, [1] op_count
  unsigned int* done_ctr;        // local device memory
  int* err_flag;                 // host-mapped pinned word (0 = ok)
  unsigned long long timeout_ns;
  int rank;
  int size;
};

#if defined(__CUDACC__)  // device code below; the structs above are shared with host-only TUs

__device__ __forceinline__ void st_release_sys_u32(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys_u32(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_relaxed_sys_u32(uint32_t* p, uint32_t v) {
  asm volatile("st.relaxed.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_relaxed_sys_u32(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}

// Spins until *flag >= v (wrap-safe).  Bounded: on timeout the error word is
// set and the wait falls through so the kernel terminates instead of hanging
// the GPU (the host surfaces the error at its next check).
__device__ __forceinline__ void wait_flag_ge(const uint32_t* flag, uint32_t v, const SyncCtx& c) {
  if (static_cast<int32_t>(ld_acquire_sys_u32(flag) - v) >= 0) return;
  const unsigned long long t0 = globaltimer_ns();
  unsigned int spins = 0;
  while (static_cast<int32_t>(ld_acquire_sys_u32(flag) - v) < 0) {
    if ((++spins & 0x3ff) == 0) {
      if (globaltimer_ns() - t0 > c.timeout_ns || *reinterpret_cast<volatile int*>(c.err_flag) != 0) {
        *reinterpret_cast<volatile int*>(c.err_flag) = kErrTimeout;
        __threadfence_system();
        return;
      }
    }
  }
}

__device__ __forceinline__ unsigned long long read_flag_base(const SyncCtx& c) {
  return reinterpret_cast<volatile unsigned long long*>(c.counters)[0];
}
__device__ __forceinline__ unsigned long long read_op_count(const SyncCtx& c) {
  return reinterpret_cast<volatile unsigned long long*>(c.counters)[1];
}

// Full barrier of block `blockIdx.x` with the same-index block on every peer.
// All of the block's earlier writes (local, peer or multicast) are released;
// all peers' writes before their matching barrier are acquired.
__device__ __forceinline__ void block_barrier_all(const SyncCtx& c, unsigned long long flag_base, int k) {
  const uint32_t v = static_cast<uint32_t>(flag_base + static_cast<unsigned long long>(k) + 1ull);
  __syncthreads();
  const int p = threadIdx.x;
  if (p < c.size && p != c.rank) {
    st_release_sys_u32(c.pads[p] + blockIdx.x * kMaxGpuPeers + c.rank, v);
    wait_flag_ge(c.pads[c.rank] + blockIdx.x * kMaxGpuPeers + p, v, c);
  }
  __syncthreads();
}

// Call once at the very end of a barrier kernel: the last block to arrive
// advances the counters (`nbarriers` = barriers this launch used per block).
__device__ __forceinline__ void finish_op(const SyncCtx& c, unsigned int nbarriers) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    const unsigned int prev = atomicAdd(c.done_ctr, 1u);
    if (prev == gridDim.x - 1) {
      *c.done_ctr = 0;
      __threadfence();
      atomicAdd(c.counters + 0, static_cast<unsigned long long>(nbarriers));
      atomicAdd(c.counters + 1, 1ull);
    }
  }
}

// ---------------------------------------------------------------------------
// 16-byte vector moves
// ---------------------------------------------------------------------------
struct alignas(16) Vec16 {
  uint32_t w[4];
};

__device__ __forceinline__ Vec16 ld_vec(const void* p) {
  Vec16 v;
  asm volatile("ld.global.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.w[0]), "=r"(v.w[1]), "=r"(v.w[2]), "=r"(v.w[3])
               : "l"(p)
               : "memory");
  return v;
}
// Streaming read of private (read-once) data: do not pollute L1.
__device__ __forceinline__ Vec16 ld_vec_stream(const void* p) {
  Vec16 v;
  asm volatile("ld.global.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.w[0]), "=r"(v.w[1]), "=r"(v.w[2]), "=r"(v.w[3])
               : "l"(p)
               : "memory");
  return v;
}
// Peer / staging reads must observe data written by other GPUs during this
// kernel: relaxed.sys bypasses the (non-coherent) L1.
__device__ __forceinline__ Vec16 ld_vec_sys(const void* p) {
  Vec16 v;
  asm volatile("ld.relaxed.sys.global.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.w[0]), "=r"(v.w[1]), "=r"(v.w[2]), "=r"(v.w[3])
               : "l"(p)
               : "memory");
  return v;
}
__device__ __forceinline__ void st_vec(void* p, const Vec16& v) {
  asm volatile("st.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.w[0]), "r"(v.w[1]), "r"(v.w[2]),
               "r"(v.w[3])
               : "memory");
}

// ---------------------------------------------------------------------------
// NVLS: NVSwitch multicast store and in-switch load-reduce (16 bytes each)
// ---------------------------------------------------------------------------
__device__ __forceinline__ void multimem_st_vec(void* mc_ptr, const Vec16& v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(mc_ptr),
               "f"(__uint_as_float(v.w[0])), "f"(__uint_as_float(v.w[1])), "f"(__uint_as_float(v.w[2])),
               "f"(__uint_as_float(v.w[3]))
               : "memory");
}

#endif  // __CUDACC__

enum class NvlsKind : int { NONE = 0, ADD_F32, ADD_BF16, ADD_F16, MAX_BF16, MIN_BF16, MAX_F16, MIN_F16 };

#if defined(__CUDACC__)

template <NvlsKind K> __device__ __forceinline__ Vec16 multimem_ld_reduce_vec(const void* mc_ptr);

#define M4T_MULTIMEM_LDRED(KIND, PTXOP)                                                        \
  template <> __device__ __forceinline__ Vec16 multimem_ld_reduce_vec<KIND>(const void* mc_ptr) { \
    Vec16 v;                                                                                   \
    asm volatile("multimem.ld_reduce.relaxed.sys.global." PTXOP " {%0,%1,%2,%3}, [%4];"       \
                 : "=r"(v.w[0]), "=r"(v.w[1]), "=r"(v.w[2]), "=r"(v.w[3])                      \
                 : "l"(mc_ptr)                                                                 \
                 : "memory");                                                                  \
    return v;                                                                                  \
  }
M4T_MULTIMEM_LDRED(NvlsKind::ADD_BF16, "add.acc::f32.v4.bf16x2")
M4T_MULTIMEM_LDRED(NvlsKind::ADD_F16, "add.acc::f32.v4.f16x2")
M4T_MULTIMEM_LDRED(NvlsKind::MAX_BF16, "max.v4.bf16x2")
M4T_MULTIMEM_LDRED(NvlsKind::MIN_BF16, "min.v4.bf16x2")
M4T_MULTIMEM_LDRED(NvlsKind::MAX_F16, "max.v4.f16x2")
M4T_MULTIMEM_LDRED(NvlsKind::MIN_F16, "min.v4.f16x2")
#undef M4T_MULTIMEM_LDRED

template <> __device__ __forceinline__ Vec16 multimem_ld_reduce_vec<NvlsKind::ADD_F32>(const void* mc_ptr) {
  Vec16 v;
  float a, b, c, d;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(a), "=f"(b), "=f"(c), "=f"(d)
               : "l"(mc_ptr)
               : "memory");
  v.w[0] = __float_as_uint(a);
  v.w[1] = __float_as_uint(b);
  v.w[2] = __float_as_uint(c);
  v.w[3] = __float_as_uint(d);
  return v;
}

#endif  // __CUDACC__

}  // namespace m4t
