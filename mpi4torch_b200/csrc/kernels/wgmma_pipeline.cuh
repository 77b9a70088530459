// Shared main loop of the Hopper GEMM kernels (gemm_wgmma.cu, wgrad_wgmma.cu).
//
// One persistent CTA per SM computes 128 x BN output tiles (BN = tile_n<FUSED>(): 256, or 128 for
// the fused kernels, whose communication warps need the registers) with BK = 64:
//   warpgroup 0 (warp 0, one lane)  TMA producer: A/B tiles -> smem ring of Tile<BN>::kStages
//   warpgroups 1, 2                 consumers: 64 rows each, wgmma m64nBNk16 into BN/2 fp32
//                                   registers per thread, epilogue straight from registers
//   further warps                   (fused kernels only) communication role
// Each operand is either K-major (one TMA box {64 k, rows}) or MN-major (boxes of
// {64 contiguous m/n, 64 k-rows}); the wgmma transpose bits select the layout, so no
// operand is ever copied transposed.
#pragma once
#include "hopper_ptx.cuh"
#include "vec_ops.cuh"

namespace m4t {
namespace wg {

constexpr int BM = 128, BK = 64;
constexpr int kBoxBytesMN = 64 * BK * 2;  // 8 KiB: one MN-major box
constexpr int kABytes = BM * BK * 2;      // 16 KiB
constexpr int kGemmThreads = 384;         // producer warpgroup + two consumer warpgroups
constexpr int kConsumerWarps = 8;
constexpr int kMaxStages = 6;

template <int BN> struct Tile {
  static_assert(BN == 128 || BN == 256, "tile width");
  static constexpr int kBBytes = BN * BK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kStages = BN == 256 ? 4 : kMaxStages;  // ~192 KiB of ring either way
  static constexpr int kSmemBytes = kStages * kStageBytes + 1024 /*align*/ + 256 /*barriers*/;
};

// The fused kernels' communication warps need registers: half-width tiles there.
template <bool FUSED> constexpr int tile_n() { return FUSED ? 128 : 256; }
// Communication warps of a fused kernel.  The wgrad owner role keeps its rows in registers, so its in-flight round
// trips scale with warps x rows.
constexpr int kCommWarps = 4;

struct __align__(8) Pipe {
  uint64_t full[kMaxStages];
  uint64_t empty[kMaxStages];
};

__device__ __forceinline__ uint8_t* aligned_smem(uint8_t* raw) {
  return reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(raw) + 1023) & ~uintptr_t(1023));
}
template <int BN> __device__ __forceinline__ Pipe* pipe_of(uint8_t* smem) {
  return reinterpret_cast<Pipe*>(smem + Tile<BN>::kStages * Tile<BN>::kStageBytes);
}

template <int BN> __device__ __forceinline__ void init_pipe(Pipe* p) {
  for (int s = 0; s < Tile<BN>::kStages; ++s) {
    tc::mbar_init(&p->full[s], 1);
    tc::mbar_init(&p->empty[s], kConsumerWarps);  // one arrive per consumer warp
  }
  tc::fence_barrier_init();
}

template <int BN> __device__ __forceinline__ void advance(int& stage, uint32_t& phase) {
  if (++stage == Tile<BN>::kStages) {
    stage = 0;
    phase ^= 1;
  }
}

// Producer: one stage = A rows [m0, m0+128) and B rows [n0, n0+BN) of the k-slice starting at k0.
// b_row0 is added to B's row coordinate (n for a K-major B, k for an MN-major one): the batched GEMMs read
// expert e's weights out of one map over the stacked weights with b_row0 = e * (rows of one expert).
template <bool A_MN, bool B_MN, int BN>
__device__ __forceinline__ void load_stage(uint8_t* smem, Pipe* p, int& stage, uint32_t& phase, const CUtensorMap* ma,
                                           const CUtensorMap* mb, int m0, int n0, int k0, int b_row0 = 0) {
  tc::mbar_wait(&p->empty[stage], phase ^ 1);
  uint8_t* sa = smem + stage * Tile<BN>::kStageBytes;
  uint8_t* sb = sa + kABytes;
  tc::mbar_arrive_expect_tx(&p->full[stage], Tile<BN>::kStageBytes);
  if (A_MN) {
#pragma unroll
    for (int ch = 0; ch < BM / 64; ++ch) tc::tma_load_2d(sa + ch * kBoxBytesMN, ma, &p->full[stage], m0 + ch * 64, k0);
  } else {
    tc::tma_load_2d(sa, ma, &p->full[stage], k0, m0);
  }
  if (B_MN) {
#pragma unroll
    for (int ch = 0; ch < BN / 64; ++ch)
      tc::tma_load_2d(sb + ch * kBoxBytesMN, mb, &p->full[stage], n0 + ch * 64, k0 + b_row0);
  } else {
    tc::tma_load_2d(sb, mb, &p->full[stage], k0, n0 + b_row0);
  }
  advance<BN>(stage, phase);
}

// Rows [rows, BK) of every 64-row MN-major box of a stage become zero, so the k-block contracts over its first
// `rows` rows only.  Both operands: a zero in one alone would still give 0 * NaN = NaN.  The two consumer warpgroups
// (256 threads) share the work, order their generic-proxy stores before the wgmma's async-proxy reads, and meet on
// named barrier 2 (the fused kernels' communication warps use barrier 1), so neither reads a row the other has not
// yet cleared.  A 128-byte swizzled row holds exactly one k-row of a box, so the swizzle does not matter here.
template <int BN>
__device__ __forceinline__ void zero_stage_rows(uint8_t* stage_base, int rows) {
  constexpr int kBoxes = Tile<BN>::kStageBytes / kBoxBytesMN;
  // consumer thread t clears 16-byte piece t % 8 of rows rows + t / 8, rows + t / 8 + 32 .. of every box
  const int t = static_cast<int>(threadIdx.x) - 128;
  for (int r = rows + (t >> 3); r < BK; r += kConsumerWarps * 32 / 8) {
    uint8_t* p = stage_base + r * 128 + (t & 7) * 16;
#pragma unroll
    for (int box = 0; box < kBoxes; ++box) *reinterpret_cast<uint4*>(p + box * kBoxBytesMN) = make_uint4(0, 0, 0, 0);
  }
  tc::fence_proxy_async();
  asm volatile("bar.sync 2, %0;" ::"n"(kConsumerWarps * 32) : "memory");
}

// Consumer warpgroup `wgi` (0/1): acc = its 64 rows of the tile, summed over k_blocks stages.
// The stage of k-block kb is handed back to the producer once the wgmma of kb + 1 has been
// issued and those of kb have retired (wait_group 1), so one k-block of MMAs is always queued.
// TAIL_ROWS (both operands MN-major): the last k-block contracts over its first tail_rows rows only
// (zero_stage_rows), the grouped wgrad's last k-block of a group.
template <bool A_MN, bool B_MN, int BN, bool TAIL_ROWS = false>
__device__ __forceinline__ void mma_tile(float (&acc)[BN / 2], uint8_t* smem, Pipe* p, int& stage, uint32_t& phase,
                                         int k_blocks, int wgi, int tail_rows = BK) {
  static_assert(!TAIL_ROWS || (A_MN && B_MN), "row masking needs MN-major boxes");
  const int lane = threadIdx.x & 31;
  int prev = -1;
  tc::fence_regs(acc);
  for (int kb = 0; kb < k_blocks; ++kb) {
    tc::mbar_wait(&p->full[stage], phase);
    if constexpr (TAIL_ROWS) {
      if (kb == k_blocks - 1 && tail_rows < BK) zero_stage_rows<BN>(smem + stage * Tile<BN>::kStageBytes, tail_rows);
    }
    const uint32_t sa = tc::smem_u32(smem + stage * Tile<BN>::kStageBytes);
    const uint32_t sb = sa + kABytes;
    // this warpgroup's 64 rows of A: one MN-major box, or 64 K-major rows of 128 bytes
    const uint32_t a0 = sa + static_cast<uint32_t>(wgi) * (A_MN ? kBoxBytesMN : 64 * 128);
    tc::wgmma_fence();
#pragma unroll
    for (int k = 0; k < BK / 16; ++k) {
      // next 16 k: 32 bytes along a K-major row, or two 8-row atoms (2048 bytes) of an MN-major box
      const uint64_t da = tc::make_desc_sw128(a0 + (A_MN ? k * 2048 : k * 32), A_MN ? kBoxBytesMN : 16);
      const uint64_t db = tc::make_desc_sw128(sb + (B_MN ? k * 2048 : k * 32), B_MN ? kBoxBytesMN : 16);
      if constexpr (BN == 256)
        tc::wgmma_m64n256k16_bf16<A_MN ? 1 : 0, B_MN ? 1 : 0>(acc, da, db, (kb | k) ? 1u : 0u);
      else
        tc::wgmma_m64n128k16_bf16<A_MN ? 1 : 0, B_MN ? 1 : 0>(acc, da, db, (kb | k) ? 1u : 0u);
    }
    tc::wgmma_commit();
    tc::wgmma_wait<1>();
    if (prev >= 0 && lane == 0) tc::mbar_arrive(&p->empty[prev]);
    prev = stage;
    advance<BN>(stage, phase);
  }
  tc::wgmma_wait<0>();
  tc::fence_regs(acc);
  if (prev >= 0 && lane == 0) tc::mbar_arrive(&p->empty[prev]);
}

// fp8 sibling of mma_tile for 128 x 128 tiles with both operands K-major.  A 128-byte stage row holds 128 fp8
// values, so one stage is a k-block of 128 and each of its four k32 steps advances the descriptors by 32 bytes,
// exactly as the bf16 k16 steps do: the ring, the swizzle and the producer are the bf16 ones.
// Split accumulation: each k-block is summed by the tensor core into `blk` (a fresh accumulator) and then added
// into `acc` in fp32, so the tensor core's fp8 accumulation never spans more than 128 products.  The block must
// have retired before it is added, so no k-block stays queued behind the adds.
template <bool A_E5M2>
__device__ __forceinline__ void mma_tile_fp8(float (&acc)[64], uint8_t* smem, Pipe* p, int& stage, uint32_t& phase,
                                             int k_blocks, int wgi) {
  const int lane = threadIdx.x & 31;
  float blk[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) acc[i] = 0.f;
  for (int kb = 0; kb < k_blocks; ++kb) {
    tc::mbar_wait(&p->full[stage], phase);
    const uint32_t sa = tc::smem_u32(smem + stage * Tile<128>::kStageBytes);
    const uint32_t sb = sa + kABytes;
    const uint32_t a0 = sa + static_cast<uint32_t>(wgi) * (64 * 128);
    tc::fence_regs(blk);
    tc::wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k)
      tc::wgmma_m64n128k32_fp8<A_E5M2>(blk, tc::make_desc_sw128(a0 + k * 32, 16), tc::make_desc_sw128(sb + k * 32, 16),
                                       k ? 1u : 0u);
    tc::wgmma_commit();
    tc::wgmma_wait<0>();
    tc::fence_regs(blk);
    if (lane == 0) tc::mbar_arrive(&p->empty[stage]);
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] += blk[i];
    advance<128>(stage, phase);
  }
}

// ---- grouped layout (DESIGN §4.4) --------------------------------------------------------------------------------
// E groups with device-resident row counts c_e share one [rows, .] operand: group e starts at row BM * pfx[e] with
// pfx[e] = sum_{j<e} ceil(c_j / BM), so no BM-row tile spans two groups.  Counts are clamped to [0, rows] and pfx to
// rows / BM: a group (or its part) past the last row has no rows, and nothing outside the operands is touched.
constexpr int kMaxGroups = 1024;
struct GroupTable {
  int pfx[kMaxGroups + 1];  // first m-block of each group; pfx[E] = m-blocks in use
  int end[kMaxGroups];      // one past the group's last valid row
};
// Bytes a grouped kernel adds to its dynamic shared memory (the table sits behind the ring's barriers).
constexpr int kGroupTableBytes = static_cast<int>(sizeof(GroupTable));
__device__ __forceinline__ GroupTable* group_table_of(Pipe* pipe) {
  return reinterpret_cast<GroupTable*>(reinterpret_cast<uint8_t*>(pipe) + 256);
}

// One thread builds the table; the kernel's first __syncthreads publishes it.
__device__ __forceinline__ void build_group_table(GroupTable* t, const int* counts, int E, int rows) {
  const int cap = rows / BM;
  int p = 0;
  t->pfx[0] = 0;
  for (int e = 0; e < E; ++e) {
    const int c = min(max(counts[e], 0), rows);
    const int start = p * BM;
    p = min(p + (c + BM - 1) / BM, cap);
    t->pfx[e + 1] = p;
    t->end[e] = min(start + c, rows);
  }
}

// The group whose m-blocks hold m_blk (m_blk < pfx[E]): the last e with pfx[e] <= m_blk, which skips empty groups.
__device__ __forceinline__ int group_of(const GroupTable* t, int E, int m_blk) {
  int lo = 0, hi = E - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (t->pfx[mid] <= m_blk) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

// Accumulator fragment of wgmma m64nN (fp32): thread (warp w of the warpgroup, lane l) holds, for
// j = 0 .. N/8 - 1, columns 8j + 2(l % 4) + {0, 1} of rows 16w + l / 4 (acc[4j], acc[4j+1]) and
// 16w + l / 4 + 8 (acc[4j+2], acc[4j+3]).
__device__ __forceinline__ int frag_row(int h) { return ((threadIdx.x >> 5) & 3) * 16 + ((threadIdx.x & 31) >> 2) + 8 * h; }
__device__ __forceinline__ int frag_col(int j) { return 8 * j + 2 * (threadIdx.x & 3); }

__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  return static_cast<uint32_t>(float_to_bf16_bits(lo)) | (static_cast<uint32_t>(float_to_bf16_bits(hi)) << 16);
}

// Cross-rank wait of the fused kernels: spins until *flag >= target (wrap-safe).  A peer that never
// publishes must end in an error, not in a hung GPU: on timeout the error word is set and the kernel traps.
__device__ __forceinline__ void bounded_wait_ge(const uint32_t* flag, uint32_t target, const SyncCtx& c) {
  if (static_cast<int32_t>(ld_acquire_sys_u32(flag) - target) >= 0) return;
  const unsigned long long t0 = globaltimer_ns();
  unsigned int spins = 0;
  while (static_cast<int32_t>(ld_acquire_sys_u32(flag) - target) < 0) {
    if ((++spins & 0x3ff) == 0 && globaltimer_ns() - t0 > c.timeout_ns) {
      *reinterpret_cast<volatile int*>(c.err_flag) = kErrTimeout;
      __threadfence_system();
      __trap();
    }
  }
}

}  // namespace wg
}  // namespace m4t
