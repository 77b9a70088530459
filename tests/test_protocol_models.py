"""Pure-Python mirrors of the index arithmetic of the fused backward kernel
(csrc/kernels/wgrad_wgmma.cu) and of the smem ring shared by the wgmma kernels
(csrc/kernels/wgmma_pipeline.cuh).  They cannot check the memory model, but they do
check what is easy to get wrong in a persistent, role-split kernel: that the work
distribution covers every element exactly once, that the counters reach exactly the
targets the host computes (csrc/runtime/cuda_backend.cpp::fused_wgrad_update), and that
every mbarrier wait is on a phase that some arrival completes."""
import itertools

import numpy as np
import pytest

BM, BN = 128, 128                     # rows / cols of a tile of G (one CTA)
K_COMM_WARPS, K_U, K_ROW_SPLIT = 4, 4, 2
K_PAIRS = BM // K_ROW_SPLIT // 2      # row pairs of one owner work item (half a warp per 256-byte row)
SIGNALS_PER_UNIT = 8                  # 2 consumer warpgroups x 4 warps
WARP_ROWS = 16                        # rows of the wgmma accumulator fragment held by one warp


def units_of_cta(cta, num_ctas, num_units):
    return range(cta, num_units, num_ctas)


def make_sched(num_tiles, num_ctas, ksplit):
    """make_sched / unit_to_tile of the kernel: whole waves of tiles run over the full batch, only the tiles
    of the last partial wave are split in `ksplit` batch slices."""
    whole = (num_tiles // num_ctas) * num_ctas if ksplit > 1 else num_tiles
    return whole, ksplit, whole + (num_tiles - whole) * ksplit


def unit_to_tile(sched, u):
    whole, split, _ = sched
    if u < whole:
        return u, 0, 1
    j = u - whole
    return whole + j // split, j % split, split


@pytest.mark.parametrize("N,K,P,num_ctas,ksplit", [(1024, 512, 4, 3, 2), (512, 256, 8, 5, 2), (768, 768, 2, 7, 1),
                                                  (4096, 4096, 8, 74, 2), (4096, 4096, 8, 132, 2)])
def test_fused_wgrad_work_distribution(N, K, P, num_ctas, ksplit):
    n_tiles, k_tiles = N // BM, K // BN
    num_tiles = n_tiles * k_tiles
    sched = make_sched(num_tiles, num_ctas, ksplit)
    num_units = sched[2]
    small = N * K <= 1 << 20

    # --- GEMM epilogue: every (split, row, col) of the staging buffers written once; tile counters ---
    staged = np.zeros((ksplit, N, K), dtype=np.int8) if small else None
    signals = np.zeros(num_tiles, dtype=np.int64)  # per rank; the owner sums over P ranks
    parts_of = np.zeros(num_tiles, dtype=np.int64)
    kb_covered = np.zeros(num_tiles, dtype=np.int64)  # batch blocks contracted per tile (in units of 1/ksplit)
    for cta in range(num_ctas):
        for u in units_of_cta(cta, num_ctas, num_units):
            t, h, parts = unit_to_tile(sched, u)
            assert 0 <= t < num_tiles and 0 <= h < parts
            parts_of[t] = parts
            kb_covered[t] += ksplit // parts
            n_blk, k_blk = divmod(t, k_tiles)
            for wgi, w in itertools.product(range(2), range(4)):
                if small:
                    r0 = n_blk * BM + wgi * 64 + w * WARP_ROWS
                    staged[h, r0:r0 + WARP_ROWS, k_blk * BN:(k_blk + 1) * BN] += 1
                signals[t] += 1
    assert (kb_covered == ksplit).all()  # every tile contracts the whole batch exactly once
    if small:
        for t in range(num_tiles):  # buffer h of tile t is written once iff the tile has a slice h
            n_blk, k_blk = divmod(t, k_tiles)
            blk = staged[:, n_blk * BM:(n_blk + 1) * BM, k_blk * BN:(k_blk + 1) * BN]
            for h in range(ksplit):
                assert (blk[h] == (1 if h < parts_of[t] else 0)).all()
    # host: tile_target = signals_per_unit * size per call; the kernel multiplies by the tile's number of units
    assert (signals * P == SIGNALS_PER_UNIT * P * parts_of).all()

    # --- owner side: every element of W updated by exactly one (rank, cta, warp, lane, trip) ---
    updated = np.zeros((N, K), dtype=np.int8) if small else None
    items_total = 0
    for r in range(P):
        owned = (num_tiles - r + P - 1) // P if r < num_tiles else 0
        for cta in range(num_ctas):
            for w_item in range(cta, owned * K_ROW_SPLIT, num_ctas):
                j, sl = divmod(w_item, K_ROW_SPLIT)
                t = r + j * P
                assert t < num_tiles and t % P == r  # the epilogue signals rank t % P
                items_total += 1
                if not small:
                    continue
                n_blk, k_blk = divmod(t, k_tiles)
                for cw in range(K_COMM_WARPS):
                    pairs = []
                    for pair0 in range(cw, K_PAIRS, K_COMM_WARPS * K_U):
                        pairs += [pair0 + u * K_COMM_WARPS for u in range(K_U) if pair0 + u * K_COMM_WARPS < K_PAIRS]
                    for pair, half in itertools.product(pairs, range(2)):  # lane >> 4 picks the row of the pair
                        g = n_blk * BM + sl * 2 * K_PAIRS + 2 * pair + half
                        updated[g, k_blk * BN:(k_blk + 1) * BN] += 1  # 16 lanes x 8 bf16 = 128 columns
    assert items_total == num_tiles * K_ROW_SPLIT
    if small:
        assert (updated == 1).all()

    # --- completion counter: every CTA of every rank reports once per call ---
    grid = num_ctas
    assert P * grid == P * num_ctas  # host: done_target = calls * size * fused_gemm_grid


def test_unit_schedule_fills_the_last_wave():
    # 256 tiles on 74 CTAs = 3 whole waves + 34 tiles; those are split in two batch halves
    # (68 units <= 74 CTAs), so the kernel takes 3.5 tile times instead of 4 and only 34 tiles have two partials
    num_ctas, ksplit, num_tiles = 74, 2, 256
    sched = make_sched(num_tiles, num_ctas, ksplit)
    assert sched == (222, 2, 290)
    cost = [0.0] * num_ctas
    for cta in range(num_ctas):
        for u in units_of_cta(cta, num_ctas, sched[2]):
            cost[cta] += 1.0 / unit_to_tile(sched, u)[2]
    assert max(cost) == 3.5
    # both halves of a split tile run in the same (last) wave on neighbouring CTAs
    for t in range(sched[0], num_tiles):
        u0 = sched[0] + 2 * (t - sched[0])
        assert u0 // num_ctas == (u0 + 1) // num_ctas == 3


def _swizzle128(byte_off: int) -> int:
    """TMA SWIZZLE_128B == cute Swizzle<3,4,3>: XOR address bits [4,7) with bits [7,10)."""
    return byte_off ^ (((byte_off >> 7) & 7) << 4)


def test_mn_major_descriptor_addresses_what_tma_wrote():
    """wgrad operand tile: TMA boxes of {64 contiguous elements, BK rows} with SWIZZLE_128B, read by
    wgmma through an MN-major SWIZZLE_128B descriptor with LBO = one box, SBO = 1024 B and a
    start-address advance of 2048 B per k16 step (make_desc_sw128, wg::mma_tile).
    The canonical MN-major layout (cute/atom/mma_traits_sm90_gmma.hpp): in 16-byte units
    ((8,n),(8,k)) : ((1,LBO),(8,SBO)), then Swizzle<3,4,3> on the byte address."""
    BK, CHUNK, ES = 64, 64, 2
    box_bytes = CHUNK * BK * ES            # 8192
    lbo, sbo = box_bytes, 1024
    mn_extent = 128                        # m/n extent of the operand tile of one CTA
    # where TMA puts element (mn, k): box c = mn // 64 starts at c * box_bytes; inside a box row k is
    # 128 bytes long and the whole box is swizzled relative to its 1024-aligned base
    def tma_addr(mn, k):
        c, j = divmod(mn, CHUNK)
        return c * box_bytes + _swizzle128(k * 128 + j * ES)

    # where the MMA with descriptor start address `start` looks for element (mn, k_local) of its
    # 16-deep slice: canonical layout + swizzle of the absolute (1024-aligned) address
    def mma_addr(start, mn, k_local):
        e, a, nn = mn % 8, (mn // 8) % 8, mn // 64
        off = e * ES + a * 16 + nn * lbo + (k_local % 8) * 128 + (k_local // 8) * sbo
        return _swizzle128(start + off)

    for kstep in range(BK // 16):
        start = kstep * 2048               # start-address advance of the issue loop: two 8-row swizzle atoms
        for mn in range(mn_extent):
            for k_local in range(16):
                assert mma_addr(start, mn, k_local) == tma_addr(mn, kstep * 16 + k_local), (kstep, mn, k_local)


def test_k_major_descriptor_addresses_what_tma_wrote():
    """Same check for the K-major operands (make_desc_sw128): TMA box {64 k, rows},
    descriptor SBO = 1024 B (8 rows), start-address advance of 32 B per k16 step inside the
    128-byte swizzle span.  Canonical K-major layout: ((8,m),(T,2)) : ((8T,SBO),(1,T)) elements."""
    ES, rows = 2, 128

    def tma_addr(r, k):
        return _swizzle128(r * 128 + k * ES)

    def mma_addr(start, r, k_local):
        off = (r % 8) * 128 + (r // 8) * 1024 + k_local * ES
        return _swizzle128(start + off)  # the hardware swizzles the final address

    for kstep in range(4):
        start = kstep * 32
        for r in range(rows):
            for k_local in range(16):
                assert mma_addr(start, r, k_local) == tma_addr(r, kstep * 16 + k_local)


@pytest.mark.parametrize("nslots,send_blocks,recv_blocks,messages", [(4, 3, 2, [5, 1, 9]), (16, 32, 32, [64, 3]), (2, 1, 5, [7])])
def test_p2p_slot_ring_protocol_never_overwrites_unread_data(nslots, send_blocks, recv_blocks, messages):
    """csrc/kernels/p2p.cu: block b of the send kernel takes chunks b, b+G, ... of a message; chunk c
    (global index) lives in slot c % nslots; head[slot] = c+1 publishes it, tail[slot] = c+1 frees it.
    Random interleaving of all blocks of both kernels (several back-to-back messages): no slot is
    overwritten before it was read, every chunk is read exactly once with the right content."""
    import random

    rng = random.Random(nslots * 1000 + send_blocks * 10 + recv_blocks)
    head, tail = [0] * nslots, [0] * nslots
    slot_content = [None] * nslots
    received = {}
    first = 0
    agents = []  # [kind, message-local chunk list iterator state...]
    for n in messages:  # kernels of consecutive messages are stream-ordered per side, modelled by per-side queues
        agents.append(("msg", first, n))
        first += n
    send_queue = [(f, n) for _, f, n in agents]
    recv_queue = list(send_queue)

    def make_blocks(first_chunk, n, nblocks):
        g = min(nblocks, n)
        return [[first_chunk + k for k in range(b, n, g)] for b in range(g)]

    send_active, recv_active = [], []
    steps = 0
    while send_queue or recv_queue or send_active or recv_active:
        steps += 1
        assert steps < 200000, "protocol model deadlocked"
        if not send_active and send_queue:
            f, n = send_queue.pop(0)
            send_active = make_blocks(f, n, send_blocks)
        if not recv_active and recv_queue:
            f, n = recv_queue.pop(0)
            recv_active = make_blocks(f, n, recv_blocks)
        side = rng.choice(["s", "r"])
        blocks = send_active if side == "s" else recv_active
        blocks[:] = [b for b in blocks if b]
        if not blocks:
            continue
        b = rng.choice(blocks)
        c = b[0]
        s = c % nslots
        if side == "s":
            if c >= nslots and tail[s] < c - nslots + 1:
                continue  # wait_flag_ge(tail[s], c - nslots + 1)
            assert slot_content[s] is None or slot_content[s] in received, f"chunk {slot_content[s]} overwritten unread"
            slot_content[s] = c
            head[s] = c + 1  # st.release after the copy
            b.pop(0)
        else:
            if head[s] < c + 1:
                continue  # wait_flag_ge(head[s], c + 1)
            assert slot_content[s] == c, f"slot {s} holds {slot_content[s]}, expected {c}"
            assert c not in received
            received[c] = True
            tail[s] = c + 1
            b.pop(0)
    assert sorted(received) == list(range(sum(messages)))


def _ce_groups(nslots, slot_bytes, nbytes, first_chunk):
    """for_each_group of csrc/kernels/p2p.cu (copy-engine path): groups of consecutive chunks that neither wrap the
    ring nor exceed half of it nor 32 slots.  Returns (cidx0, s0, g, off, length) tuples."""
    nchunks = 1 if nbytes <= 0 else (nbytes + slot_bytes - 1) // slot_bytes
    gmax = max(1, min(nslots // 2, 32))
    out, k0 = [], 0
    while k0 < nchunks:
        cidx0 = first_chunk + k0
        s0 = cidx0 % nslots
        g = min(gmax, nchunks - k0, nslots - s0)
        off = k0 * slot_bytes
        out.append((cidx0, s0, g, off, max(0, min(g * slot_bytes, nbytes - off))))
        k0 += g
    return out


@pytest.mark.parametrize("nslots", [2, 16, 64])
@pytest.mark.parametrize("messages", [[5], [1, 70, 3], [64, 64, 1, 129], [0, 7, 0, 33]])
def test_p2p_copy_engine_groups_and_flags(nslots, messages):
    """Copy-engine p2p path: the sender's DMA fills a group of slots after waiting for their tail flags, then posts the
    head flags; the receiver's DMA drains the group after waiting for the head flags, then posts the tail flags.
    Kernel-path and copy-engine messages may alternate on one ring because both use the same chunk numbering.
    Random interleaving of the two stream-ordered sides: nothing is overwritten unread, every byte range arrives
    once, groups never wrap the ring."""
    import random

    slot = 4  # bytes per slot in the model
    rng = random.Random(nslots * 7 + len(messages))
    head, tail = [0] * nslots, [0] * nslots
    content = [None] * nslots  # (message, chunk) held by a slot
    first = 0
    send_ops, recv_ops = [], []  # stream-ordered operation lists per side
    for m, nchunks_or_bytes in enumerate(messages):
        nbytes = nchunks_or_bytes * slot - (1 if nchunks_or_bytes > 1 else 0)  # ragged last chunk
        nbytes = max(nbytes, 0)
        groups = _ce_groups(nslots, slot, nbytes, first)
        covered = 0
        for cidx0, s0, g, off, length in groups:
            assert s0 + g <= nslots and 1 <= g <= max(1, min(nslots // 2, 32))
            assert off == covered
            covered += length
            send_ops.append((m, cidx0, s0, g))
            recv_ops.append((m, cidx0, s0, g))
        assert covered == nbytes
        first += 1 if nbytes <= 0 else (nbytes + slot - 1) // slot
    received = []
    si = ri = steps = 0
    while si < len(send_ops) or ri < len(recv_ops):
        steps += 1
        assert steps < 100000, "copy-engine protocol model deadlocked"
        if rng.random() < 0.5 and si < len(send_ops):
            m, cidx0, s0, g = send_ops[si]
            # p2p_flag_wait_kernel on the tail flags: slot free once chunk (c - nslots) was consumed
            if any(cidx0 + i >= nslots and tail[s0 + i] < cidx0 + i - nslots + 1 for i in range(g)):
                continue
            for i in range(g):
                assert content[s0 + i] is None or content[s0 + i] in received, "slot overwritten before it was read"
                content[s0 + i] = (m, cidx0 + i)
            for i in range(g):
                head[s0 + i] = cidx0 + i + 1  # p2p_flag_post_kernel after the DMA (stream order)
            si += 1
        elif ri < len(recv_ops):
            m, cidx0, s0, g = recv_ops[ri]
            if any(head[s0 + i] < cidx0 + i + 1 for i in range(g)):
                continue
            for i in range(g):
                assert content[s0 + i] == (m, cidx0 + i)
                received.append((m, cidx0 + i))
            for i in range(g):
                tail[s0 + i] = cidx0 + i + 1
            ri += 1
    assert len(received) == len(set(received)) == first


def test_push_epilogue_box_coordinates_cover_the_staging_area_once():
    """Peer-store mode of the fused backward (2-3 ranks): every consumer warp of every work unit stores its
    {16 rows x 128 columns} accumulator fragment into the owner's staging area for this source rank, laid out as
    [ksplit * N rows, K columns].  Mirror of the coordinates in wgrad_bf16_wgmma_kernel: each element of part h
    of tile t is written exactly once and only for the parts the schedule produces."""
    N, K, ksplit, num_ctas = 1024, 512, 2, 3
    n_tiles, k_tiles = N // BM, K // BN
    num_tiles = n_tiles * k_tiles
    sched = make_sched(num_tiles, num_ctas, ksplit)
    area = np.zeros((ksplit * N, K), dtype=np.int8)
    for u in range(sched[2]):
        t, h, parts = unit_to_tile(sched, u)
        n_blk, k_blk = divmod(t, k_tiles)
        for wgi, w in itertools.product(range(2), range(4)):
            row0 = h * N + n_blk * BM + wgi * 64 + w * WARP_ROWS
            col0 = k_blk * BN
            area[row0:row0 + WARP_ROWS, col0:col0 + BN] += 1
    for t in range(num_tiles):
        n_blk, k_blk = divmod(t, k_tiles)
        parts = 1 if t < sched[0] else sched[1]
        for h in range(ksplit):
            blk = area[h * N + n_blk * BM:h * N + (n_blk + 1) * BM, k_blk * BN:(k_blk + 1) * BN]
            assert (blk == (1 if h < parts else 0)).all(), (t, h)


# ---------------------------------------------------------------------------------------------------------------
# The smem ring of the single-GPU GEMM and wgrad kernels (csrc/kernels/wgmma_pipeline.cuh, gemm_wgmma.cu)
# ---------------------------------------------------------------------------------------------------------------
GEMM_BM, GEMM_BN, GEMM_BK = 128, 256, 64
RING_STAGES = 4        # Tile<256>::kStages
CONSUMER_WARPS = 8     # kConsumerWarps: lane 0 of every consumer warp arrives on `empty`


class _MBarrier:
    """An mbarrier: `count` arrivals complete the current phase.  try_wait.parity(p) succeeds once the phase of
    parity p has completed, i.e. while the current (incomplete) phase has the other parity."""

    def __init__(self, count):
        self.count, self.pending, self.completed = count, count, 0

    def arrive(self):
        assert self.pending > 0
        self.pending -= 1
        if self.pending == 0:
            self.completed += 1
            self.pending = self.count

    def passes(self, parity):
        return (self.completed & 1) != parity


def _advance(stage, phase):
    stage += 1
    return (0, phase ^ 1) if stage == RING_STAGES else (stage, phase)


def simulate_ring(tiles, seed):
    """One CTA: `tiles` is its list of (tile id, k_blocks) in loop order.  The producer runs load_stage for every
    k-block, each consumer warp runs mma_tile (it hands stage kb back only after the MMAs of kb + 1 are issued,
    and its last stage after the tile).  Agents interleave at random; every wait must be satisfiable.  Returns the
    producer's (stage, parity) sequence, each warp's sequence and the tiles each warp finished."""
    import random

    rng = random.Random(seed)
    full = [_MBarrier(1) for _ in range(RING_STAGES)]
    empty = [_MBarrier(CONSUMER_WARPS) for _ in range(RING_STAGES)]
    content = [None] * RING_STAGES
    held = [set() for _ in range(CONSUMER_WARPS)]  # stages a warp's in-flight MMAs still read
    fills = [0] * RING_STAGES
    prod_seq, warp_seq, done = [], [[] for _ in range(CONSUMER_WARPS)], [[] for _ in range(CONSUMER_WARPS)]

    def producer():
        stage, phase = 0, 0
        for t, kbs in tiles:
            for kb in range(kbs):
                f = fills[stage]
                yield empty[stage], phase ^ 1, f  # load_stage: wait until the f previous uses were released
                assert not any(stage in h for h in held), "TMA overwrote a stage an MMA still reads"
                content[stage] = (t, kb)
                fills[stage] += 1
                prod_seq.append((stage, phase))
                full[stage].arrive()  # arrive_expect_tx + the bytes landing
                stage, phase = _advance(stage, phase)

    def consumer(w):
        stage, phase, use = 0, 0, [0] * RING_STAGES
        for t, kbs in tiles:
            prev = None
            for kb in range(kbs):
                yield full[stage], phase, use[stage] + 1
                assert content[stage] == (t, kb), f"warp {w} read {content[stage]} for {(t, kb)}"
                use[stage] += 1
                held[w].add(stage)
                warp_seq[w].append((stage, phase))
                yield None  # the MMAs of this k-block are issued; wait_group 1 retires the previous ones
                if prev is not None:
                    held[w].discard(prev)
                    empty[prev].arrive()
                prev = stage
                stage, phase = _advance(stage, phase)
            held[w].discard(prev)  # wait_group 0, then the last stage goes back
            empty[prev].arrive()
            done[w].append(t)

    agents = [producer()] + [consumer(w) for w in range(CONSUMER_WARPS)]
    waits = [None] * len(agents)
    live = set(range(len(agents)))
    while live:
        ready = [a for a in live if waits[a] is None or waits[a][0].passes(waits[a][1])]
        assert ready, "deadlock: a wait on a parity that no arrival completes"
        a = rng.choice(ready)
        if waits[a] is not None:
            bar, _, phases = waits[a]
            assert bar.completed == phases, "a parity wait passed on the wrong phase (ABA)"
        try:
            waits[a] = next(agents[a])
        except StopIteration:
            live.discard(a)
            waits[a] = None
    return prod_seq, warp_seq, done


def gemm_cta_tiles(M, N, K, grid):
    """Tile loop of gemm_bf16_wgmma_kernel: CTA c takes tiles c, c + grid, ...; every tile has ceil(K / 64) k-blocks."""
    tiles = -(-M // GEMM_BM) * -(-N // GEMM_BN)
    kbs = -(-K // GEMM_BK)
    return [[(t, kbs) for t in range(c, tiles, grid)] for c in range(grid)], tiles


def ring_starts(cta_tiles):
    """(stage, parity) at which each tile of one CTA starts."""
    stage, phase, out = 0, 0, []
    for _, kbs in cta_tiles:
        out.append((stage, phase))
        for _ in range(kbs):
            stage, phase = _advance(stage, phase)
    return out


@pytest.mark.parametrize("M,N,K,grid", [(300, 520, 328, 3), (129, 264, 200, 2), (1, 8, 8, 1), (257, 520, 72, 5),
                                        (640, 512, 1000, 7), (256, 256, 64, 1)])
def test_gemm_ring_covers_every_tile_and_matches_parities(M, N, K, grid):
    per_cta, tiles = gemm_cta_tiles(M, N, K, min(grid, -(-M // GEMM_BM) * -(-N // GEMM_BN)))
    finished = []
    for c, cta_tiles in enumerate(per_cta):
        for seed in range(3):
            prod_seq, warp_seq, done = simulate_ring(cta_tiles, seed=c * 10 + seed)
            assert len(prod_seq) == sum(kbs for _, kbs in cta_tiles)
            for w in range(CONSUMER_WARPS):
                assert warp_seq[w] == prod_seq, "a consumer waited on a (stage, parity) out of the producer's order"
                assert done[w] == [t for t, _ in cta_tiles]
        finished += [t for t, _ in cta_tiles]
    assert sorted(finished) == list(range(tiles)), "a tile is computed twice or never"


def test_wgrad_ring_with_split_units():
    """wgrad_bf16_wgmma_kernel runs the same ring over work units of full or half batch depth (ksplit = 2)."""
    for cta_units in ([(0, 6), (5, 3), (9, 3)], [(1, 5), (2, 5), (3, 1)], [(4, 1)] * 9):
        prod_seq, warp_seq, _ = simulate_ring(cta_units, seed=len(cta_units))
        assert all(s == prod_seq for s in warp_seq)


def test_exact_arithmetic_sweep_starts_tiles_mid_ring():
    """Why the wave sweep of test_gpu_exact_arithmetic.py uses 3 and 5 k-blocks per tile: with them, every CTA that
    runs a second tile starts it at a non-zero stage of the 4-stage ring, and with 5 also on the flipped parity.
    The multi-wave shapes of the tolerance tests (4096 -> 64 and 1000 -> 16 k-blocks) always start at stage 0."""
    from test_gpu_exact_arithmetic import WAVE_KBLOCKS, gemm_wave_shape, wave_tile_counts, wgrad_wave_shape

    for S in (132, 114):  # H100 SXM, H100 PCIe
        for T in wave_tile_counts(S):
            for kbs in WAVE_KBLOCKS:
                M, N, K = gemm_wave_shape(T, kbs)
                per_cta, tiles = gemm_cta_tiles(M, N, K, min(T, S))
                assert tiles == T
                assert all(c for c in per_cta)  # the grid is capped at the tile count: no CTA idles
                assert sum(len(c) >= 2 for c in per_cta) == min(S, max(0, T - S))
                for c in per_cta:
                    starts = ring_starts(c)
                    assert starts[0] == (0, 0)
                    if len(c) >= 2:
                        assert starts[1][0] != 0
                        assert starts[1] == ((kbs % RING_STAGES), kbs // RING_STAGES)
                if T == 2 * S + 1:  # one CTA runs a third tile, the last wave of a single tile
                    assert sorted(len(c) for c in per_cta)[-2:] == [2, 3]
            for kbs in (1, 3, 5):
                Mb, Nw, Kw = wgrad_wave_shape(T, kbs)
                assert (Nw // 128) * -(-Kw // 256) == T and Mb == 64 * kbs
        for kbs in (16, 64):
            for c in gemm_cta_tiles(8192, 4096, 64 * kbs, S)[0]:
                assert all(s == (0, 0) for s in ring_starts(c))
    # the whole sweep replays without deadlock through the ring model (one CTA per distinct tile list)
    for kbs in WAVE_KBLOCKS:
        per_cta, _ = gemm_cta_tiles(*gemm_wave_shape(2 * 132 + 1, kbs), 132)
        for c in (per_cta[0], per_cta[-1]):
            prod_seq, warp_seq, _ = simulate_ring(c, seed=kbs)
            assert all(s == prod_seq for s in warp_seq)
