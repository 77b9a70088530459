"""Pure-Python mirrors of the index arithmetic of the fused backward kernel
(csrc/kernels/wgrad_wgmma.cu).  They cannot check the memory model, but they do
check what is easy to get wrong in a persistent, role-split kernel: that the work
distribution covers every element exactly once and that the counters reach exactly the
targets the host computes (csrc/runtime/cuda_backend.cpp::fused_wgrad_update)."""
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
