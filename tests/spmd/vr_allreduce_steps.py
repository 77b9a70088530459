"""Every reducing (dtype, op) pair through the host backend's all-reduce, one-phase (below 256 KiB) and two-phase, with
and without the fused scale and accumulate operand.  Each rank saves its inputs and results to
<out_dir>/rank<r>.pt; tests/test_virtual_ranks_emulator_cpu.py compares them with the emulation of the GPU kernels,
which round at the same places."""
import os
import sys

import numpy as np
import torch

from common import comm

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import virtual_ranks_emulation as emu  # noqa: E402

import mpi4torch_b200 as m4t  # noqa: E402

P, RANK = comm.size, comm.rank
TWO_PHASE_BYTES = 256 * 1024  # cpu_backend.cpp: kTwoPhaseBytes


def main(out_dir):
    records = []
    for di, dtype in enumerate(emu.ALL_DTYPES):
        es = torch.empty(0, dtype=dtype).element_size()
        scale = 0.3 if dtype.is_floating_point else 0.75
        for oi, op in enumerate(emu.ops_for(dtype)):
            for n in (1, 7, 1001, TWO_PHASE_BYTES // es + 5):
                for variant in ("none", "scale", "scale+acc"):
                    # every rank draws every rank's inputs, so the draws do not depend on the rank
                    g = np.random.default_rng(1000 * di + 10 * oi + n % 7 + 3 * len(variant))
                    xs = [emu.make_input(dtype, n, g, rank=p) for p in range(P)]
                    acc = emu.make_input(dtype, n, g, rank=P)
                    x = xs[RANK]
                    if variant == "none":
                        out = comm.Allreduce(x, emu.OPS[op])
                    else:
                        out = comm.AllreduceFused(x, emu.OPS[op], scale, acc if variant == "scale+acc" else None)
                    records.append(dict(dtype=dtype, op=op, n=n, variant=variant, scale=scale, xs=xs, acc=acc, out=out,
                                        two_phase=n * es >= TWO_PHASE_BYTES))
    torch.save(records, os.path.join(out_dir, f"rank{RANK}.pt"))
    print(f"vr_allreduce_steps np={P} rank={RANK} records={len(records)} ok=True")


if __name__ == "__main__":
    main(sys.argv[1])
    m4t.COMM_WORLD.Barrier()
