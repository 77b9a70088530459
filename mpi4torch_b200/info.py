"""``python -m mpi4torch_b200.info`` - what is installed, how it was built, which transport a job would use
and every environment knob with its default (the role of ``ompi_info`` / ``mpichversion`` next to the reference).

Run it bare for the build facts and the knob table.  With ``--world`` it also initialises ``COMM_WORLD`` of the job
it is started in (one process, or every rank of a launcher / torchrun job; rank 0 prints) and reports the transport
the ranks negotiated.

``KNOBS`` is the single documented list of environment variables; ``tests/test_unit.py`` checks it against the
variables the sources actually read, so it cannot drift.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
from typing import Dict, List, Tuple

# name -> (default, meaning)
KNOBS: Dict[str, Tuple[str, str]] = {
    # ---- transport selection / memory
    "M4T_CUDA": ("1", "0 keeps the CUDA backend off even when a GPU is visible (CPU tensors only)"),
    "M4T_NVLS": ("1", "0 disables NVSwitch multicast (multimem) even when the driver offers it"),
    "M4T_VMM": ("1", "0 skips the VMM symmetric heap and falls back to cudaIpc mappings"),
    "M4T_NVLS_MIN_RANKS": ("4", "fewest ranks for which reductions go through the switch instead of peer loads"),
    "M4T_STAGE_MB": ("2176", "size of ONE of the two staging halves of the world communicator's symmetric heap"),
    "M4T_SYMM_MB": ("512", "user arena of the symmetric heap (symmetric_empty, fused-kernel buffers)"),
    "M4T_SUB_STAGE_MB": ("256", "staging half of communicators created by Split"),
    "M4T_SUB_SYMM_MB": ("0", "user arena of communicators created by Split"),
    "M4T_ZERO_COPY_IN": ("0", "1 lets Allreduce read symmetric input tensors in place (no stage-in copy)"),
    "M4T_SLAB_CHUNK_BYTES": ("0", "lowers the per-call staging limit of Gather/Scatter/Allgather/Alltoall/"
                                  "Reduce_scatter (tests drive the piece-wise paths with it); 0 = staging half"),
    # ---- allreduce
    "M4T_ALLREDUCE_ALGO": ("0", "force an algorithm: 1 one-shot, 2 two-shot (peer loads), 3 NVLS; 0 = by size"),
    "M4T_ONESHOT_MAX_KB": ("2048", "largest message of the one-shot algorithm"),
    "M4T_ONESHOT_BLOCKS": ("32", "CTAs of the one-shot kernel"),
    "M4T_AR_BLOCKS": ("132", "CTAs of the two-shot / NVLS kernels"),
    "M4T_AR_PIPE": ("1", "0 disables the pipelined NVLS kernel for large messages"),
    "M4T_PIPE_MIN_MB": ("512", "smallest message of the pipelined NVLS kernel"),
    "M4T_CHUNK_KB": ("0", "cap on the bytes one allreduce launch moves (0 = half a staging half)"),
    "M4T_AR_DEBUG_SKIP": ("0", "timing experiments: bit mask of allreduce phases to skip (wrong results)"),
    # ---- slab collectives / p2p
    "M4T_SLAB_BLOCKS": ("128", "CTAs of the slab pull / reduce kernels"),
    "M4T_AG_PUSH": ("-1", "Allgather by multicast push: 1 always, 0 never, -1 when the shard is <= 32 MiB"),
    "M4T_P2P_BLOCKS": ("32", "CTAs of the kernel-driven p2p copy"),
    "M4T_P2P_SLOTS": ("max(16, min(64, 512/size))", "slots of each pair's ring"),
    "M4T_P2P_SLOT_KB": ("1024", "bytes per ring slot"),
    "M4T_P2P_PUSH": ("0", "1 places each pair's ring in the receiver's heap (sender pushes)"),
    "M4T_P2P_CE_MIN_KB": ("2048", "messages from this size move on the copy engines; negative = never"),
    # ---- tensor-core kernels
    "M4T_FUSED_LINEAR": ("1", "0 disables the fused Allreduce->GEMM forward"),
    "M4T_FUSED_WGRAD": ("1", "0 disables the fused backward (wgrad -> reduce-scatter -> SGD -> multicast)"),
    "M4T_WGRAD_KSPLIT": ("2", "batch split of the last partial wave of the fused backward"),
    "M4T_WGRAD_DEBUG": ("0", "timing experiments: bit mask of fused-backward phases to skip (wrong results)"),
    "M4T_FUSED_DEBUG": ("0", "timing experiments: bit mask of fused-forward phases to skip (wrong results)"),
    # ---- waits, diagnostics
    "M4T_TIMEOUT_S": ("300", "bound of every host-side wait (a mismatched collective raises instead of hanging)"),
    "M4T_DEVICE_TIMEOUT_S": ("20", "bound of every device-side flag wait"),
    "M4T_EXIT_TIMEOUT_S": ("10", "how long finalisation waits for the peers"),
    "M4T_DEBUG": ("0", "1 prints one line per operation"),
    "M4T_DEBUG_SEGV": ("0", "1 installs a SIGSEGV handler that prints a native backtrace"),
    "M4T_NVTX": ("1", "0 drops the per-op NVTX ranges"),
    "M4T_NUMA_BIND": ("1", "0 leaves CPU affinity / memory policy alone (utils.bind_to_gpu_numa)"),
    # ---- jobs that span nodes (TCP mesh)
    "M4T_NET": ("", "1 forces the TCP mesh on one node (tests), 0 forbids it; default: when LOCAL_WORLD_SIZE < WORLD_SIZE"),
    "M4T_NET_IFADDR": ("", "address other nodes should use to reach this rank (default: the one that routes to MASTER_ADDR)"),
    "M4T_NET_LOCAL_SIZE": ("", "ranks per node for the hierarchical Allreduce (default LOCAL_WORLD_SIZE; tests simulate nodes with it)"),
    "M4T_STORE_HOSTED": ("0", "1 = a launcher hosts the rendezvous store at MASTER_ADDR:MASTER_PORT (else rank 0 does)"),
    # ---- rendezvous (normally set by the launcher or torchrun)
    "M4T_RANK": ("", "rank when RANK is not set"),
    "M4T_WORLD_SIZE": ("", "world size when WORLD_SIZE is not set"),
    "M4T_JOB_ID": ("", "name of the control segment (default: derived from MASTER_PORT)"),
    # ---- build
    "M4T_NO_BUILD": ("0", "1 loads the existing extension without checking its source stamp"),
    "M4T_BUILD_VERBOSE": ("0", "1 shows the compiler commands"),
    "M4T_LIB_DIR": ("", "directory of the built extension (default: mpi4torch_b200/_lib)"),
    "M4T_EXTRA_CXXFLAGS": ("", "appended to the host compiler flags (sanitizer builds)"),
    "M4T_EXTRA_LDFLAGS": ("", "appended to the link flags"),
    "M4T_KEEP_CXX": ("0", "1 keeps $CXX instead of /usr/bin/g++"),
}


def build_facts() -> Dict[str, object]:
    import torch

    from . import _build

    so = _build.so_path()
    facts: Dict[str, object] = {
        "package": os.path.dirname(os.path.abspath(__file__)),
        "torch": torch.__version__,
        "python": sys.version.split()[0],
        "extension": str(so),
        "extension_exists": so.exists(),
        "extension_fresh": bool(so.exists() and _build.is_fresh()),
        "target": "sm_90a (compute_90a), no other architecture is built",
        "cuda_visible": bool(torch.cuda.is_available()),
        "gpus": torch.cuda.device_count() if torch.cuda.is_available() else 0,
    }
    try:
        with open(os.path.join(os.path.dirname(facts["package"]), "version.txt")) as f:
            facts["version"] = f.read().strip()
    except OSError:
        facts["version"] = "unknown"
    return facts


def world_facts() -> Dict[str, object]:
    """Initialises COMM_WORLD (collective when started under the launcher) and reports the negotiated transport."""
    import mpi4torch_b200 as m4t

    comm = m4t.COMM_WORLD
    return {
        "rank": comm.rank,
        "size": comm.size,
        "cuda_backend": bool(m4t.cuda_backend_ready()),
        "nvls": bool(m4t.has_nvls()) if m4t.cuda_backend_ready() else False,
        "heap_mode": m4t.heap_mode() if m4t.cuda_backend_ready() else "none",
        "transport": comm.describe(),
    }


def knob_rows() -> List[Tuple[str, str, str, str]]:
    return [(name, os.environ.get(name, ""), default, meaning) for name, (default, meaning) in KNOBS.items()]


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(prog="python -m mpi4torch_b200.info", description=__doc__.split("\n\n")[0])
    ap.add_argument("--world", action="store_true", help="initialise COMM_WORLD and report the transport")
    ap.add_argument("--json", action="store_true", help="machine-readable output")
    args = ap.parse_args(argv)
    facts = build_facts()
    world = world_facts() if args.world else None
    if world is not None and world["rank"] != 0:
        return 0
    if args.json:
        print(json.dumps({"build": facts, "world": world,
                          "knobs": {n: {"set": s, "default": d, "meaning": m} for n, s, d, m in knob_rows()}}))
        return 0
    print("mpi4torch_b200", facts["version"])
    for k, v in facts.items():
        if k != "version":
            print(f"  {k:18s} {v}")
    if world is not None:
        print("world")
        for k, v in world.items():
            print(f"  {k:18s} {v}")
    print("environment knobs (set value | default | meaning)")
    for name, cur, default, meaning in knob_rows():
        print(f"  {name:22s} {cur or '-':>8s} | {default:>10s} | {meaning}")
    return 0


if __name__ == "__main__":
    sys.exit(main())
