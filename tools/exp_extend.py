#!/usr/bin/env python
"""Extend-mode batches (-m 2, and -m 2 -z 100) on the two engines of abpoa_gpu_msa_batch, next to global (-m 0) runs.

The workload is the headline shape (convex_10k: 50 reads x 10 kbp per group, 5 % error, convex gaps).  Runs one batch per
mode (-m 0, -m 2, -m 2 -z 100; consensus, -r 0), once on the device-resident chain engine and once on the launch engine
(the no_chain flag: host graph fusion and a host Kahn pass between kernel launches), alternating, and reports per run the
wall time, chain_device_ms, the fuse workers' time per group (chain_fuse_ms / groups: in extend mode it includes the
serial Kahn walk of chain_kahn_order), chain_groups / chain_fallback_groups and the bytes in each direction.  It compares
the two engines' records field by field (consensus, coverage, MSA rows, DP cells, aligned counts, and every read's score,
CIGAR length and CIGAR hash) and prints the card's name, power limit and max SM clock.

    python tools/exp_extend.py --groups 200 --reps 1 [--engines chain] [--modes m2,m2z100]
"""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from abpoa_b200 import capi, synth  # noqa: E402
from abpoa_b200.aligner import PoaConfig, make_para  # noqa: E402
from abpoa_b200.batch import BatchEngine, PackedGroups  # noqa: E402

N_READS, LENGTH, ERR, SEED = 50, 10_000, 0.05, 7700
MODES = {"m0": dict(), "m2": dict(align_mode=capi.ABPOA_EXTEND_MODE), "m2z100": dict(align_mode=capi.ABPOA_EXTEND_MODE, zdrop=100)}


def card() -> str:
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        if q.returncode == 0 and q.stdout.strip():
            return q.stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError):
        pass
    return "unknown card (nvidia-smi not available)"


def same(a, b) -> str | None:
    """None if the two result lists are identical, else what differs first."""
    if len(a) != len(b):
        return f"{len(a)} vs {len(b)} groups"
    for gi, (x, y) in enumerate(zip(a, b)):
        if x.dp_cells != y.dp_cells or x.n_aligned != y.n_aligned:
            return f"group {gi}: DP cells / aligned count"
        if len(x.msa) != len(y.msa) or any(not np.array_equal(p, q) for p, q in zip(x.msa, y.msa)):
            return f"group {gi}: MSA rows"
        if len(x.cons) != len(y.cons) or any(not np.array_equal(p, q) for p, q in zip(x.cons, y.cons)):
            return f"group {gi}: consensus"
        if any(not np.array_equal(p, q) for p, q in zip(x.cov, y.cov)):
            return f"group {gi}: coverage"
        for f in ("read_best_score", "read_n_cigar", "read_cigar_hash"):
            if not np.array_equal(getattr(x, f)[1:], getattr(y, f)[1:]):
                return f"group {gi}: {f}"
    return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--groups", type=int, default=200)
    ap.add_argument("--reps", type=int, default=1)
    ap.add_argument("--engines", choices=["both", "chain", "launch"], default="both")
    ap.add_argument("--modes", default="m0,m2,m2z100", help="comma-separated subset of " + ",".join(MODES))
    args = ap.parse_args()
    print(f"card: {card()}", flush=True)
    t0 = time.time()
    groups = [synth.make_group(SEED + g, N_READS, LENGTH, ERR) for g in range(args.groups)]
    packed = PackedGroups(groups)
    print(f"convex_10k: {args.groups} groups x {N_READS} reads x {LENGTH} bp (generated in {time.time() - t0:.1f} s)", flush=True)
    lib = capi.product()
    warm = PackedGroups(groups[:2])
    for out_name in args.modes.split(","):
        abpt = make_para(lib, PoaConfig(**MODES[out_name]))
        try:
            with BatchEngine() as eng:
                for no_chain in (False, True):                          # warm-up: module load, pinned buffers, both engines
                    eng.run_packed(abpt, warm, record_reads=True, no_chain=no_chain)
                last = {}
                for rep in range(args.reps):
                    for engine, no_chain in (("chain", False), ("launch", True)):
                        if args.engines not in ("both", engine):
                            continue
                        eng.reset_stats()
                        t = time.time()
                        res = eng.run_packed(abpt, packed, record_reads=True, no_chain=no_chain)
                        wall = time.time() - t
                        st = eng.stats()
                        last[engine] = res
                        print(json.dumps({"mode": out_name, "engine": engine, "rep": rep, "wall_s": round(wall, 3),
                                          "chain_device_ms": round(st["chain_device_ms"], 1),
                                          "fuse_ms_per_group": round(st["chain_fuse_ms"] / max(st["chain_groups"], 1), 2),
                                          "dp_ms_per_group": round(st["chain_dp_ms"] / max(st["chain_groups"], 1), 2),
                                          "chain_groups": st["chain_groups"],
                                          "chain_fallback_groups": st["chain_fallback_groups"], "h2d_bytes": st["h2d_bytes"],
                                          "d2h_bytes": st["d2h_bytes"]}), flush=True)
                if len(last) < 2:
                    continue
                diff = same(last["chain"], last["launch"])
                print(f"{out_name}: chain and launch engine records {'identical' if diff is None else 'DIFFER: ' + diff}", flush=True)
                if diff is not None:
                    sys.exit(1)
        finally:
            lib.abpoa_free_para(abpt)


if __name__ == "__main__":
    main()
