#!/usr/bin/env python
"""Quality-weighted (-Q) and path-scored (-G) batches on the two engines of abpoa_gpu_msa_batch.

Every read of every group gets deterministic quality-like weights (1..40 per base, seeded per group, as
tests/cases.py:case_weights draws them).  Runs one batch of a workload per mode (-Q -r 0, -Q -r 2, -G -r 0, -Q -G -r 0 by
default; -G -r 2 on request), once on the device-resident chain engine and once on the launch engine (the
ABPOA_GPU_NO_CHAIN flag), alternating, and reports per run the wall time, chain_device_ms, chain_groups /
chain_fallback_groups and the host-to-device / device-to-host bytes.  It checks that both engines return identical records (consensus, coverage, MSA rows, DP cells,
aligned counts, and every read's score, CIGAR length and CIGAR hash) and prints the card's name and power limit.

    python tools/exp_qv.py --workload convex_10k --groups 1000 --reps 1 [--modes Q-r0,Q-r2] [--engines chain]
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

MODES = {
    "Q-r0": dict(use_qv=True, out_msa=False, out_cons=True),
    "Q-r2": dict(use_qv=True, out_msa=True, out_cons=True),
    "G-r0": dict(inc_path_score=True, out_msa=False, out_cons=True),
    "QG-r0": dict(use_qv=True, inc_path_score=True, out_msa=False, out_cons=True),
    "G-r2": dict(inc_path_score=True, out_msa=True, out_cons=True),
}


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
    for gi, (x, y) in enumerate(zip(a, b)):
        if x.dp_cells != y.dp_cells or x.n_aligned != y.n_aligned:
            return f"group {gi}: DP cells / aligned count"
        if len(x.msa) != len(y.msa) or any(not np.array_equal(p, q) for p, q in zip(x.msa, y.msa)):
            return f"group {gi}: MSA rows"
        if len(x.cons) != len(y.cons) or any(not np.array_equal(p, q) for p, q in zip(x.cons, y.cons)):
            return f"group {gi}: consensus"
        if any(not np.array_equal(p, q) for p, q in zip(x.cov, y.cov)):
            return f"group {gi}: coverage"
        if not (np.array_equal(x.read_best_score, y.read_best_score) and np.array_equal(x.read_n_cigar, y.read_n_cigar)
                and np.array_equal(x.read_cigar_hash, y.read_cigar_hash)):
            return f"group {gi}: per-read scores / CIGAR lengths / CIGAR hashes"
    return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="convex_10k")
    ap.add_argument("--groups", type=int, default=100)
    ap.add_argument("--reps", type=int, default=1)
    ap.add_argument("--modes", default="Q-r0,Q-r2,G-r0,QG-r0")
    ap.add_argument("--engines", choices=["both", "chain", "launch"], default="both")
    args = ap.parse_args()
    wl = synth.WORKLOADS[args.workload]
    print(f"card: {card()}", flush=True)
    t0 = time.time()
    groups = wl.groups(args.groups)
    weights = [[np.random.default_rng(7100 + gi).integers(1, 41, size=len(r)).astype(np.int32) for r in g] for gi, g in enumerate(groups)]
    packed = PackedGroups(groups, weights)
    print(f"{args.workload}: {args.groups} groups x {wl.n_reads} reads x {wl.length} bp, weights 1..40 "
          f"(generated in {time.time() - t0:.1f} s)", flush=True)
    lib = capi.product()
    warm = PackedGroups(groups[:2], weights[:2])
    for mode in args.modes.split(","):
        abpt = make_para(lib, PoaConfig(**{**wl.cfg.__dict__, **MODES[mode]}))
        try:
            with BatchEngine() as eng:
                for no_chain in (False, True):                          # warm-up: module load, pinned buffers, both engines
                    eng.run_packed(abpt, warm, no_chain=no_chain)
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
                        print(json.dumps({"mode": mode, "engine": engine, "rep": rep, "wall_s": round(wall, 3),
                                          "chain_device_ms": round(st["chain_device_ms"], 1), "chain_groups": st["chain_groups"],
                                          "chain_fallback_groups": st["chain_fallback_groups"], "h2d_bytes": st["h2d_bytes"],
                                          "d2h_bytes": st["d2h_bytes"]}), flush=True)
                if len(last) < 2:
                    continue
                diff = same(last["chain"], last["launch"])
                print(f"{mode}: chain and launch engine records {'identical' if diff is None else 'DIFFER: ' + diff}", flush=True)
                if diff is not None:
                    sys.exit(1)
        finally:
            lib.abpoa_free_para(abpt)


if __name__ == "__main__":
    main()
