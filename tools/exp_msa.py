#!/usr/bin/env python
"""Row-column MSA batches (-r 1 / -r 2) on the two engines of abpoa_gpu_msa_batch.

Runs one batch of a workload with out_msa set, once on the device-resident chain engine and once on the launch engine
(the ABPOA_GPU_NO_CHAIN flag: host graph fusion between kernel launches), alternating, and reports per run the wall time,
chain_device_ms, chain_groups / chain_fallback_groups and the device-to-host bytes.  It checks that both engines return
identical records (MSA rows, consensus, coverage, DP cells) and prints the card's name and power limit.

    python tools/exp_msa.py --workload convex_10k --groups 100 --reps 2
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
        if x.dp_cells != y.dp_cells:
            return f"group {gi}: DP cells"
        if len(x.msa) != len(y.msa) or any(not np.array_equal(p, q) for p, q in zip(x.msa, y.msa)):
            return f"group {gi}: MSA rows"
        if len(x.cons) != len(y.cons) or any(not np.array_equal(p, q) for p, q in zip(x.cons, y.cons)):
            return f"group {gi}: consensus"
        if any(not np.array_equal(p, q) for p, q in zip(x.cov, y.cov)):
            return f"group {gi}: coverage"
    return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="convex_10k")
    ap.add_argument("--groups", type=int, default=100)
    ap.add_argument("--reps", type=int, default=2)
    args = ap.parse_args()
    wl = synth.WORKLOADS[args.workload]
    print(f"card: {card()}", flush=True)
    t0 = time.time()
    groups = wl.groups(args.groups)
    packed = PackedGroups(groups)
    print(f"{args.workload}: {args.groups} groups x {wl.n_reads} reads x {wl.length} bp (generated in {time.time() - t0:.1f} s)", flush=True)
    lib = capi.product()
    warm = PackedGroups(groups[:2])
    for out_name, out in (("-r1", dict(out_msa=True, out_cons=False)), ("-r2", dict(out_msa=True, out_cons=True))):
        abpt = make_para(lib, PoaConfig(**{**wl.cfg.__dict__, **out}))
        try:
            with BatchEngine() as eng:
                for no_chain in (False, True):                          # warm-up: module load, pinned buffers, both engines
                    eng.run_packed(abpt, warm, no_chain=no_chain)
                last = {}
                for rep in range(args.reps):
                    for engine, no_chain in (("chain", False), ("launch", True)):
                        eng.reset_stats()
                        t = time.time()
                        res = eng.run_packed(abpt, packed, no_chain=no_chain)
                        wall = time.time() - t
                        st = eng.stats()
                        last[engine] = res
                        print(json.dumps({"out": out_name, "engine": engine, "rep": rep, "wall_s": round(wall, 3),
                                          "chain_device_ms": round(st["chain_device_ms"], 1), "chain_groups": st["chain_groups"],
                                          "chain_fallback_groups": st["chain_fallback_groups"], "d2h_bytes": st["d2h_bytes"],
                                          "msa_cols_mean": round(float(np.mean([len(r.msa[0]) for r in res if r.msa])), 1)}), flush=True)
                diff = same(last["chain"], last["launch"])
                print(f"{out_name}: chain and launch engine records {'identical' if diff is None else 'DIFFER: ' + diff}", flush=True)
                if diff is not None:
                    sys.exit(1)
        finally:
            lib.abpoa_free_para(abpt)


if __name__ == "__main__":
    main()
