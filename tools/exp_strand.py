#!/usr/bin/env python
"""Ambiguous-strand batches (-s) on the two engines of abpoa_gpu_msa_batch.

Every third read of every group is reverse-complemented (as strand_mix in tests/test_gpu_cases.py does).  Runs one batch
of a workload with amb_strand set, for -r 0 (consensus) and -r 2 (consensus + row-column MSA), once on the
device-resident chain engine and once on the launch engine (the ABPOA_GPU_NO_CHAIN flag: host graph fusion between
kernel launches, a second host round per retried read), alternating, and reports per run the wall time,
chain_device_ms, chain_groups / chain_fallback_groups, the device-to-host bytes, the reads that arrive flipped and the
reverse-complement alignments the engine ran (n_aligned counts both DPs of a retried read).  It checks that both engines
return identical records (consensus, coverage, MSA rows, DP cells, aligned counts) and prints the card's name and power
limit.

    python tools/exp_strand.py --workload convex_10k --groups 1000 --reps 1 [--engines chain]
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


def revcomp(x):
    """The reverse complement by abPOA's rule: code b < 4 becomes 3 - b, every other code 4."""
    x = np.asarray(x, dtype=np.uint8)
    return np.ascontiguousarray(np.where(x < 4, 3 - x, 4).astype(np.uint8)[::-1])


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
    return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="convex_10k")
    ap.add_argument("--groups", type=int, default=100)
    ap.add_argument("--reps", type=int, default=1)
    ap.add_argument("--engines", choices=["both", "chain", "launch"], default="both")
    args = ap.parse_args()
    wl = synth.WORKLOADS[args.workload]
    print(f"card: {card()}", flush=True)
    t0 = time.time()
    groups = [[revcomp(x) if i % 3 == 1 else x for i, x in enumerate(g)] for g in wl.groups(args.groups)]
    flipped = sum(1 for g in groups for i in range(len(g)) if i % 3 == 1)
    packed = PackedGroups(groups)
    print(f"{args.workload}: {args.groups} groups x {wl.n_reads} reads x {wl.length} bp, {flipped} reads flipped "
          f"(generated in {time.time() - t0:.1f} s)", flush=True)
    lib = capi.product()
    warm = PackedGroups(groups[:2])
    for out_name, out in (("-r0", dict(out_msa=False, out_cons=True)), ("-r2", dict(out_msa=True, out_cons=True))):
        abpt = make_para(lib, PoaConfig(**{**wl.cfg.__dict__, **out, "amb_strand": True}))
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
                        res = eng.run_packed(abpt, packed, no_chain=no_chain)
                        wall = time.time() - t
                        st = eng.stats()
                        last[engine] = res
                        print(json.dumps({"out": out_name, "engine": engine, "rep": rep, "wall_s": round(wall, 3),
                                          "chain_device_ms": round(st["chain_device_ms"], 1), "chain_groups": st["chain_groups"],
                                          "chain_fallback_groups": st["chain_fallback_groups"], "d2h_bytes": st["d2h_bytes"],
                                          "flipped_reads": flipped,
                                          "rc_alignments": int(sum(r.n_aligned - (len(g) - 1) for r, g in zip(res, groups)))}), flush=True)
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
