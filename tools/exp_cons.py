#!/usr/bin/env python
"""Most-frequent-base consensus (-a 1) batches on the two engines of abpoa_gpu_msa_batch, and against heaviest bundling.

Runs one batch of a workload with -a 1 (-r 0 and -r 2) on the device-resident chain engine and on the launch engine (the
ABPOA_GPU_NO_CHAIN flag: host graph fusion between kernel launches, consensus on the host), and with -a 0 -r 0 on the
chain engine.  Reports per run the wall time, chain_device_ms, chain_groups / chain_fallback_groups and the
device-to-host bytes, checks that both engines return identical records with -a 1 (consensus, coverage, MSA rows, DP
cells) and prints the card's name and power limit.

    python tools/exp_cons.py --workload convex_10k --groups 1000 --reps 1
"""
import argparse
import json
import sys
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
sys.path.insert(0, str(Path(__file__).resolve().parent))
from abpoa_b200 import capi, synth  # noqa: E402
from abpoa_b200.aligner import PoaConfig, make_para  # noqa: E402
from abpoa_b200.batch import BatchEngine, PackedGroups  # noqa: E402
from abpoa_b200.capi import ABPOA_HB, ABPOA_MF  # noqa: E402
from exp_msa import card, same  # noqa: E402

RUNS = [   # (name, cons_algrm, out_msa, engines)
    ("-a1 -r0", ABPOA_MF, False, ("chain", "launch")),
    ("-a1 -r2", ABPOA_MF, True, ("chain", "launch")),
    ("-a0 -r0", ABPOA_HB, False, ("chain",)),
]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="convex_10k")
    ap.add_argument("--groups", type=int, default=1000)
    ap.add_argument("--reps", type=int, default=1)
    args = ap.parse_args()
    wl = synth.WORKLOADS[args.workload]
    print(f"card: {card()}", flush=True)
    t0 = time.time()
    groups = wl.groups(args.groups)
    packed = PackedGroups(groups)
    print(f"{args.workload}: {args.groups} groups x {wl.n_reads} reads x {wl.length} bp (generated in {time.time() - t0:.1f} s)", flush=True)
    lib = capi.product()
    warm = PackedGroups(groups[:2])
    ok = True
    for name, alg, out_msa, engines in RUNS:
        abpt = make_para(lib, PoaConfig(**{**wl.cfg.__dict__, "cons_algrm": alg, "out_cons": True, "out_msa": out_msa}))
        try:
            with BatchEngine() as eng:
                for engine in engines:                                  # warm-up: module load, pinned buffers, both engines
                    eng.run_packed(abpt, warm, no_chain=engine == "launch")
                last = {}
                for rep in range(args.reps):
                    for engine in engines:
                        eng.reset_stats()
                        t = time.time()
                        res = eng.run_packed(abpt, packed, no_chain=engine == "launch")
                        wall = time.time() - t
                        st = eng.stats()
                        last[engine] = res
                        print(json.dumps({"run": name, "engine": engine, "rep": rep, "wall_s": round(wall, 3),
                                          "chain_device_ms": round(st["chain_device_ms"], 1), "chain_groups": st["chain_groups"],
                                          "chain_fallback_groups": st["chain_fallback_groups"], "d2h_bytes": st["d2h_bytes"],
                                          "cons_len_mean": round(sum(len(r.cons[0]) for r in res if r.cons) / max(1, len(res)), 1)}), flush=True)
                if len(engines) == 2:
                    diff = same(last["chain"], last["launch"])
                    print(f"{name}: chain and launch engine records {'identical' if diff is None else 'DIFFER: ' + diff}", flush=True)
                    ok = ok and diff is None
        finally:
            lib.abpoa_free_para(abpt)
    if not ok:
        sys.exit(1)


if __name__ == "__main__":
    main()
