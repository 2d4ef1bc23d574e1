#!/usr/bin/env python
"""GFA batches (-r 3 / -r 4) through abpoa_gpu_msa_batch_write on the two engines.

Runs one batch of a workload with out_gfa set, on the device-resident chain engine and on the launch engine (the
ABPOA_GPU_NO_CHAIN flag), writing to /dev/null, and reports per run the wall time, chain_device_ms, the device-to-host
bytes, chain_groups / chain_fallback_groups and the process's peak RSS.  One more run per engine writes into a pipe to a
child that counts the bytes and takes their md5, so that the two engines' texts can be compared.  Prints the card's name
and power limit first.

    python tools/exp_gfa.py --workload convex_10k --groups 1000 --reps 1
"""
import argparse
import ctypes as C
import json
import resource
import sys
import tempfile
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
sys.path.insert(0, str(Path(__file__).resolve().parent))
from abpoa_b200 import capi, synth  # noqa: E402
from abpoa_b200.aligner import PoaConfig, make_para  # noqa: E402
from abpoa_b200.batch import BatchEngine, PackedGroups  # noqa: E402
from exp_msa import card  # noqa: E402

_libc = C.CDLL(None)
for name in ("fopen", "popen"):
    getattr(_libc, name).restype = C.c_void_p
    getattr(_libc, name).argtypes = [C.c_char_p, C.c_char_p]
_libc.fclose.argtypes = [C.c_void_p]
_libc.pclose.argtypes = [C.c_void_p]

# the child behind the pipe: byte count and md5 of its stdin, on one line of stdout
COUNT_MD5 = "import hashlib,sys; h=hashlib.md5(); n=0\nfor b in iter(lambda: sys.stdin.buffer.read(1 << 22), b''): h.update(b); n += len(b)\nprint(n, h.hexdigest())"


def gfa_para(lib, cfg, out_cons):
    p = make_para(lib, PoaConfig(**{**cfg.__dict__, "out_cons": out_cons, "out_msa": False}))
    p.contents.out_gfa = 1
    lib.abpoa_post_set_para(p)
    return p


def peak_rss_mb() -> float:
    return resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 1024.0


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
    for out_name, out_cons in (("-r3", False), ("-r4", True)):
        abpt = gfa_para(lib, wl.cfg, out_cons)
        try:
            with BatchEngine() as eng:
                devnull = _libc.fopen(b"/dev/null", b"w")
                for no_chain in (False, True):                          # warm-up: module load, pinned buffers, both engines
                    eng.run_write(abpt, warm, devnull, no_chain=no_chain)
                digests = {}
                for rep in range(args.reps + 1):
                    check = rep == args.reps                            # the last run of each engine: text into the md5 pipe
                    for engine, no_chain in (("chain", False), ("launch", True)):
                        with tempfile.NamedTemporaryFile("r", suffix=".md5") as res:
                            fp = _libc.popen(f"{sys.executable} -c \"{COUNT_MD5}\" > {res.name}".encode(), b"w") if check else devnull
                            eng.reset_stats()
                            t = time.time()
                            eng.run_write(abpt, packed, fp, no_chain=no_chain)
                            wall = time.time() - t
                            st = eng.stats()
                            rec = {"out": out_name, "engine": engine, "rep": rep, "sink": "md5 pipe" if check else "/dev/null", "wall_s": round(wall, 3),
                                   "chain_device_ms": round(st["chain_device_ms"], 1), "chain_groups": st["chain_groups"],
                                   "chain_fallback_groups": st["chain_fallback_groups"], "d2h_bytes": st["d2h_bytes"], "peak_rss_mb": round(peak_rss_mb())}
                            if check:
                                _libc.pclose(fp)                        # waits for the child
                                n, digest = res.read().split()
                                rec["text_bytes"], rec["md5"] = int(n), digest
                                digests[engine] = digest
                        print(json.dumps(rec), flush=True)
                same = digests["chain"] == digests["launch"]
                ok = ok and same
                print(f"{out_name}: chain and launch engine text {'identical' if same else 'DIFFER'} (md5 {digests['chain']} / {digests['launch']})", flush=True)
                _libc.fclose(devnull)
        finally:
            lib.abpoa_free_para(abpt)
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
