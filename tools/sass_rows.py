#!/usr/bin/env python3
"""Static SASS budget of the chain engine's DP row, no GPU needed.

Cross-compiles poa_kernels.cu for sm_90a with line information, disassembles the free-running chain worker
(poa_chain_dp_worker_kernel<GAP>) and counts its instructions by the source region they come from.  Inlined helpers
count where they are called (nvdisasm -gi prints the whole inline chain).  Regions of the forward row loop of
p16_run_job are cut at its KP(n) phase markers:

  set-up       loop head .. KP(0)        band, plane-slab cursor, query-profile prefetch
  pred fetch   KP(0) .. KP(1)            predecessor planes, folded into M / X1 / X2
  recurrence   KP(1) .. btrec            H / E / F of the row's cells
  btrec        backtrace shortcut record
  fbits        F decision bytes (only in sources whose forward pass still computes them)
  stores       KP(2) .. KP(3)            ring + HBM stores
  row max      KP(3) .. KP(4)
  tail         KP(4) .. loop end         row metadata, arg-max bookkeeping, next row's loads

then the backtrace (poa_backtrack and what it calls) and everything else.  The row loop is straight-line per 256-cell
pass, so at bands up to 256 cells its static count is close to what one row issues.

    python tools/sass_rows.py [--src path/to/poa_kernels.cu] [--gap convex|affine|linear] [--ops] [--path-score]
"""
from __future__ import annotations

import argparse
import collections
import re
import subprocess
import sys
import tempfile
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
NVCC = "/usr/local/cuda/bin/nvcc"
GAPS = {"linear": 0, "affine": 1, "convex": 2}
LOOP_REGIONS = ["set-up", "pred fetch", "recurrence", "btrec", "fbits", "stores", "row max", "tail"]


def find(lines, pat, start=0, end=None):
    for k in range(start, len(lines) if end is None else end):
        if pat in lines[k]:
            return k
    return None


def body(lines, head):
    """0-based [first, last] line range of the function whose signature contains `head` (brace matching)."""
    k = find(lines, head)
    if k is None:
        return None
    depth, seen = 0, False
    for e in range(k, len(lines)):
        depth += lines[e].count("{") - lines[e].count("}")
        seen = seen or "{" in lines[e]
        if seen and depth == 0:
            return k, e
    raise SystemExit(f"unbalanced braces after {head!r}")


def regions(src: Path):
    """1-based line ranges [a, b) of the row-loop regions and of the backtrace."""
    L = src.read_text().splitlines()
    run = body(L, "__device__ __forceinline__ void p16_run_job(")
    loop = find(L, "for (int i = 1; i < n_rows - 1 && !stop; ++i)", run[0], run[1])
    kp = {}
    for n in (0, 1, 2, 3, 4):
        kp[n] = find(L, f"KP({n})", loop, run[1])
    btrec = find(L, "backtrace shortcut record (PoaBtRec)", kp[1], kp[2])
    fb = find(L, "/* FB: the insertion-step comparisons", btrec, kp[2])
    end = find(L, "cursor = cur32;", kp[4], run[1])
    cuts = [("set-up", loop, kp[0]), ("pred fetch", kp[0], kp[1]), ("recurrence", kp[1], btrec),
            ("btrec", btrec, fb if fb is not None else kp[2])]
    if fb is not None:
        cuts.append(("fbits", fb, kp[2]))
    cuts += [("stores", kp[2], kp[3]), ("row max", kp[3], kp[4]), ("tail", kp[4], end)]
    bt = [body(L, "__device__ void poa_backtrack(")]
    rc = body(L, "__device__ int fb_recompute(")
    if rc is not None and find(L, "{", rc[0], rc[0] + 3) is not None:
        bt.append(rc)
    # 0-based -> 1-based line numbers
    return [(n, a + 1, b + 1) for n, a, b in cuts], [(a + 1, b + 2) for a, b in bt]


def disassemble(src: Path, tmp: Path, gap: int, ps: bool = False):
    cubin = tmp / "k.cubin"
    subprocess.run([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
                    f"-I{ROOT / 'include'}", f"-I{ROOT / 'abpoa_b200' / 'csrc'}", "-cubin", "-o", str(cubin), str(src)], check=True)
    res = subprocess.run(["/usr/local/cuda/bin/cuobjdump", "-res-usage", str(cubin)], check=True, capture_output=True, text=True).stdout
    tail = "Lb0ELb1E" if ps else "(?:Lb0E)*"                 # without -s; with -G (ps) or without
    fn = re.search(rf"Function (_Z26poa_chain_dp_worker_kernelILi{gap}E{tail}Ev\w+):", res).group(1)
    m = re.search(re.escape(fn) + r":\s*\n\s*REG:(\d+)", res)
    regs = int(m.group(1)) if m else None
    dis = subprocess.run(["/usr/local/cuda/bin/nvdisasm", "-gi", str(cubin)], check=True, capture_output=True, text=True).stdout
    a = dis.index(f".text.{fn}:")
    b = min((k for k in (dis.find("\n.section", a + 1), dis.find("\n\t.section", a + 1)) if k > 0), default=-1)
    return dis[a: b if b > 0 else None].splitlines(), regs


def count(text, src_name, loop_regions, bt_ranges):
    ann = re.compile(r'line (\d+)')
    ins = re.compile(r'^\s*/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P[T0-9]\s+)?([A-Z][A-Z0-9_.]*)')
    counts, ops = collections.Counter(), collections.defaultdict(collections.Counter)
    chain, fresh = [], False
    for line in text:
        if line.lstrip().startswith("//##"):
            if not fresh:
                chain, fresh = [], True
            if src_name in line:
                chain += [int(x) for x in ann.findall(line)]
            continue
        m = ins.match(line)
        if not m:
            continue
        fresh = False
        where = "other"
        if any(a <= x < b for x in chain for a, b in bt_ranges):
            where = "backtrace"
        else:
            for name, a, b in loop_regions:
                if any(a <= x < b for x in chain):
                    where = name
                    break
        counts[where] += 1
        ops[where][m.group(1).split(".")[0]] += 1
    return counts, ops


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--src", type=Path, default=ROOT / "abpoa_b200" / "csrc" / "poa_kernels.cu")
    ap.add_argument("--gap", choices=list(GAPS), default="convex")
    ap.add_argument("--ops", action="store_true", help="also list the most frequent opcodes per region")
    ap.add_argument("--path-score", action="store_true", help="the path-score (-G) instantiation of the kernel")
    args = ap.parse_args()
    src = args.src.resolve()
    loop_regions, bt_ranges = regions(src)
    with tempfile.TemporaryDirectory() as tmp:
        text, regs = disassemble(src, Path(tmp), GAPS[args.gap], args.path_score)
    counts, ops = count(text, src.name, loop_regions, bt_ranges)
    print(f"poa_chain_dp_worker_kernel<{args.gap}{', -G' if args.path_score else ''}> from {src.name}: {regs} registers per thread")
    print(f"  {'region':<14}{'instructions':>13}")
    row = 0
    for name in LOOP_REGIONS:
        if name == "fbits" and not any(n == "fbits" for n, _, _ in loop_regions):
            continue
        row += counts[name]
        print(f"  {name:<14}{counts[name]:>13}" + ("   " + ", ".join(f"{o} {c}" for o, c in ops[name].most_common(6)) if args.ops else ""))
    print(f"  {'= row loop':<14}{row:>13}")
    print(f"  {'backtrace':<14}{counts['backtrace']:>13}")
    print(f"  {'other':<14}{counts['other']:>13}")
    return 0


if __name__ == "__main__":
    sys.exit(main())
