"""GPU: every DP cell of the single-alignment path against the scalar oracle (tests/planes.py), kernel by kernel.

End results (score, graph-CIGAR, end points, cells, consensus) are checked elsewhere; a wrong H / E / F cell that does not
change today's chosen path would pass those.  Here every row's band and arg-max and every plane cell are compared after
every read, and each case asserts which kernel instantiation produced the accepted result.

Switches latched per process (ABPOA_GPU_TMA, ABPOA_GPU_NO_LEAN, ABPOA_GPU_SMEM_KB are read once into statics) are tested in
a child interpreter that has the variable set from its start: `python tests/test_gpu_planes.py <case>...` runs cases and
prints one JSON line per alignment with the kernel variant and ring geometry it saw.
"""
from __future__ import annotations

import json
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

HERE = Path(__file__).resolve().parent
if __name__ == "__main__":
    sys.path[:0] = [str(HERE.parent), str(HERE)]

from abpoa_b200 import synth  # noqa: E402
from abpoa_b200.aligner import PoaConfig  # noqa: E402
from abpoa_b200.capi import ABPOA_EXTEND_MODE, ABPOA_LOCAL_MODE  # noqa: E402
from helpers import deletion_fan  # noqa: E402
from planes import run_planes  # noqa: E402

AFFINE = dict(gap_open1=4, gap_ext1=2, gap_open2=0, gap_ext2=0)
LINEAR = dict(gap_open1=0, gap_ext1=2, gap_open2=0, gap_ext2=0)
CONVEX = dict()
GAPS = {"LG": LINEAR, "AG": AFFINE, "CG": CONVEX}
INT32 = dict(match=20, mismatch=40, gap_open1=40, gap_ext1=20, gap_open2=240, gap_ext2=10)
QLENS = [1, 7, 8, 9, 255, 256, 257, 513]


def ragged(seed, lens, err=0.05):
    """The first read builds the graph; the others are prefixes of further reads of the same template."""
    base = synth.make_group(seed, len(lens), max(lens), err)
    return [np.ascontiguousarray(r[:n]) for r, n in zip(base, lens)]


def qlen_sweep(seed):
    return ragged(seed, [520] + QLENS)                      # qlen 1 .. 513 against a ~520-node graph (7: 70x shorter)


def short_long(seed):
    return ragged(seed, [1000, 60, 90]) + [synth.make_group(seed + 1, 1, 2000, 0.05)[0]]   # 10-20x shorter, 2x longer


def subgraph_reads(seed=2100):
    rng = np.random.default_rng(77)
    full = synth.make_group(seed, 4, 400, 0.06)
    reads, windows = list(full), [(0, 1)] * len(full)
    for _ in range(5):                                       # partial reads inside windows of node ids of the first read
        a = int(rng.integers(10, 150)); b = int(rng.integers(250, 390))
        piece = full[0][a:b].copy()
        piece[::17] = (piece[::17] + 1) % 4
        reads.append(piece)
        windows.append((2 + a, 2 + b - 1))                  # the first read's base i became node id 2 + i
    return reads, windows


# name -> (config, reads builder, expected: kernel bits, lean (None: either), sub-graph windows?)
CASES = {}


def case(name, cfg, reads, kernel, lean=None, windows=None):
    CASES[name] = dict(cfg=cfg, reads=reads, kernel=kernel, lean=lean, windows=windows)


for g, kw in GAPS.items():
    banded = g != "LG"          # banded linear global runs the generic "lgx" kernel; LG reaches the packed one unbanded
    case(f"packed_{g}_global_lean_qlens", dict(kw, wb=10 if banded else -1), lambda s=11: qlen_sweep(s), 15, True)
    case(f"packed_{g}_global_G", dict(kw, wb=10 if banded else -1, inc_path_score=True), lambda: synth.make_group(12, 6, 300, 0.10), 15, False)
    case(f"packed_{g}_local", dict(kw, align_mode=ABPOA_LOCAL_MODE), lambda s=13: qlen_sweep(s), 15, False)
case("packed_AG_extend_zdrop", dict(AFFINE, align_mode=ABPOA_EXTEND_MODE, zdrop=100), lambda: ragged(14, [700, 650, 300, 700, 120]), 15, False)
case("packed_CG_extend_zdrop", dict(align_mode=ABPOA_EXTEND_MODE, zdrop=100), lambda: ragged(15, [700, 650, 300, 700, 120]), 15, False)
case("packed_LG_extend_zdrop", dict(LINEAR, wb=-1, align_mode=ABPOA_EXTEND_MODE, zdrop=60), lambda: ragged(16, [500, 450, 200]), 15, False)
case("packed_CG_wide_band", dict(wb=200), lambda: synth.make_group(17, 5, 900, 0.10), 15, True)
case("packed_AG_unbanded_1k", dict(AFFINE, wb=-1), lambda: synth.make_group(18, 4, 1000, 0.08), 15, True)
case("packed_CG_short_long", dict(), lambda: short_long(19), 15, True)
case("packed_CG_fan", dict(), lambda: deletion_fan(), 15, True)
case("packed_AG_fan_G", dict(AFFINE, inc_path_score=True), lambda: deletion_fan(seed=9, n=36), 15, False)
case("packed_CG_error25", dict(), lambda: synth.make_group(20, 6, 500, 0.25), 15, True)
case("packed_CG_subgraph", dict(), lambda: subgraph_reads()[0], 15, None, windows=subgraph_reads()[1])   # whole-graph reads first, then windows
case("lgx_global", dict(LINEAR), lambda s=21: qlen_sweep(s), 16)
case("lgx_short_long", dict(LINEAR), lambda: short_long(26), 16)
case("lgx_extend", dict(LINEAR, align_mode=ABPOA_EXTEND_MODE), lambda: synth.make_group(22, 6, 400, 0.10), 16)
case("int32_CG_global", dict(INT32), lambda: ragged(23, [1700, 1650, 1700, 1600]), 32)
case("int32_AG_local", dict(INT32, gap_open2=0, gap_ext2=0, align_mode=ABPOA_LOCAL_MODE), lambda: ragged(24, [1700, 1650, 1500]), 32)
case("int32_CG_extend", dict(INT32, align_mode=ABPOA_EXTEND_MODE, zdrop=400), lambda: ragged(25, [1700, 1600, 1700]), 32)

# the generic kernel with int16 planes (ABPOA_GPU_NO_P16 is read on every call)
GENERIC16 = ["packed_CG_global_lean_qlens", "packed_AG_global_lean_qlens", "packed_LG_global_lean_qlens", "packed_CG_local",
             "packed_AG_local", "packed_LG_local", "packed_CG_extend_zdrop", "packed_CG_global_G", "packed_CG_wide_band", "packed_CG_fan",
             "packed_CG_error25", "packed_CG_subgraph"]


def run_case(name, expect_kernel=None, env_note=""):
    c = CASES[name]
    kernel = c["kernel"] if expect_kernel is None else expect_kernel
    seen = []

    def check(i, info):
        seen.append(info)
        assert info.kernel == kernel, f"{name} read {i}: accepted result came from the {info.name} kernel, expected {kernel}"
        if kernel == 15 and c["lean"] is not None and "NO_LEAN" not in env_note:
            assert info.lean == c["lean"], f"{name} read {i}: LEAN={info.lean}, expected {c['lean']}"
    run_planes(PoaConfig(**c["cfg"]), c["reads"](), windows=c["windows"], tag=name, check=check)
    assert seen, f"{name}: no alignment ran"
    return seen


def _log(name, seen, env=""):
    s = seen[-1]
    print(f"[planes] {name}{env}: {len(seen)} alignments, kernel={s.name} lean={int(s.lean)} tma={int(s.tma)} "
          f"ring={s.ring_rows}x{s.ring_cells} widest_groups={max(x.widest_groups for x in seen)} "
          f"max_inf={max(x.max_inf for x in seen)} min_finite={min(x.min_finite for x in seen)}")


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_planes(name):
    _log(name, run_case(name))


@pytest.mark.gpu
@pytest.mark.parametrize("name", GENERIC16)
def test_planes_generic_int16(monkeypatch, name):
    monkeypatch.setenv("ABPOA_GPU_NO_P16", "1")
    _log(name, run_case(name, expect_kernel=16), " NO_P16")


# ------------------------------------------------------------------------------------------- latched switches
def child(env: dict, names: list[str]) -> list[dict]:
    e = {**os.environ, **env}
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [str(Path(__file__)), *names]
    p = subprocess.run(cmd, env=e, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, f"child with {env} failed:\n{p.stdout[-3000:]}\n{p.stderr[-3000:]}"
    print(p.stdout)
    return [json.loads(ln[len("[run] "):]) for ln in p.stdout.splitlines() if ln.startswith("[run] ")]


TMA_CASES = ["packed_AG_global_lean_qlens", "packed_CG_global_lean_qlens", "packed_CG_short_long", "packed_CG_error25", "packed_CG_wide_band"]


@pytest.mark.gpu
def test_planes_tma():
    """ABPOA_GPU_TMA=1: cp.async.bulk row staging, with rows both narrower and wider than a ring slot."""
    runs = child({"ABPOA_GPU_TMA": "1"}, TMA_CASES)
    assert runs and all(r["kernel"] == 15 and r["lean"] and r["tma"] for r in runs), runs
    assert any(r["widest_groups"] > r["ring_cells"] // 8 for r in runs), "no row wider than its ring slot: the plain-store branch never ran"
    assert any(r["widest_groups"] <= r["ring_cells"] // 8 for r in runs), "no alignment kept every row inside a ring slot"


@pytest.mark.gpu
def test_planes_no_lean():
    """ABPOA_GPU_NO_LEAN=1: whole-graph global jobs take the general predecessor loop of the packed kernel."""
    runs = child({"ABPOA_GPU_NO_LEAN": "1"}, ["packed_CG_global_lean_qlens", "packed_AG_global_lean_qlens", "packed_LG_global_lean_qlens",
                                              "packed_CG_fan", "packed_CG_wide_band"])
    assert runs and all(r["kernel"] == 15 and not r["lean"] and not r["tma"] for r in runs), runs


@pytest.mark.gpu
def test_planes_small_ring():
    """ABPOA_GPU_SMEM_KB=5: two ring rows of 64 cells, so predecessors beyond the previous row come from HBM and rows wider
    than a slot are cached as a prefix (poa_pick_ring)."""
    names = ["packed_CG_global_lean_qlens", "packed_AG_local", "packed_CG_wide_band", "packed_AG_unbanded_1k", "packed_CG_fan",
             "packed_CG_subgraph", "lgx_global", "lgx_short_long", "int32_CG_global"]
    runs = child({"ABPOA_GPU_SMEM_KB": "5"}, names)
    assert runs and all(r["ring_rows"] == 2 for r in runs), runs
    assert any(r["kernel"] == 15 and r["widest_groups"] > r["ring_cells"] // 8 for r in runs), "packed kernel never saw a band wider than the ring"
    assert any(r["kernel"] != 15 and r["widest_groups"] > r["ring_cells"] // 8 for r in runs), "generic kernel never saw a band wider than the ring"


if __name__ == "__main__":
    env = " ".join(f"{k}={os.environ[k]}" for k in ("ABPOA_GPU_TMA", "ABPOA_GPU_NO_LEAN", "ABPOA_GPU_SMEM_KB") if k in os.environ)
    for n in sys.argv[1:]:
        seen = run_case(n, env_note=env)
        _log(n, seen, f" [{env}]")
        for s in seen:
            print("[run] " + json.dumps(dict(case=n, kernel=s.kernel, lean=s.lean, tma=s.tma, ring_rows=s.ring_rows,
                                             ring_cells=s.ring_cells, widest_groups=s.widest_groups)), flush=True)
