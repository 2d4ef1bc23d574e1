"""The chain engine's job function cell by cell against the scalar oracle (tests/planes.py).

The chain runs p16_run_job<GAP, GLOBAL, LEAN, no TMA, FB>: a row stores only H, E1 (, E2) (the compact layout), and the
backtrace rebuilds a row's F planes and insertion-step decision bytes (fb_recompute) the first time it needs them, in the
few rows where it inserts.  Its own tests compare end records with the launch engine only, so a wrong compact cell that
today's path never reads, or a wrong recomputed byte in a row no backtrace visits, would pass them.  Here every aligned
read of every case is checked as tests/test_gpu_planes.py checks it (five-plane kernel against the oracle), then replayed
on the chain's job function (poa_debug_chain_replay) with the chain's ring geometry and with the smallest ring (2 rows of
64 cells), and:
  1. the replay's score, end points, graph-CIGAR equal the oracle's; its cells / widest row the five-plane run's
  2. every row's band and first / last arg-max equal the five-plane run's and the oracle's
  3. the compact H / E1 (/ E2) planes pass compare_planes against the oracle
  4. ... and equal the five-plane kernel's bit for bit on every stored cell, floor cells included (successors read them)
  5. the compact slab takes ngrp * N16 units per computed row, as the chain's planner and allocator assume
  6. the F planes of every row, rebuilt right to left the way the backtrace walks, pass compare_planes against the oracle
     and equal the five-plane kernel's bit for bit
  7. every decision byte equals decision_bytes() of the five-plane kernel's planes, and of the oracle's where the oracle's
     F value is finite -- with the recompute buffer holding a whole row, the chain's buffer at (2, 64) and one pass
A row wider than the buffer keeps only its last passes, and a step left of them recomputes (the windowed branch): the
wide-band and long-insertion cases reach it in every row of the dump, and the long-insertion groups also go through the
real chain with a two-row ring (ABPOA_GPU_SMEM_KB=5, latched per process: run in a child interpreter,
`python tests/test_gpu_chain_planes.py windowed`).  The tests not marked gpu check on the oracle alone that the shapes
still contain what the GPU tests rely on."""
from __future__ import annotations

import ctypes as C
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

import score_window as sw  # noqa: E402
from abpoa_b200 import capi, synth  # noqa: E402
from abpoa_b200.aligner import PoaConfig, PoaSession  # noqa: E402
from abpoa_b200.capi import ABPOA_CINS  # noqa: E402
from cases import AFFINE, BLOSUM  # noqa: E402
from helpers import deletion_fan  # noqa: E402
from planes import ORACLE_NINF, chain_replay, compare_planes, decision_bytes, fetch_planes, run_planes  # noqa: E402
from test_gpu_chain_recompute import insert_runs, many_runs_group, run_length_group  # noqa: E402
from test_gpu_planes import qlen_sweep, short_long  # noqa: E402

GAPS = {"CG": {}, "AG": AFFINE}
SMALL_RING = (2, 64)
# the chain's recompute buffer is its ring (ring_row_bytes * ring_rows): at (2, 64) H + E1 + E2 (convex) or H + E1 (affine)
SMALL_RING_BUF = {"CG": 3 * 64 * 2 * 2, "AG": 2 * 64 * 2 * 2}
ONE_PASS = 256


def long_insert_groups(gap: str) -> list[list[np.ndarray]]:
    """Three-read groups whose second read carries one random run longer than the decision buffer of a two-row ring
    (768 cells convex, 512 affine), so that its backtrace walks left of the kept passes inside one row."""
    def substitute(x, rng, k):
        x = x.copy()
        at = rng.choice(len(x), size=k, replace=False)
        x[at] = (x[at] + rng.integers(1, 4, size=k)) % 4
        return x
    out = []
    for k, n in enumerate((800, 1000) if gap == "CG" else (560, 700)):
        rng = np.random.default_rng(8500 + 10 * k + (gap == "AG"))
        t = rng.integers(0, 4, size=1500).astype(np.uint8)
        out.append([t, substitute(insert_runs(t, rng, [n], [600 + 200 * k]), rng, 20), substitute(t, rng, 30)])
    return out


def wide(gap, **kw):
    return dict(GAPS[gap], **kw)


CASES = {}
for g in GAPS:
    s = 0 if g == "CG" else 1
    CASES[f"{g}_qlens"] = (dict(GAPS[g]), lambda s=s: qlen_sweep(11 + 20 * s))                  # qlen 1 .. 513, ~520-node graph
    CASES[f"{g}_short_long"] = (dict(GAPS[g]), lambda s=s: short_long(19 + 20 * s))             # 10-20x shorter, 2x longer
    CASES[f"{g}_error25"] = (dict(GAPS[g]), lambda s=s: synth.make_group(20 + 20 * s, 5, 500, 0.25))
    CASES[f"{g}_wf01_3k"] = (wide(g, wf=0.1), lambda s=s: synth.make_group(8300 + s, 3, 3000, 0.04))       # ~620-cell rows
    CASES[f"{g}_wb1000"] = (wide(g, wb=1000, wf=0.0), lambda s=s: synth.make_group(8310 + s, 3, 2400, 0.04))   # 2001 cells
    CASES[f"{g}_fan"] = (dict(GAPS[g]), lambda s=s: deletion_fan(seed=7 + 2 * s, n=40 + 10 * s))   # rows with 34 / 36 predecessors
    CASES[f"{g}_run_lengths"] = (dict(GAPS[g]), lambda s=s: run_length_group(8100 + s, 8, 700))
    CASES[f"{g}_many_runs"] = (dict(GAPS[g]), lambda s=s: many_runs_group(8200 + s, 7, 600))
    CASES[f"{g}_blosum62"] = (dict(GAPS[g], m=27, score_matrix=BLOSUM), lambda s=s: synth.make_group(110 + s, 4, 600, 0.10, 27))
    CASES[f"{g}_long_insert"] = (dict(GAPS[g]), lambda g=g: [r for grp in long_insert_groups(g) for r in grp[:2]])
# admitted, guard-quiet global points of the int16 score window: real cells close to the packed kernel's floor
WINDOW_POINTS = ["guard_lo_e25", "guard_band_e16", "p16_e_100", "infmin_affine_e24", "infmin_convex_e24", "infmin_affine_e64_g400",
                 "infmin_convex_e64_g400"]
for p in WINDOW_POINTS:
    CASES[f"window_{p}"] = (sw.BY_NAME[p][1], sw.BY_NAME[p][2])


def _gap(cfg: PoaConfig) -> str:
    return "CG" if cfg.gap_open2 or cfg.gap_ext2 else "AG"


def _rows(info, rowinfo, upto=None):
    """(row, beg, end, g0, ngrp) of every computed row (0 .. n_rows - 2)."""
    for r in range(info.n_rows - 1 if upto is None else upto):
        beg, end = int(rowinfo[r, 0]), int(rowinfo[r, 1])
        if end >= beg:
            yield r, beg, end, beg >> 3, (end >> 3) - (beg >> 3) + 1


class Checker:
    """The per-read checks (items 1-7 of the module docstring), run from run_planes' post-read hook."""

    def __init__(self, name: str, cfg: PoaConfig, reads):
        self.name, self.cfg, self.reads = name, cfg, reads
        self.gap = _gap(cfg)
        self.n16 = 3 if self.gap == "CG" else 2
        self.f_order = (3, 4) if self.gap == "CG" else (3,)
        self.f5 = (3, 4) if self.gap == "CG" else (2,)            # F planes in the five-plane layout
        self.pen = [(cfg.gap_open1 + cfg.gap_ext1, cfg.gap_ext1)] + ([(cfg.gap_open2 + cfg.gap_ext2, cfg.gap_ext2)] if self.gap == "CG" else [])
        self.i = -1
        self.log = dict(geoms=set(), bufs=set(), widest_passes=0, windows=0, max_windows=0, reads=0)

    def check(self, i, info):
        self.i = i
        assert info.kernel == 15 and info.lean, f"{self.name} read {i}: kernel {info.name} lean={info.lean}: not the chain's instantiation"

    def __call__(self, gpu, rows, info, o):
        qlen = len(self.reads[self.i])
        t = f"{self.name} read {self.i} (qlen {qlen})"
        five = fetch_planes(gpu, info)
        self.log["reads"] += 1
        for geom, bufs in (((0, 0), (0,)), (SMALL_RING, (-1, 0, ONE_PASS))):
            for k, buf in enumerate(bufs):
                rep = chain_replay(gpu, info, qlen, *geom, buf)
                tg = f"{t} ring {rep.ring_rows}x{rep.ring_cells} buf {rep.buf_cells}"
                if geom == SMALL_RING:
                    assert (rep.ring_rows, rep.ring_cells) == SMALL_RING
                    assert buf != 0 or rep.buf_cells == SMALL_RING_BUF[self.gap], tg
                self.log["geoms"].add((rep.ring_rows, rep.ring_cells)); self.log["bufs"].add(rep.buf_cells)
                self.log["windows"] += rep.windows; self.log["max_windows"] = max(self.log["max_windows"], rep.max_windows)
                if k == 0:
                    self.check_replay(gpu, rep, five, rows, info, o, qlen, tg)
                self.check_f(gpu, rep, five, rows, info, qlen, tg)

    # items 1-5
    def check_replay(self, gpu, rep, five, rows, info, o, qlen, t):
        rowinfo5, rowoff5, slab5 = five
        assert rep.status == 0, f"{t}: replay status {rep.status}"
        assert rep.best_score == o.best_score, f"{t}: score {rep.best_score}, oracle {o.best_score}"
        assert rep.ends == (o.node_s, o.node_e, o.query_s, o.query_e), f"{t}: end points {rep.ends}"
        assert rep.n_ops == len(o.cigar) and np.array_equal(rep.cigar, o.cigar), f"{t}: graph-CIGAR differs from the oracle"
        n = info.n_rows - 1
        w5 = rowinfo5[:n, 1].astype(np.int64) - rowinfo5[:n, 0] + 1
        assert rep.cells == int(w5.sum()) and rep.max_band == int(w5.max()), f"{t}: cells / max_band {rep.cells} / {rep.max_band}"
        assert np.array_equal(rep.rowinfo[:n], rowinfo5[:n]), f"{t}: row records differ from the five-plane run's"
        bad = compare_planes(gpu, rows, info, qlen, t + " compact", order=tuple(range(self.n16)),
                             planes=(rep.rowinfo, rep.rowoff, rep.slab))
        assert not bad, "compact planes differ from the oracle:\n  " + "\n  ".join(bad[:12])
        units = 0
        for r, beg, end, g0, ngrp in _rows(info, rep.rowinfo):
            a, b = int(rep.rowoff[r]) * 8, int(rowoff5[r]) * 8
            got = rep.slab[a: a + self.n16 * ngrp * 8]
            want = slab5[b: b + self.n16 * ngrp * 8]
            if not np.array_equal(got, want):
                j = int(np.flatnonzero(got != want)[0])
                raise AssertionError(f"{t}: row {r} plane {j // (ngrp * 8)} cell {g0 * 8 + j % (ngrp * 8)}: compact {int(got[j])}, "
                                     f"five-plane {int(want[j])} (band {beg}..{end})")
            units += ngrp * self.n16
        assert rep.plane_units_used == units, f"{t}: plane_units_used {rep.plane_units_used}, rows take {units}"
        self.log["widest_passes"] = max(self.log["widest_passes"], max((ng + 31) // 32 for *_, ng in _rows(info, rep.rowinfo)))

    # items 6-7
    def check_f(self, gpu, rep, five, rows, info, qlen, t):
        rowinfo5, rowoff5, slab5 = five
        frows = {r: v for r, v in rows.items() if 0 < r < info.n_rows - 1}
        bad = compare_planes(gpu, frows, info, qlen, t + " recomputed F", order=self.f_order, planes=(rep.rowinfo, rep.rowoff, rep.fslab))
        assert not bad, "recomputed F planes differ from the oracle:\n  " + "\n  ".join(bad[:12])
        nf = len(self.f_order)
        for r, beg, end, g0, ngrp in _rows(info, rep.rowinfo):
            if r == 0:
                continue
            a, b, gw = int(rep.rowoff[r]) * 8, int(rowoff5[r]) * 8, ngrp * 8
            f_got = rep.fslab[a: a + nf * gw].reshape(nf, gw)
            f5 = np.stack([slab5[b + p * gw: b + (p + 1) * gw] for p in self.f5])
            if not np.array_equal(f_got, f5):
                k, j = (int(x[0]) for x in np.nonzero(f_got != f5))
                raise AssertionError(f"{t}: row {r} F{k + 1} cell {g0 * 8 + j}: recomputed {int(f_got[k, j])}, five-plane {int(f5[k, j])}")
            lo, wd = beg - g0 * 8, end - beg + 1
            by = rep.fbits[a: a + gw]
            assert not by[:lo].any() and not by[lo + wd:].any(), f"{t}: row {r}: decision bytes outside the band {beg}..{end}"
            band = by[lo: lo + wd]
            h5 = slab5[b + lo: b + lo + wd]
            model = decision_bytes(h5, [f5[k, lo: lo + wd] for k in range(nf)], self.pen)
            if not np.array_equal(band, model):
                j = int(np.flatnonzero(band != model)[0])
                raise AssertionError(f"{t}: row {r} cell {beg + j}: decision byte {int(band[j]):#o}, model of the five-plane planes {int(model[j]):#o}")
            if r in rows:
                pl = rows[r][2]
                om = decision_bytes(pl[0], [pl[3 + k] for k in range(nf)], self.pen)
                for k in range(nf):
                    fin = pl[3 + k] > ORACLE_NINF // 2
                    m = np.uint8(7 << (3 * k))
                    diff = np.flatnonzero(fin & ((band & m) != (om & m)))
                    if len(diff):
                        j = int(diff[0])
                        raise AssertionError(f"{t}: row {r} cell {beg + j} F{k + 1}: decision bits {int(band[j] & m) >> 3 * k:03b}, "
                                             f"model of the oracle's planes {int(om[j] & m) >> 3 * k:03b}")


def run_case(name: str) -> dict:
    cfg_kw, make = CASES[name]
    cfg = PoaConfig(**cfg_kw)
    reads = make()
    ck = Checker(name, cfg, reads)
    run_planes(cfg, reads, tag=name, check=ck.check, after=ck)
    lg = ck.log
    assert lg["reads"], f"{name}: no alignment ran"
    print(f"[chain-planes] {name}: {lg['reads']} alignments, rings {sorted(lg['geoms'])}, buf_cells {sorted(lg['bufs'])}, "
          f"widest row {lg['widest_passes']} passes, {lg['windows']} recompute windows (at most {lg['max_windows']} in one row)")
    return lg


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_chain_planes(name):
    lg = run_case(name)
    if "wb1000" in name or "long_insert" in name:
        assert lg["max_windows"] > 1, f"{name}: no row needed a second recompute window"


# ------------------------------------------------------------------------------- the windowed branch in the real chain
def child(env: dict, args: list[str]) -> list[dict]:
    e = {**os.environ, **env}
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [str(Path(__file__)), *args]
    p = subprocess.run(cmd, env=e, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, f"child with {env} failed:\n{p.stdout[-3000:]}\n{p.stderr[-3000:]}"
    print(p.stdout)
    return [json.loads(ln[len("[run] "):]) for ln in p.stdout.splitlines() if ln.startswith("[run] ")]


def pick_ring(gap: str, band_cells: int, budget: int) -> tuple[int, int]:
    rr, rc = C.c_int(0), C.c_int(0)
    capi.product().dll.poa_pick_ring(1 if gap == "AG" else 2, 16, band_cells, C.c_size_t(budget), C.byref(rr), C.byref(rc))
    return rr.value, rc.value


def windowed_in_chain() -> list[dict]:
    """Both chain schedules over the long-insertion groups (this process has ABPOA_GPU_SMEM_KB=5 from its start)."""
    from test_gpu_chain_layout import assert_engines_agree
    out = []
    for gap in GAPS:
        # the chain's ring for these groups (poa_chain.cu: poa_pick_ring over the widest read's band, w = wb + wf * len)
        groups = long_insert_groups(gap)
        band_cells = max((2 * (10 + int(0.01 * len(r))) + 1 + 104 + 7) // 8 * 8 for grp in groups for r in grp)
        rr, rc = pick_ring(gap, band_cells, int(os.environ["ABPOA_GPU_SMEM_KB"]) * 1024)
        buf = (3 if gap == "CG" else 2) * rc * 2 * rr                # ring_row_bytes * ring_rows
        assert rr == 2 and buf <= SMALL_RING_BUF[gap], (gap, rr, rc)
        for sched in ("free-running", "rounds"):
            if sched == "rounds":
                os.environ["ABPOA_GPU_CHAIN_ROUNDS"] = "1"
            else:
                os.environ.pop("ABPOA_GPU_CHAIN_ROUNDS", None)
            assert_engines_agree(PoaConfig(**GAPS[gap]), groups)
            out.append(dict(gap=gap, schedule=sched, ring=[rr, rc], buf_cells=buf))
    os.environ.pop("ABPOA_GPU_CHAIN_ROUNDS", None)
    return out


@pytest.mark.gpu
def test_chain_windowed_recompute_small_ring():
    """ABPOA_GPU_SMEM_KB=5: the chain's ring is two rows of at most 64 cells, so its recompute buffer (at most 768 / 512
    cells) is narrower than the inserted runs; the chain must return what the launch engine returns, with no group handed
    back."""
    runs = child({"ABPOA_GPU_SMEM_KB": "5"}, ["windowed"])
    assert {(r["gap"], r["schedule"]) for r in runs} == {(g, s) for g in GAPS for s in ("free-running", "rounds")}, runs


# ------------------------------------------------------------------------------- CPU: the shapes still hold what the GPU tests rely on
def oracle_shape(cfg_kw: dict, reads) -> dict:
    """On the oracle alone: widest row (cells), longest insertion op of any read's path, most predecessors of a row
    at alignment time, rows whose band starts off the 8-cell grid."""
    from oracle_binding import oracle_align
    out = dict(max_cells=0, max_ins=0, max_pred=0, off_grid=0)
    with PoaSession(PoaConfig(**cfg_kw), capi.product()) as s:
        s.reset(max(len(r) for r in reads))
        for r in reads:
            g = s.ab.contents.abg.contents
            out["max_pred"] = max(out["max_pred"], max(g.node[k].in_edge_n for k in range(g.node_n)))
            bands = []

            def cb(user, row, beg, end, *planes):
                bands.append((beg, end))
            o, res = oracle_align(s, r, row_cb=cb)
            out["max_cells"] = max([out["max_cells"]] + [e - b + 1 for b, e in bands])
            out["off_grid"] += sum(1 for b, e in bands if e >= b and b & 7)
            for w in o.cigar[1:-1]:                    # a path's first / last op is no insertion step of a row
                if int(w) & 0xf == ABPOA_CINS:
                    out["max_ins"] = max(out["max_ins"], (int(w) >> 4) & 0x3fffffff)
            s.add(r, res, len(reads))
    return out


@pytest.mark.parametrize("gap", list(GAPS))
def test_precondition_long_insertions_exceed_the_buffer(gap):
    """Every long-insertion group's path inserts a run longer than the two-row ring's recompute buffer in one row."""
    for grp in long_insert_groups(gap):
        sh = oracle_shape(GAPS[gap], grp)
        assert sh["max_ins"] > SMALL_RING_BUF[gap], (gap, sh)
    cfg, make = CASES[f"{gap}_long_insert"]
    sh = oracle_shape(cfg, make())
    assert sh["max_ins"] > SMALL_RING_BUF[gap], (gap, sh)


@pytest.mark.parametrize("gap", list(GAPS))
def test_precondition_wide_bands(gap):
    """wb = 1000 rows are wider than 768 cells (more than three 256-cell passes); wf = 0.1 at 3 kbp rows span two passes."""
    sh = oracle_shape(CASES[f"{gap}_wb1000"][0], CASES[f"{gap}_wb1000"][1]())
    assert sh["max_cells"] > 768 and sh["max_cells"] > SMALL_RING_BUF[gap], sh
    sh = oracle_shape(CASES[f"{gap}_wf01_3k"][0], CASES[f"{gap}_wf01_3k"][1]())
    assert sh["max_cells"] > ONE_PASS, sh


@pytest.mark.parametrize("gap", list(GAPS))
def test_precondition_fan_has_more_than_32_predecessors(gap):
    sh = oracle_shape(CASES[f"{gap}_fan"][0], CASES[f"{gap}_fan"][1]())
    assert sh["max_pred"] > 32, sh


def test_precondition_insertion_bands_off_the_grid():
    """Some insertion shape has rows whose band starts inside an 8-cell group (fb_recompute's lane-0 left neighbour rule)."""
    for gap in GAPS:
        for shape in ("run_lengths", "many_runs"):
            sh = oracle_shape(CASES[f"{gap}_{shape}"][0], CASES[f"{gap}_{shape}"][1]())
            assert sh["off_grid"] > 0 and sh["max_ins"] > 0, (gap, shape, sh)


@pytest.mark.parametrize("name", WINDOW_POINTS)
def test_precondition_window_points_stay_on_the_packed_kernel(name):
    """The score-window points admitted to the packed kernel on every read, none tripping its run-time guard."""
    cfg, reads = sw.point(name)
    alns = sw.profile(cfg, reads, capi.product())
    assert alns and all(a.packed and not a.guard for a in alns), name


if __name__ == "__main__":
    for arg in sys.argv[1:]:
        if arg == "windowed":
            for r in windowed_in_chain():
                print("[run] " + json.dumps(r), flush=True)
        else:
            run_case(arg)
