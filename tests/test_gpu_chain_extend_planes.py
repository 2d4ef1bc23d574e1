"""The chain's extend (-m 2) job function cell by cell against the scalar oracle (tests/planes.py).

Extend batches run p16_run_job<GAP, EXTEND, LEAN, no TMA, FB, PS> (chain_align_read's EXT instantiation): the straight-line
rows and compact layout of global jobs, then the best cell (the first row that holds the maximum, its rightmost arg-max)
and the z-drop stop.  The launch engine aligns the same reads with its general five-plane packed kernel; every alignment
is replayed on the chain's EXTEND instantiation (poa_debug_chain_replay picks it for a banded whole-graph extend job) and
checked as tests/test_gpu_chain_planes.py checks the chain's global job function: score, end points and graph-CIGAR
against the oracle, row bands, the compact H / E planes and the recomputed F planes and decision bytes against the oracle
and bit for bit against the five-plane run, with the chain's ring and with a two-row ring of 64 cells.  Where z-drop
fires, only the rows up to the oracle's stop row are compared, and the replay's DP cells must be those rows' cells: the
replay stopped at the oracle's row.  Affine and convex gaps, with and without -G."""
from __future__ import annotations

import copy

import pytest

from abpoa_b200 import synth
from abpoa_b200.aligner import PoaConfig
from abpoa_b200.capi import ABPOA_EXTEND_MODE
from planes import chain_replay, fetch_planes, run_planes
from test_gpu_chain_planes import GAPS, ONE_PASS, SMALL_RING, SMALL_RING_BUF, Checker

CASES = {}
for g in GAPS:
    s = 0 if g == "CG" else 1
    CASES[f"{g}_lean"] = (dict(GAPS[g]), lambda s=s: synth.make_group(9700 + s, 8, 500, 0.06))
    CASES[f"{g}_error25"] = (dict(GAPS[g]), lambda s=s: synth.make_group(9710 + s, 8, 400, 0.25))
    CASES[f"{g}_zdrop"] = (dict(GAPS[g], zdrop=10), lambda s=s: synth.make_group(9720 + s, 8, 500, 0.15))


class ExtChecker(Checker):
    """Checker of tests/test_gpu_chain_planes.py on extend alignments: the launch engine runs them on its general (not LEAN)
    packed kernel; the replay is the chain's EXTEND instantiation.  Rows after a z-drop stop were never computed."""

    def __init__(self, *a):
        super().__init__(*a)
        self.stopped = 0

    def check(self, i, info):
        self.i = i
        assert info.kernel == 15 and not info.lean, f"{self.name} read {i}: kernel {info.name} lean={info.lean}: not the packed extend kernel"

    def __call__(self, gpu, rows, info, o):
        """Checker.__call__ with the checks cut at the oracle's last computed row; the planes are fetched and the replay
        run for the whole job (their buffers are sized by its rows)."""
        last = max(r for r in rows if r < info.n_rows - 1)
        cut = info
        if last < info.n_rows - 2:
            self.stopped += 1
            cut = copy.copy(info)
            cut.n_rows = last + 2                                 # rows 0 .. last
            rows = {r: v for r, v in rows.items() if r <= last}
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
                self.log["windows"] += rep.windows
                if k == 0:
                    self.check_replay(gpu, rep, five, rows, cut, o, qlen, tg)
                self.check_f(gpu, rep, five, rows, cut, qlen, tg)


def run_case(name: str, ps: bool) -> ExtChecker:
    cfg_kw, make = CASES[name]
    cfg = PoaConfig(align_mode=ABPOA_EXTEND_MODE, inc_path_score=ps, **cfg_kw)
    reads = make()
    ck = ExtChecker(name, cfg, reads)
    run_planes(cfg, reads, tag=name, check=ck.check, after=ck)
    lg = ck.log
    assert lg["reads"], f"{name}: no alignment ran"
    print(f"[ext-planes] {name} ps={ps}: {lg['reads']} alignments ({ck.stopped} stopped by z-drop), rings {sorted(lg['geoms'])}, "
          f"buf_cells {sorted(lg['bufs'])}, {lg['windows']} recompute windows")
    return ck


@pytest.mark.gpu
@pytest.mark.parametrize("ps", [False, True])
@pytest.mark.parametrize("name", list(CASES))
def test_extend_chain_planes(name, ps):
    ck = run_case(name, ps)
    if name.endswith("zdrop"):
        assert ck.stopped >= 2, f"{name}: z-drop stopped {ck.stopped} alignments"
