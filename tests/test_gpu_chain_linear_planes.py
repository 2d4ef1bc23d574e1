"""The chain's linear-gap job function cell by cell (tests/planes.py).

Linear-gap batches run p16_run_job<LG, GLOBAL, LEAN, no TMA, FB, PS, LGX>: banded rows follow the reference's vector
procedure (SURVEY 8a a7) -- stored in whole pn-lane vectors around the band, the cells right of `end` keep the running
value and successors read them, predecessor p feeds the cells below ((p.end + 1) / pn + 1) * pn only, and past the
predecessors' last vector only the even lanes of the next one keep the running value.  A single alignment through
abpoa.h runs on the generic kernel's "lgx" rows, which run_planes checks against the scalar oracle (lg_vector_row) row
by row.  Every such alignment is then replayed on the chain's job function (poa_debug_chain_replay), with the chain's
ring and with a two-row ring of 64 cells (rows wider than a ring slot: the straight-line path is refused and the general
rows read the predecessors from HBM), and:
  1. the replay's status, score, end points and graph-CIGAR equal the oracle's
  2. its row records (band, first / last arg-max) and its cell count / widest band equal the generic kernel's
  3. inside every band, each H cell equals the oracle's; cells the oracle holds minus infinity sit at or below the
     packed kernel's floor
  4. every STORED H cell of every row -- the whole vectors around the band, leaked cells included -- equals the generic
     kernel's lgx plane wherever that plane holds a finite value, and sits at or below the packed floor where the generic
     kernel holds minus infinity
  5. the slab takes exactly the rows' stored vectors (plane_units_used)
Inputs: a qlen sweep, short and long reads, 25 % error, a deletion fan (rows of more than 32 predecessors), BLOSUM62,
and the two vector widths (pn = 16 and pn = 8)."""
from __future__ import annotations

import numpy as np
import pytest

import score_window as sw
from abpoa_b200 import synth
from abpoa_b200.aligner import PoaConfig
from cases import LINEAR
from helpers import deletion_fan
from planes import FLOOR, ORACLE_NINF, chain_replay, fetch_planes, run_planes, score_bits
from test_gpu_chain_planes import oracle_shape
from test_gpu_planes import qlen_sweep, short_long

SMALL_RING = (2, 64)
PACKED_FLOOR = FLOOR[15]
E20 = dict(gap_open1=0, gap_ext1=20, gap_open2=0, gap_ext2=0)
AA = {k: v for k, v in synth.WORKLOADS["aa_blosum62_2k"].cfg.__dict__.items() if k not in LINEAR}

CASES = {
    "qlen_sweep": (dict(LINEAR), lambda: qlen_sweep(2400)),
    "short_long": (dict(LINEAR), lambda: short_long(2410)),
    "error25": (dict(LINEAR), lambda: synth.make_group(2420, 8, 400, 0.25)),
    "narrow_band": (dict(LINEAR, wb=6, wf=0.01), lambda: synth.make_group(2430, 8, 500, 0.15)),
    "fan": (dict(LINEAR), lambda: deletion_fan(seed=11, n=50)),                  # rows of > 32 predecessors
    "blosum62": (dict(LINEAR, **AA), lambda: synth.make_group(2440, 8, 300, 0.08, m=27)),
    "pn16": (dict(E20), sw.with_last(309, 3, 1000, 1637)),                     # score-window points: the reference's
    "pn8": (dict(E20), sw.with_last(309, 3, 1000, 1638)),                      # int16 / int32 vector widths
}
# cases with rows wider than the two-row ring's 64-cell slot (the others' bands fit it)
WIDE = {"qlen_sweep", "short_long", "fan", "pn16", "pn8"}


def stored_groups(beg, end, xs):
    g0 = ((beg >> xs) << xs) >> 3
    return g0, (((((end >> xs) + 1) << xs) - 1) >> 3) - g0 + 1


class Checker:
    def __init__(self, name, cfg, reads):
        self.name, self.cfg, self.reads = name, cfg, reads
        self.i = -1
        self.log = dict(reads=0, geoms=set(), pn=set(), leaked=0, small_ring_wide_rows=0)

    def check(self, i, info):
        self.i = i
        assert info.kernel in (16, 32), f"{self.name} read {i}: kernel {info.name}: not the generic kernel's lgx rows"

    def __call__(self, gpu, rows, info, o):
        qlen = len(self.reads[self.i])
        t0 = f"{self.name} read {self.i} (qlen {qlen})"
        ri5, ro5, slab5 = fetch_planes(gpu, info)
        xs = 4 if score_bits(gpu.abpt, qlen, info.n_rows) == 16 else 3
        self.log["pn"].add(1 << xs)
        self.log["reads"] += 1
        floor5 = FLOOR[info.kernel]
        n = info.n_rows - 1
        for geom in ((0, 0), SMALL_RING):
            rep = chain_replay(gpu, info, qlen, *geom)
            t = f"{t0} ring {rep.ring_rows}x{rep.ring_cells}"
            self.log["geoms"].add((rep.ring_rows, rep.ring_cells))
            assert rep.status == 0, f"{t}: replay status {rep.status}"
            assert rep.best_score == o.best_score, f"{t}: score {rep.best_score}, oracle {o.best_score}"
            assert rep.ends == (o.node_s, o.node_e, o.query_s, o.query_e), f"{t}: end points {rep.ends}"
            assert rep.n_ops == len(o.cigar) and np.array_equal(rep.cigar, o.cigar), f"{t}: graph-CIGAR differs from the oracle"
            assert np.array_equal(rep.rowinfo[:n], ri5[:n]), f"{t}: row records differ from the generic kernel's"
            w5 = ri5[:n, 1].astype(np.int64) - ri5[:n, 0] + 1
            assert rep.cells == int(w5[w5 > 0].sum()) and rep.max_band == int(w5.max()), f"{t}: cells / max_band {rep.cells} / {rep.max_band}"
            units = 0
            for r in range(n):
                beg, end = int(rep.rowinfo[r, 0]), int(rep.rowinfo[r, 1])
                if end < beg:
                    continue
                g0, ngrp = stored_groups(beg, end, xs)
                units += ngrp
                if geom == SMALL_RING and ngrp > SMALL_RING[1] // 8:
                    self.log["small_ring_wide_rows"] += 1
                got = rep.slab[int(rep.rowoff[r]) * 8: int(rep.rowoff[r]) * 8 + ngrp * 8].astype(np.int64)
                want = slab5[int(ro5[r]) * 8: int(ro5[r]) * 8 + ngrp * 8].astype(np.int64)
                fin = want > floor5
                bad = np.flatnonzero((fin & (got != want)) | (~fin & (got > PACKED_FLOOR)))
                if len(bad):
                    j = int(bad[0])
                    raise AssertionError(f"{t}: row {r} stored cell {g0 * 8 + j}: chain {int(got[j])}, generic lgx "
                                         f"{int(want[j]) if fin[j] else '-inf'} (band {beg}..{end}, {len(bad)} cells differ)")
                hi = g0 * 8 + ngrp * 8 - 1
                self.log["leaked"] += int(fin[end - g0 * 8 + 1:].sum()) if end < hi else 0
                if r in rows:
                    ob, oe, pl = rows[r]
                    assert (ob, oe) == (beg, end), f"{t}: row {r} band ({beg},{end}), oracle ({ob},{oe})"
                    h, band = pl[0], got[beg - g0 * 8: end - g0 * 8 + 1]
                    ofin = h > ORACLE_NINF // 2
                    bad = np.flatnonzero((ofin & (band != h)) | (~ofin & (band > PACKED_FLOOR)))
                    if len(bad):
                        j = int(bad[0])
                        raise AssertionError(f"{t}: row {r} column {beg + j}: chain {int(band[j])}, oracle "
                                             f"{int(h[j]) if ofin[j] else '-inf'}")
            assert rep.plane_units_used == units, f"{t}: plane_units_used {rep.plane_units_used}, stored vectors take {units}"


def run_case(name):
    cfg_kw, make = CASES[name]
    cfg = PoaConfig(**cfg_kw)
    reads = make()
    ck = Checker(name, cfg, reads)
    run_planes(cfg, reads, tag=name, check=ck.check, after=ck)
    lg = ck.log
    assert lg["reads"], f"{name}: no alignment ran"
    print(f"[linear-planes] {name}: {lg['reads']} alignments, pn {sorted(lg['pn'])}, rings {sorted(lg['geoms'])}, "
          f"{lg['leaked']} finite leaked cells compared, {lg['small_ring_wide_rows']} rows wider than the small ring")
    return lg


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_linear_chain_planes(name):
    lg = run_case(name)
    assert lg["leaked"] > 0, f"{name}: no finite leaked cell right of a band was compared"
    if name in WIDE:
        assert lg["small_ring_wide_rows"] > 0, f"{name}: no row wider than the two-row ring's slot"
    if name in ("pn16", "pn8"):
        assert {"pn16": 16, "pn8": 8}[name] in lg["pn"], f"{name}: vector width {lg['pn']}"


def test_precondition_fan_has_more_than_32_predecessors():
    """On the oracle alone: the linear deletion fan has rows of more than 32 predecessors."""
    cfg_kw, make = CASES["fan"]
    assert oracle_shape(cfg_kw, make())["max_pred"] > 32
