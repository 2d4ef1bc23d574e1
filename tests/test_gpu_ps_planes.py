"""The chain's path-score (-G) job function cell by cell against the scalar oracle (tests/planes.py).

-G batches run p16_run_job<GAP, GLOBAL, LEAN, no TMA, FB, PS>: predecessor k's path score is added to its diagonal term
(and with it to the backtrace shortcut bits) and to its E planes, on the straight-line rows of up to 4 predecessors, on
the general rows and in the backtrace's F-plane recompute.  The launch engine aligns the same reads with its five-plane
-G kernel; every alignment is replayed on the chain's path-score instantiation (poa_debug_chain_replay picks it from the
blob's predscore section) and checked as tests/test_gpu_chain_planes.py checks the chain's plain job function: score,
end points and graph-CIGAR against the oracle, the compact H / E planes and the recomputed F planes and decision bytes
against the oracle and bit for bit against the five-plane run, with the chain's ring and with a two-row ring of 64
cells.  The cases cover lean rows, rows of more than 4 (and 32) predecessors, and insertion runs longer than the
recompute buffer (the windowed recompute)."""
from __future__ import annotations

import pytest

from abpoa_b200 import synth
from abpoa_b200.aligner import PoaConfig
from helpers import deletion_fan
from planes import run_planes
from test_gpu_chain_planes import GAPS, Checker, long_insert_groups, oracle_shape
from test_gpu_chain_recompute import run_length_group

CASES = {}
for g in GAPS:
    s = 0 if g == "CG" else 1
    CASES[f"{g}_lean"] = (dict(GAPS[g]), lambda s=s: synth.make_group(9600 + s, 8, 500, 0.06))
    CASES[f"{g}_error25"] = (dict(GAPS[g]), lambda s=s: synth.make_group(9610 + s, 8, 400, 0.25))        # rows of > 4 predecessors
    CASES[f"{g}_fan"] = (dict(GAPS[g]), lambda s=s: deletion_fan(seed=7 + 2 * s, n=40 + 10 * s))           # rows of > 32 predecessors
    CASES[f"{g}_run_lengths"] = (dict(GAPS[g]), lambda s=s: run_length_group(9630 + s, 8, 600))
    CASES[f"{g}_long_insert"] = (dict(GAPS[g]), lambda g=g: [r for grp in long_insert_groups(g) for r in grp[:2]])


class PsChecker(Checker):
    """Checker of tests/test_gpu_chain_planes.py on -G alignments: the launch engine runs them on its general (not LEAN)
    packed kernel; the replay is the chain's path-score instantiation."""

    def check(self, i, info):
        self.i = i
        assert info.kernel == 15 and not info.lean, f"{self.name} read {i}: kernel {info.name} lean={info.lean}: not the packed -G kernel"


def run_case(name: str) -> dict:
    cfg_kw, make = CASES[name]
    cfg = PoaConfig(**cfg_kw, inc_path_score=True)
    reads = make()
    ck = PsChecker(name, cfg, reads)
    run_planes(cfg, reads, tag=name, check=ck.check, after=ck)
    lg = ck.log
    assert lg["reads"], f"{name}: no alignment ran"
    print(f"[ps-planes] {name}: {lg['reads']} alignments, rings {sorted(lg['geoms'])}, buf_cells {sorted(lg['bufs'])}, "
          f"{lg['windows']} recompute windows (at most {lg['max_windows']} in one row)")
    return lg


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_ps_chain_planes(name):
    lg = run_case(name)
    if "long_insert" in name:
        assert lg["max_windows"] > 1, f"{name}: no row needed a second recompute window"


@pytest.mark.parametrize("gap", list(GAPS))
def test_precondition_many_predecessors(gap):
    """On the oracle alone: the high-error groups have rows of more than 4 predecessors, the fans of more than 32."""
    assert oracle_shape(*_shape_args(f"{gap}_error25"))["max_pred"] > 4
    assert oracle_shape(*_shape_args(f"{gap}_fan"))["max_pred"] > 32


def _shape_args(name):
    cfg_kw, make = CASES[name]
    return dict(cfg_kw, inc_path_score=True), make()
