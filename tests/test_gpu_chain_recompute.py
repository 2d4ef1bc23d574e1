"""The chain engine's packed kernel stores no F planes: the backtrace recomputes a row's F planes from the predecessors'
H / E planes the first time its insertion step needs them in that row.  The launch engine keeps all five planes and is
pinned cell by cell against the scalar oracle (tests/test_gpu_planes.py), so it is the reference here: on shapes that send
the backtrace through that recompute in every corner -- inserted runs on both sides of the convex crossover (~20 bases,
where F2 takes over from F1), several runs per read, runs at a read's ends and at a band's first cell, runs in the
second or third 256-cell pass of a wide band, and rows with more than 4 and more than 32 predecessors -- both engines
must return identical records, and no group may fall back to the launch engine."""
import numpy as np
import pytest

from abpoa_b200 import synth
from abpoa_b200.aligner import PoaConfig
from cases import AFFINE
from helpers import deletion_fan
from test_gpu_chain_layout import assert_engines_agree, chain_mode  # noqa: F401  (autouse fixture: both chain schedules)

pytestmark = pytest.mark.gpu

GAPS = {"convex": {}, "affine": AFFINE}


def insert_runs(read: np.ndarray, rng, lengths, where=None) -> np.ndarray:
    """`read` with one random run per entry of `lengths` inserted at the positions `where` (random if None)."""
    pos = np.sort(rng.choice(len(read) + 1, size=len(lengths), replace=True) if where is None else np.asarray(where))
    pieces, at = [], 0
    for p, n in zip(pos, lengths):
        pieces += [read[at:p], rng.integers(0, 4, size=int(n)).astype(read.dtype)]
        at = p
    pieces.append(read[at:])
    return np.concatenate(pieces)


def run_length_group(seed: int, n_reads: int, length: int) -> list[np.ndarray]:
    """Every read after the first carries one inserted run; the lengths sweep 1..60 bases across the group."""
    rng = np.random.default_rng(seed)
    reads = synth.make_group(seed, n_reads, length, 0.02)
    return [reads[0]] + [insert_runs(r, rng, [1 + (7 * (seed + k)) % 60]) for k, r in enumerate(reads[1:])]


def many_runs_group(seed: int, n_reads: int, length: int) -> list[np.ndarray]:
    """Three to five runs of 1-30 bases per read, some at the first and the last base."""
    rng = np.random.default_rng(seed)
    out = []
    for k, r in enumerate(synth.make_group(seed, n_reads, length, 0.03)):
        if k == 0:
            out.append(r)
            continue
        n = int(rng.integers(3, 6))
        where = rng.choice(len(r) + 1, size=n, replace=True)
        if k % 3 == 1:
            where[0] = 0
        if k % 3 == 2:
            where[-1] = len(r)
        out.append(insert_runs(r, rng, rng.integers(1, 31, size=n), where))
    return out


@pytest.mark.parametrize("gap", list(GAPS))
def test_recompute_run_lengths(gap):
    groups = [run_length_group(8100 + g, 8, 700 + 50 * g) for g in range(6)]
    assert_engines_agree(PoaConfig(**GAPS[gap]), groups)


@pytest.mark.parametrize("gap", list(GAPS))
def test_recompute_several_runs_and_read_ends(gap):
    groups = [many_runs_group(8200 + g, 7, 600 + 40 * g) for g in range(6)]
    assert_engines_agree(PoaConfig(**GAPS[gap]), groups)


@pytest.mark.parametrize("gap", list(GAPS))
def test_recompute_later_passes_of_wide_bands(gap):
    """w = 10 + 0.1 * 3000: every row spans two or three passes of 256 cells, and runs land in all of them."""
    rng = np.random.default_rng(8300)
    groups = []
    for g in range(3):
        reads = synth.make_group(8300 + g, 5, 3000, 0.04)
        groups.append([reads[0]] + [insert_runs(r, rng, rng.integers(1, 41, size=4)) for r in reads[1:]])
    assert_engines_agree(PoaConfig(wf=0.1, **GAPS[gap]), groups)


@pytest.mark.parametrize("gap", list(GAPS))
def test_recompute_rows_with_many_predecessors(gap, monkeypatch):
    """deletion_fan: the node after the deleted stretch collects one in-edge per read (up to 39 predecessors).  Reads that
    insert a run right after that node make the backtrace recompute its row; smaller fans give rows with 5-8 predecessors.
    The chain's graph keeps ABPOA_GPU_CHAIN_K in-edges per node inline (12 by default): 48 lets the large fan stay on it."""
    monkeypatch.setenv("ABPOA_GPU_CHAIN_K", "48")
    rng = np.random.default_rng(8400)
    groups = []
    for n, flank in ((40, 220), (9, 160)):
        fan = deletion_fan(seed=8400 + n, n=n, flank=flank)
        t = fan[0]
        extra = [np.concatenate([t[: flank - k], t[flank: flank + 1], rng.integers(0, 4, size=L).astype(t.dtype), t[flank + 1:]])
                 for k, L in ((1, 3), (n // 2, 12), (n - 1, 25))]
        groups.append(fan + extra)
    assert_engines_agree(PoaConfig(**GAPS[gap]), groups)
