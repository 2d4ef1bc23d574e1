"""The chain engine's compact DP-row layout: its packed kernel stores H and the E planes, and instead of the F planes one
byte per cell with the outcomes of the backtrace's insertion-step comparisons, computed in the forward pass.  The launch
engine keeps the five-plane layout, which tests/test_gpu_planes.py pins cell by cell against the scalar oracle, so it is
the reference here: on shapes where the backtrace takes many insertion steps -- long inserted runs, insertions at the
first cell of a band, bands wider than one 256-cell pass (the byte of a pass's first cell needs the previous pass's last
cell) -- both engines must return identical records."""
import numpy as np
import pytest

from abpoa_b200 import synth
from abpoa_b200.aligner import PoaConfig
from abpoa_b200.batch import BatchEngine
from cases import AFFINE

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True, params=["free-running", "rounds"])
def chain_mode(request, monkeypatch):
    if request.param == "rounds":
        monkeypatch.setenv("ABPOA_GPU_CHAIN_ROUNDS", "1")
    else:
        monkeypatch.delenv("ABPOA_GPU_CHAIN_ROUNDS", raising=False)
    return request.param


def insertion_heavy_group(seed: int, n_reads: int, length: int, err: float) -> list[np.ndarray]:
    """A synthetic group whose reads carry one or two extra inserted runs of 2-20 bases, some at the read's start or end
    (few enough that the graph stays within the chain's node capacity of 10 % growth per read)."""
    rng = np.random.default_rng(seed)
    out = []
    for i, r in enumerate(synth.make_group(seed, n_reads, length, err)):
        if i == 0:
            out.append(r)
            continue
        pieces, at = [], 0
        cuts = np.sort(rng.choice(len(r) + 1, size=int(rng.integers(1, 3)), replace=False))
        if rng.random() < 0.3:
            cuts[0] = 0
        if rng.random() < 0.3:
            cuts[-1] = len(r)
        for c in cuts:
            pieces.append(r[at:c])
            pieces.append(rng.integers(0, 4, size=int(rng.integers(2, 21))).astype(r.dtype))
            at = c
        pieces.append(r[at:])
        out.append(np.concatenate(pieces))
    return out


def assert_engines_agree(cfg, groups):
    with BatchEngine() as eng:
        a = eng.run(cfg, groups, record_reads=True)
        sa = eng.stats()
        eng.reset_stats()
        b = eng.run(cfg, groups, record_reads=True, no_chain=True)
        sb = eng.stats()
    assert sa["chain_groups"] == len(groups) and sa["chain_fallback_groups"] == 0 and sb["chain_groups"] == 0, (sa, sb)
    for gi, (x, y) in enumerate(zip(a, b)):
        assert x.dp_cells == y.dp_cells, gi
        assert np.array_equal(x.read_best_score[1:], y.read_best_score[1:]), gi
        assert np.array_equal(x.read_n_cigar[1:], y.read_n_cigar[1:]) and np.array_equal(x.read_cigar_hash[1:], y.read_cigar_hash[1:]), gi
        assert all(np.array_equal(p, q) for p, q in zip(x.cons, y.cons)), gi
        assert all(np.array_equal(p, q) for p, q in zip(x.cov, y.cov)), gi


@pytest.mark.parametrize("gap", ["convex", "affine"])
def test_chain_layout_insertion_heavy(gap):
    cfg = PoaConfig(**({} if gap == "convex" else AFFINE))
    groups = [insertion_heavy_group(7100 + g, 6 + g % 4, 800 + 60 * g, 0.03 + 0.01 * (g % 2)) for g in range(8)]
    assert_engines_agree(cfg, groups)


@pytest.mark.parametrize("gap", ["convex", "affine"])
def test_chain_layout_bands_wider_than_one_pass(gap):
    """w = 10 + 0.1 * 3000: every row spans two or three passes of 256 cells."""
    cfg = PoaConfig(wf=0.1, **({} if gap == "convex" else AFFINE))
    groups = [insertion_heavy_group(7300 + g, 5, 3000, 0.06) for g in range(3)]
    assert_engines_agree(cfg, groups)
