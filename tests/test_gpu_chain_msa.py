"""GPU: row-column MSA (-r 1 / -r 2) on the device-resident chain engine (poa_chain.cu: poa_chain_msa_kernel).

Runs that ask for the MSA stay on the chain: the device keeps one read set per node, ranks the graph and writes the rows;
only the rows (and the consensus) come back.  They must equal the unmodified reference (stored digests,
tests/golden/reference_runs_msa.json, in the format of tests/reference_runs.py) and, field by field, what the launch
engine returns for the same call."""
import json
from pathlib import Path

import numpy as np
import pytest

from abpoa_b200 import synth
from abpoa_b200.aligner import PoaConfig
from abpoa_b200.batch import BatchEngine
from cases import AFFINE
from reference_runs import Reference, assert_batch_matches

pytestmark = pytest.mark.gpu

STORE_MSA = Path(__file__).resolve().parent / "golden" / "reference_runs_msa.json"


@pytest.fixture(scope="module")
def reference():
    """The unmodified reference's results on this file's inputs; recording works as in tests/reference_runs.py."""
    ref = Reference()
    ref.stored = json.loads(STORE_MSA.read_text())
    yield ref
    ref.save()

R1 = dict(out_msa=True, out_cons=False)
R2 = dict(out_msa=True, out_cons=True)


@pytest.fixture(autouse=True, params=["free-running", "rounds"])
def chain_mode(request, monkeypatch):
    """Every test runs on both schedules of the chain engine (see test_gpu_chain.py)."""
    if request.param == "rounds":
        monkeypatch.setenv("ABPOA_GPU_CHAIN_ROUNDS", "1")
    else:
        monkeypatch.delenv("ABPOA_GPU_CHAIN_ROUNDS", raising=False)
    return request.param


# ---- inputs (tests/golden/reference_runs.json holds the reference's digests of the ones checked against it) ----
def kind_cfg(kind, out):
    if kind == "aa":
        return PoaConfig(**{**synth.WORKLOADS["aa_blosum62_2k"].cfg.__dict__, **out})
    return PoaConfig(**({} if kind == "convex" else AFFINE), **out)


def kind_groups(kind):
    if kind == "aa":
        return [synth.make_group(8100 + g, 10, 500, 0.10, m=27) for g in range(6)]
    seed = 8000 if kind == "convex" else 8050
    return [synth.make_group(seed + g, 6 + g % 5, 300 + 50 * (g % 6), 0.04 + 0.01 * (g % 5)) for g in range(12)]


def word_edge_groups():
    return [synth.make_group(8200 + n, n, 150, 0.06) for n in (64, 65, 130)]


def mixed_groups():
    """Ragged groups, a 2-read group, a 1-read group and an empty group (the last two never reach the chain)."""
    rng = np.random.default_rng(17)
    groups = []
    for g in range(8):
        base = synth.make_group(8300 + g, 3 + 2 * (g % 4), 700, 0.06)
        groups.append([np.ascontiguousarray(r[: int(rng.integers(5, len(r)))]) if i % 3 == 1 else r for i, r in enumerate(base)])
    groups += [synth.make_group(8320, 2, 400, 0.05), synth.make_group(8321, 1, 90, 0.0), []]
    return groups


REFERENCE_INPUTS = {f"{kind}-{r}": (lambda kind=kind, out=out: (kind_cfg(kind, out), kind_groups(kind)))
                    for kind in ("convex", "affine", "aa") for r, out in (("r1", R1), ("r2", R2))}
REFERENCE_INPUTS["word-edges-r2"] = lambda: (PoaConfig(**R2), word_edge_groups())
REFERENCE_INPUTS["mixed-r1"] = lambda: (PoaConfig(**R1), mixed_groups())
REFERENCE_INPUTS["mixed-r2"] = lambda: (PoaConfig(**R2), mixed_groups())


# ---- helpers ----
def run(cfg, groups, **kw):
    with BatchEngine() as eng:
        got = eng.run(cfg, groups, record_reads=True, **kw)
        st = eng.stats()
    return got, st


def assert_same_records(a, b, groups):
    """Chain vs launch engine, field by field."""
    for gi, (x, y, g) in enumerate(zip(a, b, groups)):
        tag = f"group {gi}"
        assert len(x.msa) == len(y.msa), f"{tag}: n_msa_rows {len(x.msa)} vs {len(y.msa)}"
        if x.msa:
            assert len(x.msa[0]) == len(y.msa[0]), f"{tag}: msa_len {len(x.msa[0])} vs {len(y.msa[0])}"
        for k, (p, q) in enumerate(zip(x.msa, y.msa)):
            assert np.array_equal(p, q), f"{tag}: MSA row {k} differs at column {int(np.argmax(p != q))}"
        assert len(x.cons) == len(y.cons) and all(np.array_equal(p, q) for p, q in zip(x.cons, y.cons)), f"{tag}: consensus"
        assert all(np.array_equal(p, q) for p, q in zip(x.cov, y.cov)), f"{tag}: coverage"
        assert x.dp_cells == y.dp_cells and x.n_aligned == y.n_aligned, f"{tag}: DP cells / aligned reads"
        if len(g) > 1:
            assert np.array_equal(x.read_best_score[1:], y.read_best_score[1:]), f"{tag}: per-read scores"
            assert np.array_equal(x.read_n_cigar[1:], y.read_n_cigar[1:]), f"{tag}: per-read CIGAR lengths"
            assert np.array_equal(x.read_cigar_hash[1:], y.read_cigar_hash[1:]), f"{tag}: per-read CIGAR hashes"


def n_chainable(groups):
    return sum(1 for g in groups if len(g) >= 2)


# ---- tests ----
@pytest.mark.parametrize("name", [k for k in REFERENCE_INPUTS if not k.startswith("mixed")])
def test_chain_msa_matches_reference(reference, name):
    cfg, groups = REFERENCE_INPUTS[name]()
    got, st = run(cfg, groups)
    assert_batch_matches(got, groups, reference.batch(cfg, groups, want_msa=True), tag=name)
    assert st["chain_groups"] == len(groups) and st["chain_fallback_groups"] == 0, st
    for r, g in zip(got, groups):
        assert len(r.msa) == len(g) + int(cfg.out_cons)


@pytest.mark.parametrize("out", ["r1", "r2"])
def test_chain_msa_mixed_groups_in_one_call(reference, out):
    cfg, groups = REFERENCE_INPUTS[f"mixed-{out}"]()
    got, st = run(cfg, groups)
    assert_batch_matches(got, groups, reference.batch(cfg, groups, want_msa=True), tag=out)
    assert st["chain_groups"] == n_chainable(groups) and st["chain_fallback_groups"] == 0, st
    want, _ = run(cfg, groups, no_chain=True)
    assert_same_records(got, want, groups)


@pytest.mark.parametrize("out", ["r1", "r2"])
@pytest.mark.parametrize("kind", ["convex", "affine", "aa"])
def test_chain_msa_equals_launch_engine(kind, out):
    cfg, groups = kind_cfg(kind, R1 if out == "r1" else R2), kind_groups(kind)
    a, sa = run(cfg, groups)
    b, sb = run(cfg, groups, no_chain=True)
    assert sa["chain_groups"] == len(groups) and sb["chain_groups"] == 0
    assert_same_records(a, b, groups)


def test_chain_msa_word_edges_equal_launch_engine():
    """64, 65 and 130 reads: read sets of one, two and three words in one wave (W = 3 for all of them)."""
    groups = word_edge_groups()
    for out in (R1, R2):
        a, sa = run(PoaConfig(**out), groups)
        b, _ = run(PoaConfig(**out), groups, no_chain=True)
        assert sa["chain_groups"] == 3 and sa["chain_fallback_groups"] == 0, sa
        assert_same_records(a, b, groups)


def test_chain_msa_groups_handed_back(monkeypatch):
    """Two edge slots per node: most groups leave the chain and are finished by the launch engine -- same rows."""
    groups = [synth.make_group(8400 + g, 8, 400, 0.10) for g in range(10)]
    cfg = PoaConfig(**R2)
    b, _ = run(cfg, groups, no_chain=True)
    monkeypatch.setenv("ABPOA_GPU_CHAIN_K", "2")
    a, sa = run(cfg, groups)
    assert sa["chain_fallback_groups"] > 0 and sa["chain_groups"] + sa["chain_fallback_groups"] == 10, sa
    assert_same_records(a, b, groups)


def test_chain_msa_with_graph_export(monkeypatch):
    """ABPOA_GPU_CHAIN_EXPORT_GRAPH=1: the host rebuilds the graph and computes the consensus on it; the rows are still the
    device's.  Both must equal the launch engine's."""
    groups = [synth.make_group(8500 + g, 9, 450, 0.08) for g in range(6)]
    cfg = PoaConfig(**R2)
    b, _ = run(cfg, groups, no_chain=True)
    monkeypatch.setenv("ABPOA_GPU_CHAIN_EXPORT_GRAPH", "1")
    a, sa = run(cfg, groups)
    assert sa["chain_groups"] == 6 and sa["chain_fallback_groups"] == 0, sa
    assert_same_records(a, b, groups)


def test_chain_msa_headline_shape():
    """4 groups of the headline shape (50 x 10 kbp, convex) with -r 2: all on the chain, rows equal to the launch engine's."""
    wl = synth.WORKLOADS["convex_10k"]
    cfg = PoaConfig(**{**wl.cfg.__dict__, **R2})
    groups = wl.groups(4)
    a, sa = run(cfg, groups)
    assert sa["chain_groups"] == 4 and sa["chain_fallback_groups"] == 0, sa
    b, _ = run(cfg, groups, no_chain=True)
    assert_same_records(a, b, groups)
