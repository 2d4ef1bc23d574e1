"""GPU: quality weights (-Q) on the device-resident chain engine.

Every base's weight is added to the graph edge that enters its node (chain_seed / chain_fuse, poa_chain.cuh); the weights
go up with the reads, one byte per base.  Batches with weights must stay on the chain and give the unmodified reference's
per-read scores, CIGARs, consensus, coverage and MSA rows (tests/golden/reference_runs_qv.json, see
tests/qv_reference.py), and the launch engine's records and text field by field.  A group with a weight that does not
fit a byte is finished by the launch engine, with the same results."""
import subprocess
from pathlib import Path

import numpy as np
import pytest

from abpoa_b200 import synth
from abpoa_b200.aligner import make_para
from abpoa_b200.batch import BatchEngine, PackedGroups
from abpoa_b200.capi import product
from gfa_reference import md5, reference_cli_md5, with_file
from mf_reference import set_outputs
from qv_reference import (BATCH_KINDS, CLI_LIST_OPTS, TEXT_R, fastq_files, group_weights, kind_cfg, kind_groups, quality_weights,
                          qv_cfg, qv_reference, reference_group, result_digest, unit_filled)
from reference_runs import assert_batch_matches
from test_gpu_chain_msa import assert_same_records, run

pytestmark = pytest.mark.gpu

BIN = Path(__file__).resolve().parent.parent / "abpoa_b200" / "bin" / "abpoa"


@pytest.fixture(scope="module")
def reference():
    ref = qv_reference()
    yield ref
    ref.save()


@pytest.fixture(autouse=True, params=["free-running", "rounds"])
def chain_mode(request, monkeypatch):
    """Every test runs on both schedules of the chain engine (see test_gpu_chain.py)."""
    if request.param == "rounds":
        monkeypatch.setenv("ABPOA_GPU_CHAIN_ROUNDS", "1")
    else:
        monkeypatch.delenv("ABPOA_GPU_CHAIN_ROUNDS", raising=False)
    return request.param


def write_text(cfg, groups, weights, r, no_chain=False):
    """abpoa_gpu_msa_batch_write with -r r: (text, results, stats)."""
    lib = product()
    abpt = make_para(lib, cfg)
    set_outputs(lib, abpt, r)
    packed = PackedGroups(groups, weights)
    try:
        with BatchEngine() as eng:
            got = []
            text = with_file(lambda fp: got.extend(eng.run_write(abpt, packed, fp, record_reads=True, no_chain=no_chain)))
            st = eng.stats()
    finally:
        lib.abpoa_free_para(abpt)
    return text, got, st


# ---- batches against the reference ----
@pytest.mark.parametrize("kind", BATCH_KINDS)
def test_batch_matches_reference(reference, kind):
    cfg = kind_cfg(kind)
    groups, weights = kind_groups(kind)
    got, st = run(cfg, groups, weights=weights)
    assert st["chain_groups"] == len(groups) and st["chain_fallback_groups"] == 0, st
    for gi, (g, w, r) in enumerate(zip(groups, group_weights(groups, weights), got)):
        assert result_digest(r) == reference_group(reference, cfg, g, w)["digest"], f"{kind} group {gi}: consensus, coverage or MSA rows"
    if kind != "strand":        # per-read scores, CIGAR lengths and hashes, DP cells
        gw = [unit_filled(g, w) for g, w in zip(groups, group_weights(groups, weights))]
        assert_batch_matches(got, groups, reference.batch(cfg, groups, want_msa=True, weights=gw), tag=kind)


# ---- the chain against the launch engine ----
@pytest.mark.parametrize("r", TEXT_R)
@pytest.mark.parametrize("kind", BATCH_KINDS)
def test_batch_equals_launch_engine(kind, r):
    """Records and the text abpoa_gpu_msa_batch_write prints, -r 0 / -r 2 / -r 4."""
    cfg = kind_cfg(kind, out_msa=False)
    groups, weights = kind_groups(kind)
    text, a, sa = write_text(cfg, groups, weights, r)
    want, b, sb = write_text(cfg, groups, weights, r, no_chain=True)
    assert sa["chain_groups"] == len(groups) and sa["chain_fallback_groups"] == 0 and sb["chain_groups"] == 0, (sa, sb)
    assert text == want, f"{kind} -r {r}: text differs from the launch engine's"
    for x, y in zip(a, b):
        assert len(x.cons) == len(y.cons) and all(np.array_equal(p, q) for p, q in zip(x.cons, y.cons))
        assert all(np.array_equal(p, q) for p, q in zip(x.cov, y.cov))
        assert x.dp_cells == y.dp_cells and x.n_aligned == y.n_aligned
        assert np.array_equal(x.read_cigar_hash, y.read_cigar_hash) and np.array_equal(x.read_best_score, y.read_best_score)


def test_weights_outside_a_byte_take_the_launch_engine():
    """A group with a weight of 256 and one with a negative weight are finished by the launch engine; the others stay on
    the chain.  Every record equals an all-launch-engine run's."""
    cfg = kind_cfg("convex")
    groups, weights = kind_groups("convex")
    weights[2][1][7] = 256
    weights[5][0][0] = -3
    a, sa = run(cfg, groups, weights=weights)
    b, sb = run(cfg, groups, weights=weights, no_chain=True)
    assert sa["chain_groups"] == len(groups) - 2 and sa["chain_fallback_groups"] == 0 and sb["chain_groups"] == 0, (sa, sb)
    assert_same_records(a, b, groups)


@pytest.mark.parametrize("r", [0, 2])
def test_groups_handed_back(monkeypatch, r):
    """Two edge slots per node: most groups leave the chain and are finished by the launch engine -- same records."""
    cfg = kind_cfg("convex", out_msa=r == 2)
    groups, weights = kind_groups("convex")
    b, _ = run(cfg, groups, weights=weights, no_chain=True)
    monkeypatch.setenv("ABPOA_GPU_CHAIN_K", "2")
    a, sa = run(cfg, groups, weights=weights)
    assert sa["chain_fallback_groups"] > 0 and sa["chain_groups"] + sa["chain_fallback_groups"] == len(groups), sa
    assert_same_records(a, b, groups)


@pytest.mark.parametrize("kind", ["affine", "strand"])
def test_graph_export(monkeypatch, kind):
    """ABPOA_GPU_CHAIN_EXPORT_GRAPH=1: the host rebuilds the weighted graph and computes the consensus on it."""
    cfg = kind_cfg(kind)
    groups, weights = kind_groups(kind)
    b, _ = run(cfg, groups, weights=weights, no_chain=True)
    monkeypatch.setenv("ABPOA_GPU_CHAIN_EXPORT_GRAPH", "1")
    a, sa = run(cfg, groups, weights=weights)
    assert sa["chain_groups"] == len(groups) and sa["chain_fallback_groups"] == 0, sa
    assert_same_records(a, b, groups)


# ---- the CLI ----
@pytest.mark.parametrize("opts", CLI_LIST_OPTS, ids=lambda o: "".join(o))
def test_cli_list_mode_fastq(reference, tmp_path, monkeypatch, opts):
    """abpoa -l on FASTQ files with qualities (and heter.fq): byte for byte the reference CLI's, on both engines."""
    files = fastq_files(tmp_path)
    lst = tmp_path / "list.txt"
    lst.write_text("".join(f"{p}\n" for p in files))
    want = reference_cli_md5(reference, [*opts, "-l"], files)
    p = subprocess.run([str(BIN), *opts, "-l", str(lst)], capture_output=True, timeout=600)
    assert p.returncode == 0, p.stderr[-2000:]
    assert md5(p.stdout) == want
    monkeypatch.setenv("ABPOA_GPU_NO_CHAIN", "1")
    assert md5(subprocess.run([str(BIN), *opts, "-l", str(lst)], capture_output=True, timeout=600).stdout) == want


# ---- the headline shape ----
def test_headline_shape():
    """4 groups of the headline shape (50 x 10 kbp, convex) with quality-like weights: all on the chain, records equal to
    the launch engine's."""
    wl = synth.WORKLOADS["convex_10k"]
    groups = wl.groups(4)
    weights = [quality_weights(9800 + gi, g) for gi, g in enumerate(groups)]
    cfg = qv_cfg(wl.cfg)
    a, sa = run(cfg, groups, weights=weights)
    assert sa["chain_groups"] == 4 and sa["chain_fallback_groups"] == 0, sa
    b, _ = run(cfg, groups, weights=weights, no_chain=True)
    assert_same_records(a, b, groups)
