"""GPU: extend-mode (-m 2, with and without z-drop -z) batches on the device-resident chain engine.

The chain runs extend jobs on its job function's EXTEND instantiation (the same straight-line rows and compact layout as
global jobs, then the first row that holds the maximum and the z-drop stop), with the rows in the reference's Kahn order,
which the fuse builds on the device (chain_kahn_order; tests/test_chain_emul_extend.py pins it against the host layer on
the CPU).  Every extend batch must stay on the chain and give the stored reference's records and the launch engine's
field by field: consensus, coverage, MSA rows, DP cells, aligned reads, and each read's score, CIGAR length and CIGAR hash.

The reference counts a read's DP cells over every row's band record, also over the rows it never computed after a
z-drop stop; with z-drop on its cell counts are not comparable, and only there the comparison with the reference leaves
them out (the launch engine's cells are compared everywhere).  A small z-drop at 15-25 % error stops most alignments early,
and every read's unaligned tail then enters SINK through an edge of its own: those kinds run with 32 edge slots per node
(ABPOA_GPU_CHAIN_K), as a caller with such reads would set, so that no group is handed back."""
import subprocess
from pathlib import Path

import pytest

from abpoa_b200 import synth
from abpoa_b200.capi import ABPOA_MF
from extend_reference import CLI_LIST_OPTS, KINDS, ext_cfg, extend_reference, kind_input, sweep_groups
from gfa_reference import list_files, md5, reference_cli_md5
from qv_reference import fastq_files, quality_weights
from reference_runs import batch_digest
from strand_reference import revcomp
from test_gpu_chain_msa import assert_same_records, run

pytestmark = pytest.mark.gpu

BIN = Path(__file__).resolve().parent.parent / "abpoa_b200" / "bin" / "abpoa"
ZDROP_FIRES = {"zdrop_fires", "affine_zdrop_error_fan"}      # kinds whose SINK gets more in-edges than the default 12 slots


@pytest.fixture(autouse=True, params=["free-running", "rounds"])
def chain_mode(request, monkeypatch):
    """Every test runs on both schedules of the chain engine (see test_gpu_chain.py)."""
    if request.param == "rounds":
        monkeypatch.setenv("ABPOA_GPU_CHAIN_ROUNDS", "1")
    else:
        monkeypatch.delenv("ABPOA_GPU_CHAIN_ROUNDS", raising=False)
    return request.param


def n_chainable(groups):
    return sum(1 for g in groups if len(g) >= 2)


def on_chain(st, groups):
    return st["chain_groups"] == n_chainable(groups) and st["chain_fallback_groups"] == 0


@pytest.fixture(scope="module")
def reference():
    ref = extend_reference()
    yield ref
    ref.save()


def assert_matches_reference(got, groups, want, tag, cells=True):
    assert len(got) == len(want) == len(groups)
    for gi, (r, g, w) in enumerate(zip(got, groups, want)):
        w_cells, unaligned, w_hash = w.split(":")
        if cells:
            assert r.dp_cells == int(w_cells), f"{tag} group {gi}: DP cells {r.dp_cells}, reference {w_cells}"
        assert batch_digest(r, len(g), unaligned).split(":")[2] == w_hash, \
            f"{tag} group {gi}: per-read scores / CIGAR lengths / CIGAR hashes, consensus, coverage or RC-MSA differ from the reference"


@pytest.mark.parametrize("kind", KINDS)
def test_batch_matches_reference_and_launch_engine(reference, kind, monkeypatch):
    """Every group on the chain; the reference's records (tests/golden/reference_runs_extend.json) and the launch
    engine's."""
    if kind in ZDROP_FIRES:
        monkeypatch.setenv("ABPOA_GPU_CHAIN_K", "32")
    cfg, groups = kind_input(kind, out_msa=True)
    a, sa = run(cfg, groups)
    b, sb = run(cfg, groups, no_chain=True)
    assert on_chain(sa, groups) and sb["chain_groups"] == 0, (sa, sb)
    assert_same_records(a, b, groups)
    assert_matches_reference(a, groups, reference.batch(cfg, groups, want_msa=True), kind, cells=cfg.zdrop <= 0)


@pytest.mark.parametrize("zdrop", [-1, 30])
@pytest.mark.parametrize("opt", ["cons", "msa", "mf", "strand", "qv", "path_score", "qv_path_score"])
def test_options_equal_launch_engine(opt, zdrop):
    """-r 0 / -r 2, -a 1, -s, -Q, -G and -Q -G with -m 2, with and without z-drop: the chain gives the launch engine's
    records.  -s runs on groups with every third read reverse-complemented."""
    groups, weights = sweep_groups(0, 12), None
    kw = dict(zdrop=zdrop, out_msa=opt != "cons")
    if opt == "strand":
        kw["amb_strand"] = True
        groups = [[revcomp(r) if i % 3 == 2 else r for i, r in enumerate(g)] for g in groups]
    if opt in ("qv", "qv_path_score"):
        weights = [quality_weights(7870 + gi, g) for gi, g in enumerate(groups)]
        kw["use_qv"] = True
    if opt in ("path_score", "qv_path_score"):
        kw["inc_path_score"] = True
    if opt == "mf":
        kw["cons_algrm"] = ABPOA_MF
    cfg = ext_cfg(**kw)
    a, sa = run(cfg, groups, weights=weights)
    b, sb = run(cfg, groups, weights=weights, no_chain=True)
    assert on_chain(sa, groups), sa
    assert_same_records(a, b, groups)


@pytest.mark.parametrize("opts", CLI_LIST_OPTS)
@pytest.mark.parametrize("fmt", ["fasta", "fastq"])
def test_cli_list_mode(reference, tmp_path, monkeypatch, fmt, opts):
    """abpoa -l -m 2 [-z 100] -r 0..4 on FASTA and FASTQ lists: byte for byte the reference CLI's, on both engines."""
    files = list_files(tmp_path) if fmt == "fasta" else fastq_files(tmp_path)
    lst = tmp_path / "list.txt"
    lst.write_text("".join(f"{p}\n" for p in files))
    want = reference_cli_md5(reference, [*opts, "-l"], files)
    p = subprocess.run([str(BIN), *opts, "-l", str(lst)], capture_output=True, timeout=600)
    assert p.returncode == 0, p.stderr[-2000:]
    assert md5(p.stdout) == want
    monkeypatch.setenv("ABPOA_GPU_NO_CHAIN", "1")
    assert md5(subprocess.run([str(BIN), *opts, "-l", str(lst)], capture_output=True, timeout=600).stdout) == want


@pytest.mark.parametrize("kind", sorted(ZDROP_FIRES))
def test_zdrop_tails_with_default_edge_slots(kind):
    """The same kinds with the default 12 edge slots: the groups whose SINK needs more are handed back and finished by
    the launch engine -- the same records either way."""
    cfg, groups = kind_input(kind, out_msa=True)
    a, sa = run(cfg, groups)
    b, _ = run(cfg, groups, no_chain=True)
    assert sa["chain_groups"] + sa["chain_fallback_groups"] == n_chainable(groups), sa
    assert_same_records(a, b, groups)


def test_groups_handed_back(monkeypatch):
    """Two edge slots per node: most groups leave the chain and the launch engine finishes them -- same records."""
    cfg, groups = ext_cfg(zdrop=50, out_msa=True), sweep_groups(0, 16)
    b, _ = run(cfg, groups, no_chain=True)
    monkeypatch.setenv("ABPOA_GPU_CHAIN_K", "2")
    a, sa = run(cfg, groups)
    assert sa["chain_fallback_groups"] > 0 and sa["chain_groups"] + sa["chain_fallback_groups"] == len(groups), sa
    assert_same_records(a, b, groups)


def test_graph_export(monkeypatch):
    """The whole graph comes back and the host computes consensus and MSA on it: the same records."""
    cfg, groups = ext_cfg(zdrop=50, out_msa=True), sweep_groups(0, 12)
    b, _ = run(cfg, groups, no_chain=True)
    monkeypatch.setenv("ABPOA_GPU_CHAIN_EXPORT_GRAPH", "1")
    a, sa = run(cfg, groups)
    assert sa["chain_groups"] == len(groups), sa
    assert_same_records(a, b, groups)


@pytest.mark.parametrize("zdrop", [-1, 100])
def test_headline_shape(zdrop):
    """Four 50 x 10 kbp groups (the headline shape with -m 2): all on the chain, the launch engine's records."""
    cfg = ext_cfg(zdrop=zdrop)
    groups = [synth.make_group(7880 + g, 50, 10_000, 0.05) for g in range(4)]
    a, sa = run(cfg, groups)
    b, _ = run(cfg, groups, no_chain=True)
    assert on_chain(sa, groups), sa
    assert_same_records(a, b, groups)
