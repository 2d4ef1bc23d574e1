"""GPU: banded linear-gap (-O 0) batches on the device-resident chain engine.

The chain's job function runs linear-gap rows the way the reference's vector procedure does (p16_run_job's LGX rows, see
poa_kernels.cu): rows stored in whole pn-lane vectors, leaked cells right of the band, vector-granular predecessor reach and
the incomplete scan.  The launch engine runs the same jobs on the generic kernel's "lgx" rows, which
tests/test_gpu_cases.py::test_linear_banded_lane_exact_sweep / _int32_width hold to the live reference.  Here every linear
batch must stay on the chain (no hand-backs) and give the launch engine's records field by field: consensus, coverage, MSA
rows, DP cells, aligned reads, and each read's score, CIGAR length and CIGAR hash."""
import pytest

import subprocess
from pathlib import Path

from abpoa_b200 import synth
from abpoa_b200.capi import ABPOA_MF
from gfa_reference import list_files, md5, reference_cli_md5
from linear_reference import CLI_LIST_OPTS, KINDS, kind_input, lin_cfg, linear_reference, sweep_groups
from qv_reference import fastq_files, quality_weights
from reference_runs import assert_batch_matches
from test_gpu_chain_msa import assert_same_records, run

pytestmark = pytest.mark.gpu


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


BIN = Path(__file__).resolve().parent.parent / "abpoa_b200" / "bin" / "abpoa"


@pytest.fixture(scope="module")
def reference():
    ref = linear_reference()
    yield ref
    ref.save()


@pytest.mark.parametrize("kind", KINDS)
def test_batch_matches_reference(reference, kind):
    """Every group on the chain; per-read scores, CIGAR lengths and hashes, DP cells, consensus, coverage and MSA rows
    equal the reference's (tests/golden/reference_runs_linear.json)."""
    cfg, groups = kind_input(kind, out_msa=True)
    got, st = run(cfg, groups)
    assert st["chain_groups"] == n_chainable(groups) and st["chain_fallback_groups"] == 0, st
    assert_batch_matches(got, groups, reference.batch(cfg, groups, want_msa=True), tag=kind)


@pytest.mark.parametrize("opts", CLI_LIST_OPTS)
@pytest.mark.parametrize("fmt", ["fasta", "fastq"])
def test_cli_list_mode(reference, tmp_path, monkeypatch, fmt, opts):
    """abpoa -l -O 0 -r 0..4 on FASTA and FASTQ lists: byte for byte the reference CLI's, on both engines."""
    files = list_files(tmp_path) if fmt == "fasta" else fastq_files(tmp_path)
    lst = tmp_path / "list.txt"
    lst.write_text("".join(f"{p}\n" for p in files))
    want = reference_cli_md5(reference, [*opts, "-l"], files)
    p = subprocess.run([str(BIN), *opts, "-l", str(lst)], capture_output=True, timeout=600)
    assert p.returncode == 0, p.stderr[-2000:]
    assert md5(p.stdout) == want
    monkeypatch.setenv("ABPOA_GPU_NO_CHAIN", "1")
    assert md5(subprocess.run([str(BIN), *opts, "-l", str(lst)], capture_output=True, timeout=600).stdout) == want


@pytest.mark.parametrize("kind", KINDS)
def test_batch_equals_launch_engine(kind):
    cfg, groups = kind_input(kind)
    a, sa = run(cfg, groups)
    b, sb = run(cfg, groups, no_chain=True)
    assert sa["chain_groups"] == n_chainable(groups) and sa["chain_fallback_groups"] == 0 and sb["chain_groups"] == 0, (sa, sb)
    assert_same_records(a, b, groups)


@pytest.mark.parametrize("opt", ["msa", "strand", "qv", "path_score", "mf"])
def test_options_equal_launch_engine(opt):
    """-r 2 (MSA rows), -s, -Q, -G and -a 1 with linear gaps: the chain gives the launch engine's records.  -s runs on the
    sweep's forward-strand groups, whose weak hits at 15-25 % error take the retry.  Known limitation: with reads that
    arrive reverse-complemented, the wrong-strand pass of a linear-gap alignment can fail its backtrace; the launch engine
    then stops the process with "Error in dp_backtrack" (as before this engine took linear gaps)."""
    groups, weights = sweep_groups(0, 12), None
    kw = dict(out_msa=True)
    if opt == "strand":
        kw["amb_strand"] = True
    elif opt == "qv":
        weights = [quality_weights(9870 + gi, g) for gi, g in enumerate(groups)]
        kw["use_qv"] = True
    elif opt == "path_score":
        kw["inc_path_score"] = True
    elif opt == "mf":
        kw["cons_algrm"] = ABPOA_MF
    cfg = lin_cfg(**kw)
    a, sa = run(cfg, groups, weights=weights)
    b, sb = run(cfg, groups, weights=weights, no_chain=True)
    assert sa["chain_groups"] == n_chainable(groups) and sa["chain_fallback_groups"] == 0, sa
    assert_same_records(a, b, groups)


def test_groups_handed_back(monkeypatch):
    """Two edge slots per node: most groups leave the chain and the launch engine finishes them -- same records."""
    cfg, groups = lin_cfg(out_msa=True), sweep_groups(0, 16)
    b, _ = run(cfg, groups, no_chain=True)
    monkeypatch.setenv("ABPOA_GPU_CHAIN_K", "2")
    a, sa = run(cfg, groups)
    assert sa["chain_fallback_groups"] > 0 and sa["chain_groups"] + sa["chain_fallback_groups"] == len(groups), sa
    assert_same_records(a, b, groups)


def test_graph_export(monkeypatch):
    """The whole graph comes back and the host computes consensus and MSA on it: the same records."""
    cfg, groups = lin_cfg(out_msa=True), sweep_groups(0, 12)
    b, _ = run(cfg, groups, no_chain=True)
    monkeypatch.setenv("ABPOA_GPU_CHAIN_EXPORT_GRAPH", "1")
    a, sa = run(cfg, groups)
    assert sa["chain_groups"] == len(groups), sa
    assert_same_records(a, b, groups)


def test_headline_shape():
    """Four 50 x 10 kbp groups (the headline shape with -O 0 -E 2): all on the chain, the launch engine's records."""
    cfg = lin_cfg()
    groups = [synth.make_group(9880 + g, 50, 10_000, 0.05) for g in range(4)]
    a, sa = run(cfg, groups)
    b, _ = run(cfg, groups, no_chain=True)
    assert sa["chain_groups"] == len(groups) and sa["chain_fallback_groups"] == 0, sa
    assert_same_records(a, b, groups)
