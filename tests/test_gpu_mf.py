"""GPU: the most-frequent-base consensus (-a 1) for single groups and batches.

Single groups (abpoa_msa, the single-file CLI, msa_aligner) run the host's most_frequent (poa_cons.c); batches run on the
device-resident chain engine (poa_chain.cu: poa_chain_consensus_kernel with chain_mf_consensus), whose record, -r 2 rows
and -r 4 GFA text must equal the unmodified reference's (tests/golden/reference_runs_mf.json, see tests/mf_reference.py)
and, field by field, the launch engine's."""
import subprocess
from pathlib import Path

import pytest

from abpoa_b200 import synth
from abpoa_b200.capi import product
from gfa_reference import aa_file, list_files, md5, reference_cli_md5
from helpers import INPUTS, read_fasta
from mf_reference import (BATCH_INPUTS, CLI_LIST_OPTS, CLI_SINGLE, GFA_INPUTS, group_text, kind_cfg, kind_groups, mf_cfg, mf_reference,
                          pyabpoa_digest, reference_batch_md5, reference_group_md5, reference_pyabpoa, reference_subgraph_walk,
                          subgraph_inputs, subgraph_walk_mf)
from reference_runs import assert_batch_matches
from test_gpu_chain_msa import assert_same_records, n_chainable, run
from test_gpu_gfa import first_diff, write_batch
from test_gpu_gfa import assert_same_records as assert_same_gfa_records

pytestmark = pytest.mark.gpu

BIN = Path(__file__).resolve().parent.parent / "abpoa_b200" / "bin" / "abpoa"


@pytest.fixture(scope="module")
def reference():
    ref = mf_reference()
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


def cli(args):
    return subprocess.run([str(BIN), *args], capture_output=True, timeout=600)


# ---- batches (abpoa_gpu_msa_batch) ----
@pytest.mark.parametrize("name", list(BATCH_INPUTS))
def test_batch_mf_matches_reference(reference, name):
    cfg, groups = BATCH_INPUTS[name]()
    got, st = run(cfg, groups)
    assert st["chain_groups"] == n_chainable(groups) and st["chain_fallback_groups"] == 0, st
    assert_batch_matches(got, groups, reference.batch(cfg, groups, want_msa=cfg.out_msa), tag=name)


@pytest.mark.parametrize("r", [0, 2])
@pytest.mark.parametrize("kind", ["convex", "affine", "aa"])
def test_batch_mf_equals_launch_engine(kind, r):
    cfg, groups = kind_cfg(kind, r), kind_groups(kind)
    a, sa = run(cfg, groups)
    b, sb = run(cfg, groups, no_chain=True)
    assert sa["chain_groups"] == len(groups) and sb["chain_groups"] == 0
    assert_same_records(a, b, groups)


@pytest.mark.parametrize("r", [0, 2])
def test_batch_mf_groups_handed_back(monkeypatch, r):
    """Two edge slots per node: most groups leave the chain and are finished by the launch engine -- same records."""
    groups = [synth.make_group(9500 + g, 8, 400, 0.10) for g in range(10)]
    cfg = mf_cfg(out_msa=r == 2)
    b, _ = run(cfg, groups, no_chain=True)
    monkeypatch.setenv("ABPOA_GPU_CHAIN_K", "2")
    a, sa = run(cfg, groups)
    assert sa["chain_fallback_groups"] > 0 and sa["chain_groups"] + sa["chain_fallback_groups"] == 10, sa
    assert_same_records(a, b, groups)


@pytest.mark.parametrize("r", [0, 2])
def test_batch_mf_with_graph_export(monkeypatch, r):
    """ABPOA_GPU_CHAIN_EXPORT_GRAPH=1: the host rebuilds the graph and computes the consensus on it; -r 2 rows (and their
    consensus row) are still the device's.  Both must equal the launch engine's."""
    groups = [synth.make_group(9600 + g, 9, 450, 0.08) for g in range(6)]
    cfg = mf_cfg(out_msa=r == 2)
    b, _ = run(cfg, groups, no_chain=True)
    monkeypatch.setenv("ABPOA_GPU_CHAIN_EXPORT_GRAPH", "1")
    a, sa = run(cfg, groups)
    assert sa["chain_groups"] == 6 and sa["chain_fallback_groups"] == 0, sa
    assert_same_records(a, b, groups)


def test_batch_mf_headline_shape():
    """4 groups of the headline shape (50 x 10 kbp, convex) with -a 1, consensus and -r 2: all on the chain, records equal
    to the launch engine's."""
    wl = synth.WORKLOADS["convex_10k"]
    groups = wl.groups(4)
    for out_msa in (False, True):
        cfg = mf_cfg(wl.cfg, out_msa=out_msa)
        a, sa = run(cfg, groups)
        assert sa["chain_groups"] == 4 and sa["chain_fallback_groups"] == 0, sa
        b, _ = run(cfg, groups, no_chain=True)
        assert_same_records(a, b, groups)
        assert all(len(r.cons) == 1 and len(r.cons[0]) > 9000 for r in a)


# ---- abpoa_gpu_msa_batch_write with -r 4 ----
@pytest.mark.parametrize("name", list(GFA_INPUTS))
def test_batch_write_mf_gfa(reference, name):
    cfg, groups = GFA_INPUTS[name]()
    text, got, st = write_batch(cfg, groups, True)
    assert st["chain_groups"] == n_chainable(groups) and st["chain_fallback_groups"] == 0, st
    assert md5(text) == reference_batch_md5(reference, cfg, groups, 4), f"{name}: GFA differs from the reference's"
    want, launch, _ = write_batch(cfg, groups, True, no_chain=True)
    assert text == want, f"{name}: chain and launch engine differ at byte {first_diff(text, want)}"
    assert_same_gfa_records(got, launch, groups)


# ---- single groups ----
@pytest.mark.parametrize("r", [2, 4, 5])
def test_single_group_abpoa_msa(reference, r):
    """abpoa_msa on 3alleles.fa (the CPU suite recorded the reference's output for the same group)."""
    reads = read_fasta(INPUTS / "3alleles.fa")
    cfg = mf_cfg(out_msa=True)
    assert md5(group_text(product(), cfg, reads, r)) == reference_group_md5(reference, cfg, reads, r)


def test_subgraph_walk_with_sub_aln(reference):
    """The loop of the reference's sub_example.c: -a 1 with sub_aln = 1, gaps counted against n_span_read."""
    reads, windows = subgraph_inputs()
    assert subgraph_walk_mf(product(), reads, windows) == reference_subgraph_walk(reference)


def test_msa_aligner_mf(reference):
    """msa_aligner(cons_algrm="MF") gives every field the reference library gives."""
    got = pyabpoa_digest(product())
    want = reference_pyabpoa(reference)
    for g, w in zip(got, want):
        assert g == w


# ---- the CLI ----
@pytest.mark.parametrize("args,fname", CLI_SINGLE, ids=[" ".join(a) + " " + f for a, f in CLI_SINGLE])
def test_cli_single_file_mf(reference, args, fname):
    p = cli([*args, str(INPUTS / fname)])
    assert p.returncode == 0, p.stderr[-2000:]
    assert md5(p.stdout) == reference_cli_md5(reference, args, [INPUTS / fname])


@pytest.mark.parametrize("r", ["0", "2"])
def test_cli_amino_acid_mf(reference, tmp_path, r):
    aa = aa_file(tmp_path)
    assert md5(cli(["-a", "1", "-c", "-r", r, str(aa)]).stdout) == reference_cli_md5(reference, ["-a", "1", "-c", "-r", r], [aa])


@pytest.mark.parametrize("opts", CLI_LIST_OPTS, ids=[" ".join(o) for o in CLI_LIST_OPTS])
def test_cli_list_mode_mf(reference, tmp_path, monkeypatch, opts):
    """-l: every file is one group of one GPU batch; the same bytes on the launch engine."""
    files = list_files(tmp_path)
    lst = tmp_path / "list.txt"
    lst.write_text("".join(f"{p}\n" for p in files))
    want = reference_cli_md5(reference, [*opts, "-l"], files)
    assert md5(cli([*opts, "-l", str(lst)]).stdout) == want
    monkeypatch.setenv("ABPOA_GPU_NO_CHAIN", "1")
    assert md5(cli([*opts, "-l", str(lst)]).stdout) == want


def test_cli_multi_consensus_still_aborts():
    """-d 2 -a 1 is out of scope: the process ends with the library's message and exit code 1."""
    p = cli(["-d", "2", "-a", "1", str(INPUTS / "seq.fa")])
    assert p.returncode == 1 and b"max_n_cons > 1" in p.stderr, (p.returncode, p.stderr[-2000:])
