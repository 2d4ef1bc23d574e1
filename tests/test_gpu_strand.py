"""GPU: ambiguous-strand alignment (-s) on the device-resident chain engine.

The alignment warp re-aligns a weak forward hit as the reverse complement and keeps the better strand
(poa_kernels.cu: chain_align_read); the fuse reads the winning bases through the slot's strand bytes, which come back
and set the reads' strands for the writers.  Batches of groups in which every third read arrives reverse-complemented
must stay on the chain and give the unmodified reference's strands, consensus, coverage and MSA rows
(tests/golden/reference_runs_strand.json, see tests/strand_reference.py), and the launch engine's records field by
field, DP cells of both strands included."""
import subprocess
from pathlib import Path

import pytest

from abpoa_b200 import synth
from gfa_reference import md5, reference_cli_md5
from strand_reference import (BATCH_KINDS, CLI_LIST_R, kind_cfg, kind_groups, list_files, reference_group, result_digest, revcomp,
                              strand_cfg, strand_reference)
from test_gpu_chain_msa import assert_same_records, run
from test_gpu_gfa import assert_same_records as assert_same_gfa_records
from test_gpu_gfa import first_diff, write_batch

pytestmark = pytest.mark.gpu

BIN = Path(__file__).resolve().parent.parent / "abpoa_b200" / "bin" / "abpoa"


@pytest.fixture(scope="module")
def reference():
    ref = strand_reference()
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


def n_second_dps(results, groups):
    """Reverse-complement alignments the engine ran: n_aligned counts both DPs of a retried read."""
    return sum(r.n_aligned - (len(g) - 1) for r, g in zip(results, groups))


# ---- batches against the reference ----
@pytest.mark.parametrize("kind", BATCH_KINDS)
def test_batch_matches_reference(reference, kind):
    cfg, groups = kind_cfg(kind), kind_groups(kind)
    got, st = run(cfg, groups)
    assert st["chain_groups"] == len(groups) and st["chain_fallback_groups"] == 0, st
    for gi, (g, r) in enumerate(zip(groups, got)):
        assert result_digest(r) == reference_group(reference, cfg, g)["digest"], f"{kind} group {gi}: consensus, coverage or MSA rows"
    assert n_second_dps(got, groups) > 0, "no read was re-aligned as its reverse complement"


# ---- the chain against the launch engine ----
@pytest.mark.parametrize("r", [0, 2])
@pytest.mark.parametrize("kind", BATCH_KINDS)
def test_batch_equals_launch_engine(kind, r):
    cfg, groups = kind_cfg(kind, out_msa=r == 2), kind_groups(kind)
    a, sa = run(cfg, groups)
    b, sb = run(cfg, groups, no_chain=True)
    assert sa["chain_groups"] == len(groups) and sa["chain_fallback_groups"] == 0 and sb["chain_groups"] == 0, (sa, sb)
    assert_same_records(a, b, groups)


@pytest.mark.parametrize("kind", ["convex", "mf"])
def test_batch_write_gfa_equals_launch_engine(kind):
    """-r 4 through abpoa_gpu_msa_batch_write: the same text (P lines of flipped reads reversed, with '-') and records."""
    cfg, groups = kind_cfg(kind, out_msa=False), kind_groups(kind)
    text, got, st = write_batch(cfg, groups, True)
    assert st["chain_groups"] == len(groups) and st["chain_fallback_groups"] == 0, st
    want, launch, _ = write_batch(cfg, groups, True, no_chain=True)
    assert b"-" in text and text == want, f"{kind}: chain and launch engine differ at byte {first_diff(text, want)}"
    assert_same_gfa_records(got, launch, groups)


@pytest.mark.parametrize("r", [0, 2])
def test_groups_handed_back(monkeypatch, r):
    """Two edge slots per node: most groups leave the chain and are finished by the launch engine -- same records."""
    cfg, groups = kind_cfg("convex", out_msa=r == 2), kind_groups("convex")
    b, _ = run(cfg, groups, no_chain=True)
    monkeypatch.setenv("ABPOA_GPU_CHAIN_K", "2")
    a, sa = run(cfg, groups)
    assert sa["chain_fallback_groups"] > 0 and sa["chain_groups"] + sa["chain_fallback_groups"] == len(groups), sa
    assert_same_records(a, b, groups)


@pytest.mark.parametrize("r", [0, 2])
def test_graph_export(monkeypatch, r):
    """ABPOA_GPU_CHAIN_EXPORT_GRAPH=1: the host rebuilds the graph and computes the consensus on it, the strands still
    come from the device."""
    cfg, groups = kind_cfg("affine", out_msa=r == 2), kind_groups("affine")
    b, _ = run(cfg, groups, no_chain=True)
    monkeypatch.setenv("ABPOA_GPU_CHAIN_EXPORT_GRAPH", "1")
    a, sa = run(cfg, groups)
    assert sa["chain_groups"] == len(groups) and sa["chain_fallback_groups"] == 0, sa
    assert_same_records(a, b, groups)


def test_graph_export_gfa(monkeypatch):
    cfg, groups = kind_cfg("convex", out_msa=False), kind_groups("convex")
    want, _, _ = write_batch(cfg, groups, True, no_chain=True)
    monkeypatch.setenv("ABPOA_GPU_CHAIN_EXPORT_GRAPH", "1")
    text, _, st = write_batch(cfg, groups, True)
    assert st["chain_groups"] == len(groups) and st["chain_fallback_groups"] == 0, st
    assert text == want, f"differs from the launch engine at byte {first_diff(text, want)}"


# ---- the CLI ----
@pytest.mark.parametrize("r", CLI_LIST_R)
def test_cli_list_mode(reference, tmp_path, monkeypatch, r):
    """abpoa -l -s on named FASTA files with flipped reads: _reverse_complement names and '-' P lines, byte for byte the
    reference CLI's; the same bytes on the launch engine."""
    files = list_files(tmp_path)
    lst = tmp_path / "list.txt"
    lst.write_text("".join(f"{p}\n" for p in files))
    want = reference_cli_md5(reference, ["-s", "-r", r, "-l"], files)
    p = subprocess.run([str(BIN), "-s", "-r", r, "-l", str(lst)], capture_output=True, timeout=600)
    assert p.returncode == 0, p.stderr[-2000:]
    assert md5(p.stdout) == want
    if r in ("1", "2"):
        assert b"_reverse_complement" in p.stdout
    monkeypatch.setenv("ABPOA_GPU_NO_CHAIN", "1")
    assert md5(subprocess.run([str(BIN), "-s", "-r", r, "-l", str(lst)], capture_output=True, timeout=600).stdout) == want


# ---- the headline shape ----
def test_headline_shape():
    """4 groups of the headline shape (50 x 10 kbp, convex) with every third read reverse-complemented: all on the chain,
    records equal to the launch engine's."""
    wl = synth.WORKLOADS["convex_10k"]
    groups = [[revcomp(x) if i % 3 == 1 else x for i, x in enumerate(g)] for g in wl.groups(4)]
    cfg = strand_cfg(wl.cfg)
    a, sa = run(cfg, groups)
    assert sa["chain_groups"] == 4 and sa["chain_fallback_groups"] == 0, sa
    b, _ = run(cfg, groups, no_chain=True)
    assert_same_records(a, b, groups)
    assert n_second_dps(a, groups) >= 4 * 16
