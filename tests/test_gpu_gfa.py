"""GPU: GFA output (-r 3 / -r 4) for single groups and batches.

A single group (abpoa_msa, the single-file CLI) is written by the host writer; batches on the device-resident chain
engine (poa_chain.cu: poa_chain_gfa_kernel) bring back one record per group, which the same formatter prints.  The text
must equal the unmodified reference's (md5s in tests/golden/reference_runs_gfa.json, see tests/gfa_reference.py) and
the launch engine's; the result records must equal the launch engine's field by field."""
import subprocess
from pathlib import Path

import numpy as np
import pytest

from abpoa_b200 import synth
from abpoa_b200.aligner import PoaConfig
from abpoa_b200.batch import BatchEngine, PackedGroups
from abpoa_b200.capi import product
from gfa_reference import (BATCH_INPUTS, CLI_LIST_OPTS, CLI_SINGLE, aa_file, gfa_para, gfa_reference, list_files, md5, mixed_groups,
                           reference_batch_md5, reference_cli_md5, with_file)
from helpers import INPUTS

pytestmark = pytest.mark.gpu

BIN = Path(__file__).resolve().parent.parent / "abpoa_b200" / "bin" / "abpoa"


@pytest.fixture(scope="module")
def reference():
    ref = gfa_reference()
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


def cli_md5(args):
    return md5(subprocess.run([str(BIN), *args], capture_output=True, check=True).stdout)


def write_batch(cfg, groups, out_cons, no_chain=False, writer=True):
    """abpoa_gpu_msa_batch_write (or, writer=False, abpoa_gpu_msa_batch) with -r 3 / -r 4: (text, results, stats)."""
    lib = product()
    abpt = gfa_para(lib, cfg, out_cons)
    packed = PackedGroups(groups)
    try:
        with BatchEngine() as eng:
            if writer:
                got = []
                text = with_file(lambda fp: got.extend(eng.run_write(abpt, packed, fp, record_reads=True, no_chain=no_chain)))
            else:
                text, got = b"", eng.run_packed(abpt, packed, record_reads=True, no_chain=no_chain)
            st = eng.stats()
    finally:
        lib.abpoa_free_para(abpt)
    return text, got, st


def assert_same_records(a, b, groups):
    """Chain vs launch engine, field by field."""
    for gi, (x, y, g) in enumerate(zip(a, b, groups)):
        tag = f"group {gi}"
        assert len(x.msa) == len(y.msa) == 0, f"{tag}: MSA rows with GFA output"
        assert len(x.cons) == len(y.cons) and all(np.array_equal(p, q) for p, q in zip(x.cons, y.cons)), f"{tag}: consensus"
        assert all(np.array_equal(p, q) for p, q in zip(x.cov, y.cov)), f"{tag}: coverage"
        assert x.dp_cells == y.dp_cells and x.n_aligned == y.n_aligned, f"{tag}: DP cells / aligned reads"
        if len(g) > 1:
            assert np.array_equal(x.read_best_score[1:], y.read_best_score[1:]), f"{tag}: per-read scores"
            assert np.array_equal(x.read_n_cigar[1:], y.read_n_cigar[1:]), f"{tag}: per-read CIGAR lengths"
            assert np.array_equal(x.read_cigar_hash[1:], y.read_cigar_hash[1:]), f"{tag}: per-read CIGAR hashes"


def n_chainable(groups):
    return sum(1 for g in groups if len(g) >= 2)


def first_diff(a: bytes, b: bytes) -> int:
    return next((k for k, (x, y) in enumerate(zip(a, b)) if x != y), min(len(a), len(b)))


# ---- CLI ----
@pytest.mark.parametrize("args,fname", CLI_SINGLE, ids=[" ".join(a) + " " + f for a, f in CLI_SINGLE])
def test_cli_single_file_gfa(reference, args, fname):
    assert cli_md5([*args, str(INPUTS / fname)]) == reference_cli_md5(reference, args, [INPUTS / fname])


@pytest.mark.parametrize("r", ["-r3", "-r4"])
def test_cli_amino_acid_gfa(reference, tmp_path, r):
    aa = aa_file(tmp_path)
    assert cli_md5(["-c", r, str(aa)]) == reference_cli_md5(reference, ["-c", r], [aa])


@pytest.mark.parametrize("opts", CLI_LIST_OPTS, ids=[" ".join(o) for o in CLI_LIST_OPTS])
def test_cli_list_mode_gfa(reference, tmp_path, monkeypatch, opts):
    """-l: every file is one group of one GPU batch, each file's GFA with its own H line; the same bytes on the launch engine."""
    files = list_files(tmp_path)
    lst = tmp_path / "list.txt"
    lst.write_text("".join(f"{p}\n" for p in files))
    want = reference_cli_md5(reference, [*opts, "-l"], files)
    assert cli_md5([*opts, "-l", str(lst)]) == want
    monkeypatch.setenv("ABPOA_GPU_NO_CHAIN", "1")
    assert cli_md5([*opts, "-l", str(lst)]) == want


# ---- abpoa_gpu_msa_batch_write ----
@pytest.mark.parametrize("name", list(BATCH_INPUTS))
def test_batch_write_gfa(reference, name):
    cfg, groups = BATCH_INPUTS[name]()
    out_cons = name.endswith("r4")
    text, got, st = write_batch(cfg, groups, out_cons)
    assert st["chain_groups"] == n_chainable(groups) and st["chain_fallback_groups"] == 0, st
    assert md5(text) == reference_batch_md5(reference, cfg, groups, out_cons), f"{name}: GFA differs from the reference's"
    want, launch, sl = write_batch(cfg, groups, out_cons, no_chain=True)
    assert sl["chain_groups"] == 0
    assert text == want, f"{name}: chain and launch engine differ at byte {first_diff(text, want)}"
    assert_same_records(got, launch, groups)
    for r, g in zip(got, groups):
        assert len(r.cons) == (1 if out_cons and len(g) > 0 else 0), "the writer computes the consensus with -r 4 only"


def test_batch_write_gfa_groups_handed_back(monkeypatch):
    """Two edge slots per node: most groups leave the chain and are finished by the launch engine -- same text."""
    groups = [synth.make_group(8400 + g, 8, 400, 0.10) for g in range(10)]
    want, launch, _ = write_batch(PoaConfig(), groups, True, no_chain=True)
    monkeypatch.setenv("ABPOA_GPU_CHAIN_K", "2")
    text, got, st = write_batch(PoaConfig(), groups, True)
    assert st["chain_fallback_groups"] > 0 and st["chain_groups"] + st["chain_fallback_groups"] == 10, st
    assert text == want, f"differs at byte {first_diff(text, want)}"
    assert_same_records(got, launch, groups)


@pytest.mark.parametrize("out_cons", [False, True])
def test_batch_write_gfa_with_graph_export(monkeypatch, out_cons):
    """ABPOA_GPU_CHAIN_EXPORT_GRAPH=1: the host rebuilds the graph; the GFA is still the device record's."""
    groups = [synth.make_group(8500 + g, 9, 450, 0.08) for g in range(6)]
    want, launch, _ = write_batch(PoaConfig(), groups, out_cons, no_chain=True)
    monkeypatch.setenv("ABPOA_GPU_CHAIN_EXPORT_GRAPH", "1")
    text, got, st = write_batch(PoaConfig(), groups, out_cons)
    assert st["chain_groups"] == 6 and st["chain_fallback_groups"] == 0, st
    assert text == want, f"differs at byte {first_diff(text, want)}"
    assert_same_records(got, launch, groups)


@pytest.mark.parametrize("out_cons", [False, True])
def test_batch_without_writer_computes_nothing(out_cons):
    """abpoa_gpu_msa_batch with out_gfa and no writer: as abpoa_msa(..., NULL), nothing is printed or computed -- no
    consensus even with -r 4 -- and both engines return the same records."""
    groups = mixed_groups()
    _, got, st = write_batch(PoaConfig(), groups, out_cons, writer=False)
    _, launch, _ = write_batch(PoaConfig(), groups, out_cons, no_chain=True, writer=False)
    assert st["chain_groups"] == n_chainable(groups) and st["chain_fallback_groups"] == 0, st
    assert_same_records(got, launch, groups)
    assert all(len(r.cons) == 0 for r in got)


def test_batch_write_gfa_headline_shape():
    """4 groups of the headline shape (50 x 10 kbp, convex) with -r 4: all on the chain, text equal to the launch engine's."""
    wl = synth.WORKLOADS["convex_10k"]
    groups = wl.groups(4)
    text, got, st = write_batch(wl.cfg, groups, True)
    assert st["chain_groups"] == 4 and st["chain_fallback_groups"] == 0, st
    want, launch, _ = write_batch(wl.cfg, groups, True, no_chain=True)
    assert text == want, f"differs at byte {first_diff(text, want)}"
    assert_same_records(got, launch, groups)
    assert text.count(b"\nP\t") == 4 * 51, "50 read paths and the consensus path per group"
