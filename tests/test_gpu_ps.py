"""GPU: path scores (-G) on the device-resident chain engine.

The fuse kernel's flatten writes every in-edge's score max(round(ln(edge_w / node_w)), -20) into the next job
(chain_path_score, poa_chain.cuh) and the chain's DP kernels run their path-score instantiation, which adds predecessor
k's score to its diagonal term and its E planes on the straight-line rows, the general rows and the backtrace's F-plane
recompute.  -G batches, alone and with -Q, -s and -a 1, must stay on the chain and give the unmodified reference's
per-read scores, CIGARs, consensus, coverage and MSA rows (tests/golden/reference_runs_ps.json, see
tests/ps_reference.py), and the launch engine's records and text field by field.  Groups handed back, and groups whose
node weights could pass POA_PS_MAX_NODE_W, are finished by the launch engine with the same results."""
import ctypes as C
import math
import subprocess
from pathlib import Path

import numpy as np
import pytest

from abpoa_b200 import synth
from abpoa_b200.capi import c_int_p, product
from gfa_reference import md5, reference_cli_md5
from ps_reference import (CLI_LIST_OPTS, KINDS, batch_weights, group_weights, headline_groups, kind_cfg, kind_groups, ps_cfg,
                          ps_reference)
from qv_reference import CLI_LIST_OPTS as QV_CLI_LIST_OPTS, TEXT_R, fastq_files, quality_weights, qv_reference, reference_group, result_digest
from reference_runs import assert_batch_matches
from test_gpu_chain_msa import assert_same_records, run
from test_gpu_qv import write_text

pytestmark = pytest.mark.gpu

BIN = Path(__file__).resolve().parent.parent / "abpoa_b200" / "bin" / "abpoa"
MAX_NODE_W = 1 << 20            # POA_PS_MAX_NODE_W in poa_chain.cuh


@pytest.fixture(scope="module")
def reference():
    ref = ps_reference()
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


# ---- batches against the reference ----
@pytest.mark.parametrize("kind", KINDS)
def test_batch_matches_reference(reference, kind):
    cfg = kind_cfg(kind)
    groups, weights = kind_groups(kind)
    got, st = run(cfg, groups, weights=weights)
    assert st["chain_groups"] == len(groups) and st["chain_fallback_groups"] == 0, st
    for gi, (g, w, r) in enumerate(zip(groups, group_weights(groups, weights), got)):
        assert result_digest(r) == reference_group(reference, cfg, g, w)["digest"], f"{kind} group {gi}: consensus, coverage or MSA rows"
    if not kind.startswith("strand"):       # per-read scores, CIGAR lengths and hashes, DP cells
        assert_batch_matches(got, groups, reference.batch(cfg, groups, want_msa=True, weights=batch_weights(groups, weights)), tag=kind)


def test_headline_shape(reference):
    """4 groups of the headline shape (50 x 10 kbp, convex) with -G: all on the chain, per-read scores, CIGARs, DP cells and
    consensus equal to the reference's."""
    cfg, groups = headline_groups()
    got, st = run(cfg, groups)
    assert st["chain_groups"] == 4 and st["chain_fallback_groups"] == 0, st
    assert_batch_matches(got, groups, reference.batch(cfg, groups, want_msa=False), tag="headline", msa=False)


# ---- the chain against the launch engine ----
@pytest.mark.parametrize("r", TEXT_R)
@pytest.mark.parametrize("kind", ["convex", "qv", "strand", "mf"])
def test_batch_equals_launch_engine(kind, r):
    """-G, -Q -G, -s -G and -a 1 -G: records and the text abpoa_gpu_msa_batch_write prints, -r 0 / -r 2 / -r 4."""
    cfg = kind_cfg(kind, out_msa=False)
    groups, weights = kind_groups(kind)
    text, a, sa = write_text(cfg, groups, weights, r)
    want, b, sb = write_text(cfg, groups, weights, r, no_chain=True)
    assert sa["chain_groups"] == len(groups) and sa["chain_fallback_groups"] == 0 and sb["chain_groups"] == 0, (sa, sb)
    assert text == want, f"{kind} -r {r}: text differs from the launch engine's"
    assert_same_records(a, b, groups)


@pytest.mark.parametrize("r", [0, 2])
def test_groups_handed_back(monkeypatch, r):
    """Two edge slots per node: most groups leave the chain and are finished by the launch engine -- same records."""
    cfg = kind_cfg("qv", out_msa=r == 2)
    groups, weights = kind_groups("qv")
    b, _ = run(cfg, groups, weights=weights, no_chain=True)
    monkeypatch.setenv("ABPOA_GPU_CHAIN_K", "2")
    a, sa = run(cfg, groups, weights=weights)
    assert sa["chain_fallback_groups"] > 0 and sa["chain_groups"] + sa["chain_fallback_groups"] == len(groups), sa
    assert_same_records(a, b, groups)


def test_node_weight_bound_takes_the_launch_engine():
    """-Q -G: a group of 4113 reads could weigh 255 x 4113 > POA_PS_MAX_NODE_W at a node, so the launch engine finishes it;
    the other groups stay on the chain.  Every record equals an all-launch-engine run's."""
    assert 255 * 4112 <= MAX_NODE_W < 255 * 4113
    groups = [synth.make_group(9960, 6, 300, 0.05), synth.make_group(9961, 4113, 24, 0.05), synth.make_group(9962, 5, 280, 0.06)]
    weights = [quality_weights(9965 + gi, g) for gi, g in enumerate(groups)]
    cfg = ps_cfg(use_qv=True)
    a, sa = run(cfg, groups, weights=weights)
    b, sb = run(cfg, groups, weights=weights, no_chain=True)
    assert sa["chain_groups"] == 2 and sa["chain_fallback_groups"] == 0 and sb["chain_groups"] == 0, (sa, sb)
    assert_same_records(a, b, groups)


def test_graph_export(monkeypatch):
    """ABPOA_GPU_CHAIN_EXPORT_GRAPH=1: the host rebuilds the -G -Q graph and computes the consensus on it."""
    cfg = kind_cfg("qv")
    groups, weights = kind_groups("qv")
    b, _ = run(cfg, groups, weights=weights, no_chain=True)
    monkeypatch.setenv("ABPOA_GPU_CHAIN_EXPORT_GRAPH", "1")
    a, sa = run(cfg, groups, weights=weights)
    assert sa["chain_groups"] == len(groups) and sa["chain_fallback_groups"] == 0, sa
    assert_same_records(a, b, groups)


# ---- the CLI ----
@pytest.mark.parametrize("opts", [o for o in QV_CLI_LIST_OPTS if "-G" in o] + CLI_LIST_OPTS, ids=lambda o: "".join(o))
def test_cli_list_mode_fastq(reference, tmp_path, monkeypatch, opts):
    """abpoa -l with -G on FASTQ files (and heter.fq): byte for byte the reference CLI's, on both engines."""
    files = fastq_files(tmp_path)
    lst = tmp_path / "list.txt"
    lst.write_text("".join(f"{p}\n" for p in files))
    want = reference_cli_md5(reference if opts in CLI_LIST_OPTS else qv_reference(), [*opts, "-l"], files)
    p = subprocess.run([str(BIN), *opts, "-l", str(lst)], capture_output=True, timeout=600)
    assert p.returncode == 0, p.stderr[-2000:]
    assert md5(p.stdout) == want
    monkeypatch.setenv("ABPOA_GPU_NO_CHAIN", "1")
    assert md5(subprocess.run([str(BIN), *opts, "-l", str(lst)], capture_output=True, timeout=600).stdout) == want


# ---- the score function on the device ----
def host_score(ew: int, nw: int) -> int:
    """The reference's expression with glibc's log, rounded half away from zero as C's round."""
    if ew == 0 or nw == 0:
        return 0
    x = math.log(ew / nw)
    return max(int(math.copysign(math.floor(abs(x) + 0.5), x)), -20)


def test_device_score_function():
    """chain_path_score on the GPU against the host's expression: every pair edge_w <= node_w <= 600, and for node weights
    up to POA_PS_MAX_NODE_W the edge weights around every rounding boundary n e^-(k + 1/2)."""
    ew, nw = [], []
    for n in range(601):
        ew.extend(range(n + 1)); nw.extend([n] * (n + 1))
    for n in list(range(601, MAX_NODE_W + 1, 997)) + [MAX_NODE_W]:
        for k in range(20):
            t = math.floor(n * math.exp(-(k + 0.5)))
            for e in (t - 1, t, t + 1, t + 2):
                if 0 <= e <= n:
                    ew.append(e); nw.append(n)
    ew = np.ascontiguousarray(ew, dtype=np.int32)
    nw = np.ascontiguousarray(nw, dtype=np.int32)
    out = np.zeros(len(ew), dtype=np.int32)
    d = product().dll
    d.poa_debug_path_scores.restype = C.c_int
    d.poa_debug_path_scores.argtypes = [c_int_p, c_int_p, C.c_int, c_int_p]
    assert d.poa_debug_path_scores(ew.ctypes.data_as(c_int_p), nw.ctypes.data_as(c_int_p), len(ew), out.ctypes.data_as(c_int_p)) == len(ew)
    want = np.array([host_score(int(e), int(n)) for e, n in zip(ew, nw)], dtype=np.int32)
    bad = np.flatnonzero(out != want)
    assert bad.size == 0, f"{bad.size} pairs differ, first ({ew[bad[0]]}, {nw[bad[0]]}): device {out[bad[0]]}, host {want[bad[0]]}"
