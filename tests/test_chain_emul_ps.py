"""CPU suite: path scores (-G) on the chain engine's graph code.

The device-side graph code (abpoa_b200/csrc/poa_chain.cuh) is compiled for the host and driven read by read next to the
product's host graph layer, with every alignment from the scalar oracle (which runs -G).  After every read the graph
arrays and the next job blob must agree byte for byte with poa_blob_fill's, including the predscore section that
chain_flatten writes with chain_path_score; after the last read the device's consensus must be the host's and its -r 0 /
-r 2 / -r 4 text the reference's (md5s in tests/golden/reference_runs_ps.json, see tests/ps_reference.py).

The device's log may round differently from glibc's in the last bit.  test_no_ratio_near_a_rounding_boundary proves on
the CPU that for every node weight up to POA_PS_MAX_NODE_W (the largest the chain admits) no edge weight puts
ln(edge_w / node_w) within 1024 ulp of a rounding boundary -(k + 1/2), so the two round alike; the GPU suite compares the
device's function with the host's over a sweep."""
import ctypes as C
import math
import subprocess
from pathlib import Path

import numpy as np
import pytest

from abpoa_b200 import capi, synth
from abpoa_b200.aligner import PoaConfig, PoaSession
from abpoa_b200.batch import fnv1a_words
from abpoa_b200.capi import c_int_p, c_u8_p
from cases import AFFINE, CASES, case_reads
from gfa_reference import md5
from mf_reference import set_outputs
from oracle_binding import oracle_align
from ps_reference import ps_cfg, ps_reference
from qv_reference import quality_weights, reference_group, reference_group_md5, unit_filled
from strand_reference import revcomp, strand_mix
from test_chain_emul_gfa import bind_product
from test_chain_emul_qv import consensus_text, set_strands
from test_chain_emul_strand import arr, compare_graphs, device_cigar, device_text, host_weak_hit

HERE = Path(__file__).resolve().parent
ROOT = HERE.parent
SO = HERE / "emul" / "libchain_emul_ps.so"
MAX_NODE_W = 1 << 20            # POA_PS_MAX_NODE_W in poa_chain.cuh


@pytest.fixture(scope="module")
def reference():
    ref = ps_reference()
    yield ref
    ref.save()


@pytest.fixture(scope="module")
def emul():
    """tests/emul/chain_emul_ps.cpp (chain_emul_qv.cpp + the -G exports) compiled for the host."""
    srcs = [HERE / "emul" / "chain_emul_ps.cpp", HERE / "emul" / "chain_emul_qv.cpp", HERE / "emul" / "chain_emul_strand.cpp",
            HERE / "emul" / "chain_emul.cpp", ROOT / "abpoa_b200" / "csrc" / "poa_chain.cuh"]
    if not SO.exists() or SO.stat().st_mtime < max(p.stat().st_mtime for p in srcs):
        subprocess.run(["g++", "-O1", "-g", "-fPIC", "-shared", f"-I{ROOT / 'abpoa_b200' / 'csrc'}", f"-I{ROOT / 'include'}", f"-I{HERE / 'emul'}",
                        "-o", str(SO), str(srcs[0])], check=True)
    d = C.CDLL(str(SO))
    d.chain_emul_ps_new.restype = C.c_void_p
    d.chain_emul_ps_new.argtypes = [C.c_int, c_int_p, C.POINTER(c_u8_p), c_int_p] + [C.c_int] * 11
    d.chain_emul_free.argtypes = [C.c_void_p]
    d.chain_emul_ps_seed.argtypes = [C.c_void_p]
    d.chain_emul_ps_fuse.restype = C.c_int
    d.chain_emul_ps_fuse.argtypes = [C.c_void_p, C.POINTER(C.c_uint64), C.c_int, C.c_int, C.c_int64]
    d.chain_emul_n_nodes.argtypes = [C.c_void_p]
    d.chain_emul_array.restype = c_int_p
    d.chain_emul_array.argtypes = [C.c_void_p, C.c_int]
    d.chain_emul_bases.restype = c_u8_p
    d.chain_emul_bases.argtypes = [C.c_void_p]
    d.chain_emul_blob.restype = c_u8_p
    d.chain_emul_blob.argtypes = [C.c_void_p]
    d.chain_emul_hashes.restype = C.POINTER(C.c_uint64)
    d.chain_emul_hashes.argtypes = [C.c_void_p]
    d.chain_emul_cells.restype = C.c_int64
    d.chain_emul_cells.argtypes = [C.c_void_p]
    d.chain_emul_consensus.restype = C.c_int
    d.chain_emul_consensus.argtypes = [C.c_void_p, c_int_p, C.c_int]
    d.chain_emul_weak_hit.restype = C.c_int
    d.chain_emul_weak_hit.argtypes = [C.c_int] * 4
    d.chain_emul_set_read_rc.argtypes = [C.c_void_p, c_u8_p]
    d.chain_emul_set_read_qw.argtypes = [C.c_void_p, c_u8_p]
    d.chain_emul_msa.restype = C.c_int
    d.chain_emul_msa.argtypes = [C.c_void_p, C.c_int, c_u8_p, C.c_int64]
    d.chain_emul_gfa.restype = C.c_int64
    d.chain_emul_gfa.argtypes = [C.c_void_p, C.c_int, c_int_p, C.c_int64]
    d.chain_emul_path_scores.argtypes = [c_int_p, c_int_p, C.c_int, c_int_p]
    d.chain_emul_ps_layout_check.restype = C.c_int
    d.chain_emul_ps_layout_check.argtypes = [C.c_int] * 9
    return d


def compare_predscore(d, e, blob_buf, i, stats):
    """The predscore section of the device's next job blob against poa_blob_fill's (compare_graphs has just filled
    blob_buf and checked the header, which holds the section's offset)."""
    want = blob_buf
    hdr = want[:68].view(np.int32)
    n_rows, off_rm, off_ps = int(hdr[0]), int(hdr[4]), int(hdr[6])
    assert off_ps > 0, f"read {i}: the host blob has no predscore section"
    n_pred = int(want[off_rm + 8 * n_rows: off_rm + 8 * n_rows + 4].view(np.int32)[0])
    got = np.ctypeslib.as_array(d.chain_emul_blob(e), shape=(off_ps + 4 * n_pred,))[off_ps:]
    w = want[off_ps: off_ps + 4 * n_pred]
    assert np.array_equal(got, w), f"read {i}: job blob for read {i + 1}: section predscore differs at byte {off_ps + int(np.argmax(got != w))}"
    ps = w.view(np.int32)
    stats["nonzero"] += int(np.count_nonzero(ps))
    stats["min"] = min(stats["min"], int(ps.min()) if len(ps) else 0)
    rm = want[off_rm: off_rm + 8 * (n_rows + 1)].view(np.int32)
    stats["max_np"] = max(stats["max_np"], int(np.max(np.diff(rm[0::2]))))


def drive_ps(d, product_lib, reference, cfg: PoaConfig, reads, weights=None, K=12):
    """Fuse `reads` (with their -Q `weights`, per read an int array or None) with the emulated device code and the host
    graph layer side by side, every job flattened with path scores; with cfg.amb_strand each read on the strand the
    alignment warp would pick.  Returns what the predscore sections held (non-zero scores, the smallest score, the most
    predecessors of a row)."""
    pd = bind_product(product_lib)
    weights = [None] * len(reads) if weights is None else weights
    A = cfg.m - 1
    n = len(reads)
    W = (n + 63) // 64
    arrs = [np.ascontiguousarray(x, dtype=np.uint8) for x in reads]
    lens = (C.c_int * n)(*[len(x) for x in arrs])
    ptrs = (c_u8_p * n)(*[x.ctypes.data_as(c_u8_p) for x in arrs])
    n_cap = 2 + sum(len(x) for x in arrs)
    read_rc = np.full(n, 0xcd, dtype=np.uint8)
    read_qw = np.ascontiguousarray(np.concatenate(unit_filled(arrs, weights)).astype(np.uint8))
    hcfg = PoaConfig(**{**cfg.__dict__, "out_msa": True})       # read ids on the host side
    stats = {"nonzero": 0, "min": 0, "max_np": 0}
    with PoaSession(hcfg, product_lib) as s:
        a = s.abpt.contents
        ws = (C.c_int * n)(*[(-1 if a.wb < 0 else a.wb + int(np.float32(a.wf) * np.float32(len(x)))) for x in arrs])
        e = d.chain_emul_ps_new(n, lens, ptrs, ws, n_cap, K, A, a.m, a.max_mat, a.min_mis, a.gap_open1, a.gap_ext1,
                                a.gap_open1 + a.gap_ext1, a.gap_open2 + a.gap_ext2, W)
        if cfg.amb_strand:
            d.chain_emul_set_read_rc(e, read_rc.ctypes.data_as(c_u8_p))
        if cfg.use_qv:
            d.chain_emul_set_read_qw(e, read_qw.ctypes.data_as(c_u8_p))
        try:
            s.reset(max(len(x) for x in arrs))
            s.lib.dll.poa_graph_set_fast_order(s.ab.contents.abg, 1)
            s.lib.dll.poa_debug_blob.restype = C.c_int
            s.lib.dll.poa_debug_blob.argtypes = [C.c_void_p, C.c_void_p, c_u8_p, C.c_int, c_u8_p, C.c_int]
            blob_buf = np.zeros(64 + 16 * n_cap * 9 + max(len(x) for x in arrs) + 256, dtype=np.uint8)
            tot_cells = 0
            for i, x in enumerate(arrs):
                w = weights[i] if cfg.use_qv else None
                if i == 0:
                    _, res = oracle_align(s, x)
                    s.add(x, res, n, w)
                    d.chain_emul_ps_seed(e)
                else:
                    node_n = s.ab.contents.abg.contents.node_n
                    al, res = oracle_align(s, x)
                    seq, flag, cells = x, 0, al.cells
                    if cfg.amb_strand and d.chain_emul_weak_hit(al.best_score, len(x), node_n, a.max_mat):
                        assert host_weak_hit(al.best_score, len(x), node_n, a.max_mat)
                        al2, res2 = oracle_align(s, revcomp(x))
                        cells += al2.cells
                        if al2.best_score > al.best_score:
                            if res.n_cigar > 0:
                                capi.libc_free(res.graph_cigar)
                            seq, al, res, flag = revcomp(x), al2, res2, 3
                            w = None if w is None else np.ascontiguousarray(np.asarray(w)[::-1])
                        else:
                            if res2.n_cigar > 0:
                                capi.libc_free(res2.graph_cigar)
                            flag = 2
                    dev = device_cigar(s, al)
                    read_rc[i] = flag
                    tot_cells += cells
                    s.add(seq, res, n, w)
                    failed = d.chain_emul_ps_fuse(e, dev.ctypes.data_as(C.POINTER(C.c_uint64)), len(dev), al.best_score, cells)
                    assert failed == 0, f"read {i}: device chain gave up with flags {failed:#x}"
                    assert arr(d, e, 12, n)[i] == al.best_score and arr(d, e, 13, n)[i] == len(al.cigar)
                    assert int(np.ctypeslib.as_array(d.chain_emul_hashes(e), shape=(n,))[i]) == fnv1a_words(al.cigar), f"read {i}: CIGAR hash"
                nxt = arrs[i + 1] if i + 1 < n else None
                compare_graphs(d, e, s, i, K, A, nxt, blob_buf)
                if nxt is not None:
                    compare_predscore(d, e, blob_buf, i, stats)
            assert d.chain_emul_cells(e) == tot_cells
            s.lib.dll.poa_graph_set_fast_order(s.ab.contents.abg, 0)
            g = s.ab.contents.abg.contents
            g.is_topological_sorted = 0
            s.lib.abpoa_topological_sort(s.ab.contents.abg, s.abpt)

            # ---- consensus and coverage: the device's record against the host's on the same graph ----
            out = np.zeros(g.node_n + 1, dtype=np.int32)
            ln = d.chain_emul_consensus(e, out.ctypes.data_as(c_int_p), g.node_n)
            set_outputs(s.lib, s.abpt, 0)
            s.lib.abpoa_clean_msa_cons(s.ab)
            g.is_called_cons = 0
            s.lib.abpoa_generate_consensus(s.ab, s.abpt)
            assert ln == len(s.consensus()[0]), "consensus length"
            assert np.array_equal(out[1:1 + ln] & 0xff, s.consensus()[0]), "consensus bases"
            assert np.array_equal(out[1:1 + ln] >> 8, s.consensus_cov()[0]), "coverage"

            # ---- the device's -r 0 / -r 2 / -r 4 text, printed with the device's strands, is the reference's ----
            is_rc = [int(f & 1) for f in read_rc] if cfg.amb_strand else [0] * n
            if cfg.amb_strand:
                assert is_rc == reference_group(reference, cfg, reads, weights)["is_rc"], "strands differ from the reference's abpoa_msa"
            set_strands(s, n, is_rc)
            assert md5(consensus_text(d, pd, e, s, n, g.node_n)) == reference_group_md5(reference, cfg, reads, weights, 0), "-r 0"
            for r in (2, 4):
                got = device_text(d, pd, e, s, n, g.node_n, W, sum(len(x) for x in arrs), r)
                assert md5(got) == reference_group_md5(reference, cfg, reads, weights, r), f"-G -r {r}: device output differs from the reference's"
            return stats
        finally:
            d.chain_emul_free(e)


# ---- the graph code read by read ----
def test_syn_path_score(emul, product_lib, reference):
    c = CASES["syn_path_score"]
    st = drive_ps(emul, product_lib, reference, ps_cfg(PoaConfig(**c["cfg"])), case_reads(c))
    assert st["nonzero"] > 0 and st["min"] < 0, st


@pytest.mark.parametrize("seed", [0, 1])
def test_qv_weights_0_and_255(emul, product_lib, reference, seed):
    """-G -Q: zero-weight edges score 0 (and so do edges out of a node whose out-edges all weigh 0), 255s add up far past
    a byte."""
    reads = synth.make_group(9760 + seed, 9, 400, 0.08)
    weights = quality_weights(9770 + seed, reads)
    rng = np.random.default_rng(9780 + seed)
    for w in weights:
        u = rng.random(len(w))
        w[u < 0.25] = 0
        w[u > 0.75] = 255
    st = drive_ps(emul, product_lib, reference, ps_cfg(use_qv=True), reads, weights)
    assert st["nonzero"] > 0, st


@pytest.mark.parametrize("gap", ["convex", "affine"])
def test_strand_flipped_reads(emul, product_lib, reference, gap):
    """-G -s: the flatten scores the graph the flipped reads were fused into."""
    cfg = ps_cfg(PoaConfig(**({} if gap == "convex" else AFFINE)), amb_strand=True)
    reads = strand_mix(9790 + (gap == "affine"), 10, 350)
    drive_ps(emul, product_lib, reference, cfg, reads)


def test_amino_acids(emul, product_lib, reference):
    cfg = ps_cfg(PoaConfig(**synth.WORKLOADS["aa_blosum62_2k"].cfg.__dict__))
    reads = synth.make_group(9800, 7, 300, 0.08, m=27)
    drive_ps(emul, product_lib, reference, cfg, reads, K=32)


def test_rows_with_many_predecessors(emul, product_lib, reference):
    """A high-error group: rows with more than 4 predecessors (past the DP kernel's straight-line rows), scores down to
    the -20 clamp's neighbourhood."""
    reads = synth.make_group(9810, 16, 300, 0.25)
    st = drive_ps(emul, product_lib, reference, ps_cfg(), reads, K=24)
    assert st["max_np"] > 4, st


# ---- the score function ----
def reference_score(ew: int, nw: int) -> int:
    """The reference's expression with glibc's log (Python's math.log), rounded half away from zero as C's round."""
    if ew == 0 or nw == 0:
        return 0
    x = math.log(ew / nw)
    return max(int(math.copysign(math.floor(abs(x) + 0.5), x)), -20)


def test_score_function_all_pairs(emul):
    """chain_path_score against the reference's expression on every pair edge_w <= node_w <= 300, on pairs whose ratio
    sits near a rounding boundary, on node weights up to the admitted bound, and on 1 / 2^k past it (the -20 clamp)."""
    ew, nw = [], []
    for n in range(0, 301):
        for e in range(0, n + 1):
            ew.append(e); nw.append(n)
    for k in range(20):
        for n in (1000, 65521, 255 * 4000, MAX_NODE_W):
            t = n * math.exp(-(k + 0.5))
            for e in (math.floor(t) - 1, math.floor(t), math.floor(t) + 1, math.floor(t) + 2):
                if 0 <= e <= n:
                    ew.append(e); nw.append(n)
    for k in range(31):                 # 1 / 2^k: every score down to the -20 clamp
        ew.append(1); nw.append(1 << k)
    ew = np.ascontiguousarray(ew, dtype=np.int32)
    nw = np.ascontiguousarray(nw, dtype=np.int32)
    out = np.zeros(len(ew), dtype=np.int32)
    emul.chain_emul_path_scores(ew.ctypes.data_as(c_int_p), nw.ctypes.data_as(c_int_p), len(ew), out.ctypes.data_as(c_int_p))
    want = np.array([reference_score(int(e), int(n)) for e, n in zip(ew, nw)], dtype=np.int32)
    bad = np.flatnonzero(out != want)
    assert bad.size == 0, f"({ew[bad[0]]}, {nw[bad[0]]}): {out[bad[0]]} vs {want[bad[0]]}"
    assert set(out.tolist()) == set(range(-20, 1)), "every score -20..0 occurs"


def test_no_ratio_near_a_rounding_boundary():
    """For every node weight n <= POA_PS_MAX_NODE_W and every boundary -(k + 1/2), k = 0..19, the two edge weights around
    n e^-(k + 1/2) -- the only ones whose ln(e / n) can come near it -- keep ln(e / n) more than 1024 ulp of (k + 1/2) away
    from the boundary, in 64-bit extended precision.  A double division is exact to half an ulp and a log within a few ulp
    on the CPU and on the device, so both round every admitted ratio to the same integer."""
    assert np.finfo(np.longdouble).nmant >= 63, "needs x86 extended precision"
    n = np.arange(1, MAX_NODE_W + 1, dtype=np.longdouble)
    logn = np.log(n)
    worst = math.inf
    for k in range(20):
        b = np.longdouble(k) + np.longdouble(0.5)
        t = np.floor(n * np.exp(-b))
        for e in (t, t + 1):
            ok = (e >= 1) & (e <= n)
            if not ok.any():
                continue
            margin = np.abs(np.log(e[ok]) - logn[ok] + b)
            ulps = float(margin.min()) / float(np.spacing(np.float64(k + 0.5)))
            worst = min(worst, ulps)
    assert worst > 1024, f"a ratio lies {worst:.3g} ulp from a rounding boundary"


# ---- layouts ----
@pytest.mark.parametrize("strand", [0, 1])
@pytest.mark.parametrize("n_cap,qmax,n_reads,K,A,m,W,record", [(600, 300, 2, 12, 4, 5, 0, 0), (33_800, 10_500, 50, 12, 4, 5, 1, 1),
                                                              (2_000, 800, 130, 32, 26, 27, 3, 1)])
def test_layout_without_path_scores_unchanged(emul, n_cap, qmax, n_reads, K, A, m, W, record, strand):
    """A run without -G lays out its group exactly as before; -G grows the job blob by the predscore section only."""
    assert emul.chain_emul_ps_layout_check(n_cap, qmax, n_reads, K, A, m, W, record, strand) == 0
