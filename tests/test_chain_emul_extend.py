"""CPU suite: the device graph code in extend mode (-m 2, with and without z-drop).

In extend mode the DP result depends on the order of the rows (the best cell is the first row in row order that holds
the maximum; the z-drop stop is the first row that meets its condition), so the chain keeps the reference's FIFO Kahn
order there (chain_kahn_order in poa_chain.cuh, chain_fuse's KO instantiation) instead of its spliced order.

1. tests/test_chain_emul.py's drive() on the KO fuse: read by read next to the product's host graph layer (which runs the
   full Kahn pass after every read in extend mode), the row order, every graph array (edge lists in their order, aligned
   sets, n_read) and the whole next job blob must equal the host's.  The alignments are the scalar oracle's extend /
   z-drop alignments.
2. The spliced order is a different topological order on these inputs, and an extend alignment to the graph in the
   spliced order gives a different result than in the Kahn order: a fuse that fell back to the splice would fail (1)."""
import ctypes as C
import subprocess
from pathlib import Path

import numpy as np
import pytest

from abpoa_b200 import synth
from abpoa_b200.aligner import PoaConfig, PoaSession
from abpoa_b200.capi import ABPOA_EXTEND_MODE, c_int_p, c_u8_p
from cases import AFFINE, CASES, case_reads
from oracle_binding import oracle_align
from test_chain_emul import drive

HERE = Path(__file__).resolve().parent
ROOT = HERE.parent
SO = HERE / "emul" / "libchain_emul_extend.so"
AA = synth.WORKLOADS["aa_blosum62_2k"].cfg


@pytest.fixture(scope="module")
def xemul():
    src = HERE / "emul" / "chain_emul_extend.cpp"
    deps = [src, HERE / "emul" / "chain_emul.cpp", ROOT / "abpoa_b200" / "csrc" / "poa_chain.cuh"]
    if not SO.exists() or SO.stat().st_mtime < max(p.stat().st_mtime for p in deps):
        subprocess.run(["g++", "-O1", "-g", "-fPIC", "-shared", f"-I{ROOT / 'abpoa_b200' / 'csrc'}", f"-I{ROOT / 'include'}", "-o", str(SO), str(src)], check=True)
    d = C.CDLL(str(SO))
    d.chain_emul_new.restype = C.c_void_p
    d.chain_emul_new.argtypes = [C.c_int, c_int_p, C.POINTER(c_u8_p), c_int_p] + [C.c_int] * 11
    d.chain_emul_free.argtypes = [C.c_void_p]
    d.chain_emul_seed.argtypes = [C.c_void_p]
    for f in (d.chain_emul_fuse, d.chain_emul_x_fuse):
        f.restype = C.c_int
        f.argtypes = [C.c_void_p, C.POINTER(C.c_uint64), C.c_int, C.c_int, C.c_int64]
    d.chain_emul_n_nodes.argtypes = [C.c_void_p]
    d.chain_emul_failed.argtypes = [C.c_void_p]
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
    d.chain_emul_kahn.restype = C.c_int
    d.chain_emul_kahn.argtypes = [C.c_void_p, c_int_p]
    return d


class KahnFuse:
    """The emulator library with chain_emul_fuse bound to the extend runs' (KO) fuse, for drive()."""

    def __init__(self, d):
        self._d = d
        self.chain_emul_fuse = d.chain_emul_x_fuse

    def __getattr__(self, name):
        return getattr(self._d, name)


def ext(**kw):
    return PoaConfig(align_mode=ABPOA_EXTEND_MODE, **kw)


def ragged():
    rng = np.random.default_rng(21)
    base = synth.make_group(7100, 12, 700, 0.08)
    return [np.ascontiguousarray(r[: int(rng.integers(15, len(r)))]) if i % 3 == 1 else r for i, r in enumerate(base)]


EMUL_CASES = {
    "syn_extend_affine": lambda: (case_reads(CASES["syn_extend_affine"]), PoaConfig(**CASES["syn_extend_affine"]["cfg"])),
    "syn_extend_convex_zdrop": lambda: (case_reads(CASES["syn_extend_convex_zdrop"]), PoaConfig(**CASES["syn_extend_convex_zdrop"]["cfg"])),
    "convex_5pct": lambda: (synth.make_group(7001, 14, 900, 0.05), ext()),
    "affine_25pct": lambda: (synth.make_group(7002, 10, 500, 0.25), ext(**AFFINE)),
    "convex_25pct_zdrop": lambda: (synth.make_group(7003, 10, 500, 0.25), ext(zdrop=30)),
    "convex_zdrop_fires": lambda: (synth.make_group(7004, 10, 600, 0.15), ext(zdrop=10)),
    "ragged_convex": lambda: (ragged(), ext()),
    "ragged_affine_zdrop": lambda: (ragged(), ext(zdrop=50, **AFFINE)),
    "amino_acids": lambda: (synth.make_group(7005, 10, 300, 0.20, m=27), ext(m=27, score_matrix=AA.score_matrix, **AFFINE)),
    "amino_acids_zdrop": lambda: (synth.make_group(7006, 8, 300, 0.10, m=27), ext(m=27, score_matrix=AA.score_matrix, zdrop=40, **AFFINE)),
}


@pytest.mark.parametrize("name", list(EMUL_CASES))
def test_device_graph_code_extend(xemul, product_lib, name):
    """After every read: the Kahn row order, every graph array and the next job blob equal the host layer's."""
    reads, cfg = EMUL_CASES[name]()
    drive(KahnFuse(xemul), product_lib, cfg, reads, K=32 if cfg.m > 5 else 12)


def host_graph_stats(product_lib, cfg, reads):
    """(nodes with in-degree >= 2, largest aligned set) of the host graph after the group, the oracle aligning."""
    with PoaSession(cfg, product_lib) as s:
        s.reset(max(len(r) for r in reads))
        for r in reads:
            _, res = oracle_align(s, r)
            s.add(r, res, len(reads))
        sig = s.graph_signature()
    return sum(len(e) >= 2 for e in sig["in_edges"]), max(len(a) for a in sig["aligned"])


def test_inputs_cover_merges_and_full_aligned_sets(product_lib):
    """The high-error groups have nodes with in-degree >= 2, the DNA ones full aligned sets (a column of all four bases:
    three siblings), the amino-acid one sets of four or more."""
    for name in ("affine_25pct", "convex_25pct_zdrop", "amino_acids"):
        reads, cfg = EMUL_CASES[name]()
        merges, aln = host_graph_stats(product_lib, cfg, reads)
        assert merges > 20, name
        assert aln >= (3 if cfg.m == 5 else 4), f"{name}: largest aligned set {aln}"


def test_zdrop_stops_the_oracle_early(product_lib):
    """On convex_zdrop_fires z-drop ends alignments early: the oracle computes fewer cells, and reaches a different
    alignment, than without z-drop on the same graphs."""
    reads, cfg = EMUL_CASES["convex_zdrop_fires"]()
    fired = changed = 0
    with PoaSession(cfg, product_lib) as s:
        s.reset(max(len(r) for r in reads))
        for r in reads:
            a, res = oracle_align(s, r)
            if a.aligned:
                s.abpt.contents.zdrop = -1               # the same graph, without z-drop
                try:
                    b, _ = oracle_align(s, r)
                finally:
                    s.abpt.contents.zdrop = cfg.zdrop
                fired += a.cells < b.cells
                changed += a.best_score != b.best_score or not np.array_equal(a.cigar, b.cigar)
            s.add(r, res, len(reads))
    assert fired >= 3 and changed >= 1, (fired, changed)


def test_spliced_order_would_change_extend_results(xemul, product_lib):
    """Next to the KO fuse, a second emulator keeps the spliced order of the global fuse on the same graph.  The two orders
    differ, and aligning the next read (scalar oracle, extend mode) to the graph in the spliced order gives another
    score or graph-CIGAR than in the Kahn order on some reads: the row order is part of the extend result."""
    d = xemul
    differ_order = differ_result = 0
    for name in ("convex_5pct", "affine_25pct", "convex_25pct_zdrop"):
        reads, cfg = EMUL_CASES[name]()
        arrs = [np.ascontiguousarray(r, dtype=np.uint8) for r in reads]
        n = len(arrs)
        lens = (C.c_int * n)(*[len(a) for a in arrs])
        ptrs = (c_u8_p * n)(*[a.ctypes.data_as(c_u8_p) for a in arrs])
        n_cap = 2 + sum(len(a) for a in arrs)
        with PoaSession(cfg, product_lib) as s:
            a = s.abpt.contents
            ws = (C.c_int * n)(*[a.wb + int(np.float32(a.wf) * np.float32(len(x))) for x in arrs])
            args = (n, lens, ptrs, ws, n_cap, 12, cfg.m - 1, a.m, a.max_mat, a.min_mis, a.gap_open1, a.gap_ext1,
                    a.gap_open1 + a.gap_ext1, a.gap_open2 + a.gap_ext2, 0)
            ek, es = d.chain_emul_new(*args), d.chain_emul_new(*args)
            try:
                s.reset(max(len(x) for x in arrs))
                for i, r in enumerate(arrs):
                    al, res = oracle_align(s, r)
                    if i == 0:
                        s.add(r, res, n)
                        d.chain_emul_seed(ek)
                        d.chain_emul_seed(es)
                        continue
                    cig = al.cigar[::-1].copy()
                    is_ins = (cig & np.uint64(0xf)) == np.uint64(1)
                    ids = (cig >> np.uint64(34)).astype(np.int64)
                    for e, fuse in ((ek, d.chain_emul_x_fuse), (es, d.chain_emul_fuse)):
                        nn = d.chain_emul_n_nodes(e)
                        row_of = np.ctypeslib.as_array(d.chain_emul_array(e, 10), shape=(nn,)).copy()
                        dev = np.where(is_ins, cig, (row_of[ids % nn].astype(np.uint64) << np.uint64(34)) | (cig & np.uint64(0x3ffffffff)))
                        dev = np.ascontiguousarray(dev, dtype=np.uint64)
                        assert fuse(e, dev.ctypes.data_as(C.POINTER(C.c_uint64)), len(dev), al.best_score, al.cells) == 0
                    s.add(r, res, n)
                    if i + 1 == n:
                        break
                    g = s.ab.contents.abg.contents
                    if not g.is_topological_sorted:
                        s.lib.abpoa_topological_sort(s.ab.contents.abg, s.abpt)
                    nn = g.node_n
                    kahn = np.ctypeslib.as_array(d.chain_emul_array(ek, 9), shape=(nn,)).copy()
                    spliced = np.ctypeslib.as_array(d.chain_emul_array(es, 9), shape=(nn,)).copy()
                    host_order = np.ctypeslib.as_array(g.index_to_node_id, shape=(nn,))
                    host_index = np.ctypeslib.as_array(g.node_id_to_index, shape=(nn,))
                    assert np.array_equal(kahn, host_order), f"{name} read {i}: Kahn order"
                    if np.array_equal(kahn, spliced):
                        continue
                    differ_order += 1
                    want, _ = oracle_align(s, arrs[i + 1])
                    host_order[:] = spliced                      # the host graph in the spliced order, for one alignment
                    host_index[spliced] = np.arange(nn, dtype=np.int32)
                    try:
                        got, _ = oracle_align(s, arrs[i + 1])
                    finally:
                        host_order[:] = kahn
                        host_index[kahn] = np.arange(nn, dtype=np.int32)
                    differ_result += got.best_score != want.best_score or not np.array_equal(got.cigar, want.cigar)
            finally:
                d.chain_emul_free(ek)
                d.chain_emul_free(es)
    assert differ_order >= 5 and differ_result >= 1, (differ_order, differ_result)


def test_kahn_walk_flags_a_graph_that_is_not_a_dag(xemul, product_lib):
    """A cycle (an out-edge back to SRC's successor) leaves nodes that never become ready: the walk flags the order."""
    d = xemul
    reads = synth.make_group(7007, 2, 50, 0.0)
    arrs = [np.ascontiguousarray(r, dtype=np.uint8) for r in reads]
    lens = (C.c_int * 2)(*[len(a) for a in arrs])
    ptrs = (c_u8_p * 2)(*[a.ctypes.data_as(c_u8_p) for a in arrs])
    e = d.chain_emul_new(2, lens, ptrs, (C.c_int * 2)(20, 20), 200, 12, 4, 5, 2, 4, 4, 2, 6, 25, 0)
    try:
        d.chain_emul_seed(e)
        order = np.zeros(52, dtype=np.int32)
        assert d.chain_emul_kahn(e, order.ctypes.data_as(c_int_p)) == 0
        assert list(order) == [0] + list(range(2, 52)) + [1]
        nn = d.chain_emul_n_nodes(e)
        in_cnt = np.ctypeslib.as_array(d.chain_emul_array(e, 0), shape=(nn,))
        out_cnt = np.ctypeslib.as_array(d.chain_emul_array(e, 1), shape=(nn,))
        in_id = np.ctypeslib.as_array(d.chain_emul_array(e, 4), shape=(nn * 12,))
        out_id = np.ctypeslib.as_array(d.chain_emul_array(e, 6), shape=(nn * 12,))
        out_id[30 * 12 + 1] = 10                         # node 30 -> node 10: a cycle 10 .. 30 -> 10
        out_cnt[30] = 2
        in_id[10 * 12 + 1] = 30
        in_cnt[10] = 2
        assert d.chain_emul_kahn(e, order.ctypes.data_as(c_int_p)) & 0x08
    finally:
        d.chain_emul_free(e)
