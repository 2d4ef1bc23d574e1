"""CPU suite: the DEVICE-side graph code (abpoa_b200/csrc/poa_chain.cuh: fusing a graph-CIGAR, spliced
topological order, edge order, max_remain, flattening into the next alignment job) compiled for the host
and driven read by read next to the product's host graph layer, which is pinned to the reference.

After every read every array must agree: bases, in/out edge lists with weights (order included),
aligned sets, n_read, the spliced row order, and the complete job blob for the next read byte for byte.
The alignments come from the scalar oracle (test harness arrangement, as in test_oracle.py)."""
import ctypes as C
import subprocess
from pathlib import Path

import numpy as np
import pytest

from abpoa_b200.aligner import PoaConfig, PoaSession
from abpoa_b200.batch import fnv1a_words
from abpoa_b200.capi import c_int_p, c_u8_p
from cases import CASES, case_reads
from oracle_binding import oracle_align

HERE = Path(__file__).resolve().parent
ROOT = HERE.parent
SO = HERE / "emul" / "libchain_emul.so"


@pytest.fixture(scope="module")
def emul():
    src = HERE / "emul" / "chain_emul.cpp"
    hdr = ROOT / "abpoa_b200" / "csrc" / "poa_chain.cuh"
    if not SO.exists() or SO.stat().st_mtime < max(src.stat().st_mtime, hdr.stat().st_mtime):
        subprocess.run(["g++", "-O1", "-g", "-fPIC", "-shared", f"-I{ROOT / 'abpoa_b200' / 'csrc'}", f"-I{ROOT / 'include'}", "-o", str(SO), str(src)], check=True)
    d = C.CDLL(str(SO))
    d.chain_emul_new.restype = C.c_void_p
    d.chain_emul_new.argtypes = [C.c_int, c_int_p, C.POINTER(c_u8_p), c_int_p] + [C.c_int] * 11
    d.chain_emul_free.argtypes = [C.c_void_p]
    d.chain_emul_seed.argtypes = [C.c_void_p]
    d.chain_emul_fuse.restype = C.c_int
    d.chain_emul_fuse.argtypes = [C.c_void_p, C.POINTER(C.c_uint64), C.c_int, C.c_int, C.c_int64]
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
    return d


def arr(d, e, which, n):
    return np.ctypeslib.as_array(d.chain_emul_array(e, which), shape=(n,)).copy()


def drive(emul, product_lib, cfg: PoaConfig, reads, K=12, A=None, n_cap=None):
    d = emul
    A = A if A is not None else cfg.m - 1
    n = len(reads)
    arrs = [np.ascontiguousarray(r, dtype=np.uint8) for r in reads]
    lens = (C.c_int * n)(*[len(a) for a in arrs])
    ptrs = (c_u8_p * n)(*[a.ctypes.data_as(c_u8_p) for a in arrs])
    n_cap = n_cap or (2 + sum(len(a) for a in arrs))
    with PoaSession(cfg, product_lib) as s:
        a = s.abpt.contents
        ws = (C.c_int * n)(*[(-1 if a.wb < 0 else a.wb + int(np.float32(a.wf) * np.float32(len(x)))) for x in arrs])
        e = d.chain_emul_new(n, lens, ptrs, ws, n_cap, K, A, a.m, a.max_mat, a.min_mis, a.gap_open1, a.gap_ext1,
                             a.gap_open1 + a.gap_ext1, a.gap_open2 + a.gap_ext2, 0)
        try:
            s.reset(max(len(x) for x in arrs))
            s.lib.dll.poa_graph_set_fast_order(s.ab.contents.abg, 1)
            s.lib.dll.poa_debug_blob.restype = C.c_int
            s.lib.dll.poa_debug_blob.argtypes = [C.c_void_p, C.c_void_p, c_u8_p, C.c_int, c_u8_p, C.c_int]
            blob_buf = np.zeros(64 + 16 * n_cap * 6 + max(len(x) for x in arrs) + 256, dtype=np.uint8)
            tot_cells = 0
            for i, r in enumerate(arrs):
                al, res = oracle_align(s, r)
                if i == 0:
                    assert not al.aligned
                    s.add(r, res, n)
                    d.chain_emul_seed(e)
                else:
                    g = s.ab.contents.abg.contents
                    row_of = np.ctypeslib.as_array(g.node_id_to_index, shape=(g.node_n,)).copy()
                    # the device's CIGAR: backtrack order, DP rows instead of node ids
                    cig = al.cigar[::-1].copy()
                    is_ins = (cig & np.uint64(0xf)) == np.uint64(1)
                    rows = row_of[(cig >> np.uint64(34)).astype(np.int64) % len(row_of)].astype(np.uint64)
                    dev = np.where(is_ins, cig, (rows << np.uint64(34)) | (cig & np.uint64(0x3ffffffff)))
                    dev = np.ascontiguousarray(dev, dtype=np.uint64)
                    tot_cells += al.cells
                    s.add(r, res, n)
                    failed = d.chain_emul_fuse(e, dev.ctypes.data_as(C.POINTER(C.c_uint64)), len(dev), al.best_score, al.cells)
                    assert failed == 0, f"read {i}: device chain gave up with flags {failed:#x}"
                    assert arr(d, e, 12, n)[i] == al.best_score and arr(d, e, 13, n)[i] == len(al.cigar)
                    assert int(np.ctypeslib.as_array(d.chain_emul_hashes(e), shape=(n,))[i]) == fnv1a_words(al.cigar), f"read {i}: CIGAR hash"
                # ---- compare the two graphs ----
                g = s.ab.contents.abg.contents
                if not g.is_topological_sorted:
                    s.lib.abpoa_topological_sort(s.ab.contents.abg, s.abpt)
                sig = s.graph_signature()
                nn = sig["node_n"]
                assert d.chain_emul_n_nodes(e) == nn, f"read {i}: node_n"
                bases = np.ctypeslib.as_array(d.chain_emul_bases(e), shape=(nn,))
                assert list(bases[2:]) == sig["bases"], f"read {i}: bases"
                in_cnt, out_cnt, aln_cnt, n_read = (arr(d, e, w, nn) for w in range(4))
                in_id, in_w, out_id, out_w = (arr(d, e, w, nn * K).reshape(nn, K) for w in range(4, 8))
                aln_id = arr(d, e, 8, nn * A).reshape(nn, A)
                for v in range(nn):
                    assert tuple(zip(in_id[v, : in_cnt[v]].tolist(), in_w[v, : in_cnt[v]].tolist())) == sig["in_edges"][v], f"read {i} node {v}: in-edges"
                    assert tuple(zip(out_id[v, : out_cnt[v]].tolist(), out_w[v, : out_cnt[v]].tolist())) == sig["out_edges"][v], f"read {i} node {v}: out-edges"
                    assert tuple(aln_id[v, : aln_cnt[v]].tolist()) == sig["aligned"][v], f"read {i} node {v}: aligned set"
                    assert n_read[v] == sig["n_read"][v][0], f"read {i} node {v}: n_read"
                assert np.array_equal(arr(d, e, 9, nn), sig["index_to_node_id"]), f"read {i}: spliced order"
                assert np.array_equal(arr(d, e, 10, nn), sig["node_id_to_index"]), f"read {i}: node -> row"
                if i + 1 < n:
                    nxt = arrs[i + 1]
                    nb = s.lib.dll.poa_debug_blob(s.ab, s.abpt, nxt.ctypes.data_as(c_u8_p), len(nxt), blob_buf.ctypes.data_as(c_u8_p), len(blob_buf))
                    assert nb > 0
                    got = np.ctypeslib.as_array(d.chain_emul_blob(e), shape=(nb,))
                    want = blob_buf[:nb]
                    hdr = want[:68].view(np.int32)           # PoaJobHeader: n_rows qlen w node_n off_rowmeta off_pred off_predscore off_live off_qs rsv[4] blob_bytes pn pad[2]
                    n_rows, off_rm, off_pred, off_qs, nbytes = int(hdr[0]), int(hdr[4]), int(hdr[5]), int(hdr[8]), int(hdr[13])
                    n_pred = int(want[off_rm + 8 * n_rows: off_rm + 8 * n_rows + 4].view(np.int32)[0])
                    # every section byte for byte (the 16-byte alignment gaps between sections are never written by either side)
                    for name_, a, b in (("header", 0, 68), ("rowmeta", off_rm, off_rm + 8 * (n_rows + 1)), ("pred", off_pred, off_pred + 4 * n_pred), ("query", off_qs, nbytes)):
                        assert np.array_equal(got[a:b], want[a:b]), f"read {i}: job blob for read {i + 1}: section {name_} differs at byte {a + int(np.argmax(got[a:b] != want[a:b]))}"
            assert d.chain_emul_cells(e) == tot_cells
            # ---- consensus computed by the device code vs the host's heaviest bundling on the same graph ----
            s.lib.dll.poa_graph_set_fast_order(s.ab.contents.abg, 0)
            s.ab.contents.abs.contents.n_seq = n
            s.generate()
            out = np.zeros(n_cap + 1, dtype=np.int32)
            ln = d.chain_emul_consensus(e, out.ctypes.data_as(c_int_p), len(out))
            cons, cov = s.consensus()[0], s.consensus_cov()[0]
            assert ln == len(cons), f"device consensus length {ln} vs host {len(cons)}"
            assert np.array_equal(out[1: 1 + ln] & 0xff, cons) and np.array_equal(out[1: 1 + ln] >> 8, cov), "device consensus / coverage differs from the host's"
        finally:
            d.chain_emul_free(e)


CHAIN_CASES = [n for n, c in CASES.items()
               if c["cfg"].get("align_mode", 0) == 0 and "weights" not in c and not c["cfg"].get("inc_path_score") and c["cfg"].get("wb", 10) >= 0]


@pytest.mark.parametrize("name", CHAIN_CASES)
def test_device_graph_code_matches_host_layer(emul, product_lib, name):
    case = CASES[name]
    cfg = PoaConfig(**case["cfg"])
    drive(emul, product_lib, cfg, case_reads(case), K=32 if cfg.m > 5 else 12)


def test_device_graph_code_deep_group(emul, product_lib):
    from abpoa_b200 import synth
    drive(emul, product_lib, PoaConfig(), synth.make_group(3100, 40, 700, 0.12))


def test_device_graph_capacity_flags(emul, product_lib):
    """Too few edge slots / node capacity: the chain must give up with a flag, never write out of bounds."""
    from abpoa_b200 import synth
    reads = synth.make_group(3200, 12, 300, 0.15)
    with pytest.raises(AssertionError, match="gave up"):
        drive(emul, product_lib, PoaConfig(), reads, K=2)
    with pytest.raises(AssertionError, match="gave up"):
        drive(emul, product_lib, PoaConfig(), reads, n_cap=330)


def test_device_graph_code_ragged_lengths(emul, product_lib):
    """Reads of very different lengths in one group (short reads fused into a long backbone and the other way round)."""
    from abpoa_b200 import synth
    rng = np.random.default_rng(11)
    base = synth.make_group(3300, 14, 600, 0.08)
    reads = [np.ascontiguousarray(r[: int(rng.integers(20, len(r)))]) if i % 3 == 1 else r for i, r in enumerate(base)]
    drive(emul, product_lib, PoaConfig(), reads)


def test_device_graph_code_high_error_amino_acid(emul, product_lib):
    """27-letter alphabet, BLOSUM62, 20 % error: aligned sets of up to 26 members, many mismatch siblings per column."""
    from abpoa_b200 import synth
    cfg = synth.WORKLOADS["aa_blosum62_2k"].cfg
    drive(emul, product_lib, cfg, synth.make_group(3400, 16, 250, 0.20, m=27), K=32)
