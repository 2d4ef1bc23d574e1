"""CPU suite: the chain engine's row-column MSA (abpoa_b200/csrc/poa_chain.cuh: read sets in chain_seed / chain_fuse,
chain_msa_rank, chain_msa_rows) compiled for the host and driven read by read next to the product's host graph layer,
which is pinned to the reference.

After every read, the device read set of each node must equal the union of the host graph's per-edge read sets of that
node.  After the last read, the device ranks, msa_len and rows (with and without the consensus row) must equal what
abpoa_generate_rc_msa computes on the host graph, byte for byte."""
import ctypes as C
import subprocess
from pathlib import Path

import numpy as np
import pytest

from abpoa_b200 import synth
from abpoa_b200.aligner import PoaConfig, PoaSession
from abpoa_b200.capi import c_int_p, c_u8_p
from cases import AFFINE, CASES, case_reads
from helpers import INPUTS, read_fasta
from oracle_binding import oracle_align
from test_chain_emul import CHAIN_CASES

HERE = Path(__file__).resolve().parent
ROOT = HERE.parent
SO = HERE / "emul" / "libchain_emul_msa.so"


@pytest.fixture(scope="module")
def emul():
    """tests/emul/chain_emul_msa.cpp (chain_emul.cpp + the RC-MSA exports) compiled for the host."""
    srcs = [HERE / "emul" / "chain_emul_msa.cpp", HERE / "emul" / "chain_emul.cpp", ROOT / "abpoa_b200" / "csrc" / "poa_chain.cuh"]
    if not SO.exists() or SO.stat().st_mtime < max(p.stat().st_mtime for p in srcs):
        subprocess.run(["g++", "-O1", "-g", "-fPIC", "-shared", f"-I{ROOT / 'abpoa_b200' / 'csrc'}", f"-I{ROOT / 'include'}", f"-I{HERE / 'emul'}",
                        "-o", str(SO), str(srcs[0])], check=True)
    d = C.CDLL(str(SO))
    d.chain_emul_new.restype = C.c_void_p
    d.chain_emul_new.argtypes = [C.c_int, c_int_p, C.POINTER(c_u8_p), c_int_p] + [C.c_int] * 10
    d.chain_emul_msa_free.argtypes = [C.c_void_p]
    d.chain_emul_seed.argtypes = [C.c_void_p]
    d.chain_emul_fuse.restype = C.c_int
    d.chain_emul_fuse.argtypes = [C.c_void_p, C.POINTER(C.c_uint64), C.c_int, C.c_int, C.c_int64]
    d.chain_emul_n_nodes.argtypes = [C.c_void_p]
    d.chain_emul_enable_msa.argtypes = [C.c_void_p, C.c_int]
    d.chain_emul_read_set.restype = C.POINTER(C.c_uint64)
    d.chain_emul_read_set.argtypes = [C.c_void_p]
    d.chain_emul_msa_ranks.restype = c_int_p
    d.chain_emul_msa_ranks.argtypes = [C.c_void_p]
    d.chain_emul_msa.restype = C.c_int
    d.chain_emul_msa.argtypes = [C.c_void_p, C.c_int, c_u8_p, C.c_int64]
    return d


def host_read_sets(s, W):
    """[node_n, W] union of the per-edge read sets of every node's out-edges in the host graph."""
    g = s.ab.contents.abg.contents
    out = np.zeros((g.node_n, W), dtype=np.uint64)
    for v in range(g.node_n):
        nd = g.node[v]
        for e in range(nd.out_edge_n):
            for wd in range(min(nd.read_ids_n, W)):
                out[v, wd] |= np.uint64(nd.read_ids[e][wd])
    return out


def drive_msa(d, product_lib, cfg: PoaConfig, reads, K=12, extra_words=0):
    """Fuse `reads` with the emulated device code and the host graph layer side by side (alignments from the scalar
    oracle), comparing read sets after every read and the RC-MSA after the last one."""
    A = cfg.m - 1
    n = len(reads)
    W = (n + 63) // 64 + extra_words
    arrs = [np.ascontiguousarray(r, dtype=np.uint8) for r in reads]
    lens = (C.c_int * n)(*[len(a) for a in arrs])
    ptrs = (c_u8_p * n)(*[a.ctypes.data_as(c_u8_p) for a in arrs])
    n_cap = 2 + sum(len(a) for a in arrs)
    cfg = PoaConfig(**{**cfg.__dict__, "out_msa": True})        # per-edge read sets on the host side
    with PoaSession(cfg, product_lib) as s:
        a = s.abpt.contents
        ws = (C.c_int * n)(*[(-1 if a.wb < 0 else a.wb + int(np.float32(a.wf) * np.float32(len(x)))) for x in arrs])
        e = d.chain_emul_new(n, lens, ptrs, ws, n_cap, K, A, a.m, a.max_mat, a.min_mis, a.gap_open1, a.gap_ext1,
                             a.gap_open1 + a.gap_ext1, a.gap_open2 + a.gap_ext2)
        try:
            d.chain_emul_enable_msa(e, W)
            s.reset(max(len(x) for x in arrs))
            s.lib.dll.poa_graph_set_fast_order(s.ab.contents.abg, 1)
            for i, r in enumerate(arrs):
                al, res = oracle_align(s, r)
                if i == 0:
                    s.add(r, res, n)
                    d.chain_emul_seed(e)
                else:
                    g = s.ab.contents.abg.contents
                    row_of = np.ctypeslib.as_array(g.node_id_to_index, shape=(g.node_n,)).copy()
                    cig = al.cigar[::-1].copy()                  # backtrack order, DP rows instead of node ids
                    is_ins = (cig & np.uint64(0xf)) == np.uint64(1)
                    rows = row_of[(cig >> np.uint64(34)).astype(np.int64) % len(row_of)].astype(np.uint64)
                    dev = np.ascontiguousarray(np.where(is_ins, cig, (rows << np.uint64(34)) | (cig & np.uint64(0x3ffffffff))), dtype=np.uint64)
                    s.add(r, res, n)
                    failed = d.chain_emul_fuse(e, dev.ctypes.data_as(C.POINTER(C.c_uint64)), len(dev), al.best_score, al.cells)
                    assert failed == 0, f"read {i}: device chain gave up with flags {failed:#x}"
                nn = s.ab.contents.abg.contents.node_n
                assert d.chain_emul_n_nodes(e) == nn, f"read {i}: node_n"
                got = np.ctypeslib.as_array(d.chain_emul_read_set(e), shape=(nn * W,)).reshape(nn, W)
                want = host_read_sets(s, W)
                bad = np.nonzero((got != want).any(axis=1))[0]
                assert bad.size == 0, f"read {i}: read set of node {int(bad[0])}: device {got[bad[0]]}, host {want[bad[0]]}"
            # ---- RC-MSA after the last read: -r1 (no consensus row) and -r2 ----
            s.lib.dll.poa_graph_set_fast_order(s.ab.contents.abg, 0)
            nn = s.ab.contents.abg.contents.node_n
            buf = np.zeros((n + 1) * nn, dtype=np.uint8)
            for with_cons in (0, 1):
                a.out_cons = with_cons
                s.generate()
                want_rows = s.msa_rows()
                g = s.ab.contents.abg.contents
                want_rank = np.ctypeslib.as_array(g.node_id_to_msa_rank, shape=(nn,)).copy()
                buf[:] = 0xee
                msa_len = d.chain_emul_msa(e, with_cons, buf.ctypes.data_as(c_u8_p), len(buf))
                got_rank = np.ctypeslib.as_array(d.chain_emul_msa_ranks(e), shape=(nn,))
                assert np.array_equal(got_rank, want_rank), "MSA ranks differ from poa_set_msa_rank's"
                assert msa_len == len(want_rows[0]), f"msa_len {msa_len}, host {len(want_rows[0])}"
                assert len(want_rows) == n + with_cons
                for k, w in enumerate(want_rows):
                    row = buf[k * msa_len: (k + 1) * msa_len]
                    assert np.array_equal(row, w), f"with_cons={with_cons}: MSA row {k} differs at column {int(np.argmax(row != w))}"
                assert (buf[len(want_rows) * msa_len:] == 0xee).all(), "rows written past the record"
        finally:
            d.chain_emul_msa_free(e)


@pytest.mark.parametrize("name", CHAIN_CASES)
def test_device_msa_matches_host_layer(emul, product_lib, name):
    case = CASES[name]
    cfg = PoaConfig(**case["cfg"])
    drive_msa(emul, product_lib, cfg, case_reads(case), K=32 if cfg.m > 5 else 12)


@pytest.mark.parametrize("gap", ["convex", "affine"])
def test_device_msa_two_word_read_sets(emul, product_lib, gap):
    """3alleles.fa: 126 reads, so every read set spans two 64-bit words."""
    drive_msa(emul, product_lib, PoaConfig(**({} if gap == "convex" else AFFINE)), read_fasta(INPUTS / "3alleles.fa"))


@pytest.mark.parametrize("n_reads", [63, 64, 65, 128])
def test_device_msa_word_edges(emul, product_lib, n_reads):
    """Groups at the edges of a read-set word: the last read in bit 62, 63, 0 of the second word, 63 of the second word."""
    drive_msa(emul, product_lib, PoaConfig(), synth.make_group(7100 + n_reads, n_reads, 120, 0.08))


def test_device_msa_wider_read_sets_than_the_group_needs(emul, product_lib):
    """W comes from the largest group of a wave: a small group with spare words gives the same rows."""
    drive_msa(emul, product_lib, PoaConfig(), synth.make_group(7200, 9, 300, 0.10), extra_words=2)
