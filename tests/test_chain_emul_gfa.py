"""CPU suite: GFA output (-r 3 / -r 4).

The chain engine's GFA record (abpoa_b200/csrc/poa_chain.cuh: chain_gfa_order, chain_gfa_size, chain_gfa_record) is
compiled for the host and built read by read next to the product's host graph layer, from the scalar oracle's
alignments.  After the last read:
  - the device's FIFO order equals the host writer's;
  - the record, printed by the product's formatter (poa_gfa_record_text), equals what abpoa_generate_gfa prints on the
    host graph, byte for byte, with and without the consensus path;
  - that text equals the unmodified reference's (md5s in tests/golden/reference_runs_gfa.json, see
    tests/gfa_reference.py)."""
import ctypes as C
import subprocess
from pathlib import Path

import numpy as np
import pytest

from abpoa_b200 import synth
from abpoa_b200.aligner import PoaConfig, PoaSession
from abpoa_b200.capi import c_int_p, c_u8_p
from cases import AFFINE, CASES, case_reads
from gfa_reference import gfa_reference, md5, reference_msa_md5, with_file
from helpers import INPUTS, read_fasta
from oracle_binding import oracle_align
from test_chain_emul import CHAIN_CASES

HERE = Path(__file__).resolve().parent
ROOT = HERE.parent
SO = HERE / "emul" / "libchain_emul_gfa.so"


@pytest.fixture(scope="module")
def reference():
    ref = gfa_reference()
    yield ref
    ref.save()


@pytest.fixture(scope="module")
def emul():
    """tests/emul/chain_emul_gfa.cpp (chain_emul.cpp + the GFA exports) compiled for the host."""
    srcs = [HERE / "emul" / "chain_emul_gfa.cpp", HERE / "emul" / "chain_emul.cpp", ROOT / "abpoa_b200" / "csrc" / "poa_chain.cuh"]
    if not SO.exists() or SO.stat().st_mtime < max(p.stat().st_mtime for p in srcs):
        subprocess.run(["g++", "-O1", "-g", "-fPIC", "-shared", f"-I{ROOT / 'abpoa_b200' / 'csrc'}", f"-I{ROOT / 'include'}", f"-I{HERE / 'emul'}",
                        "-o", str(SO), str(srcs[0])], check=True)
    d = C.CDLL(str(SO))
    d.chain_emul_new.restype = C.c_void_p
    d.chain_emul_new.argtypes = [C.c_int, c_int_p, C.POINTER(c_u8_p), c_int_p] + [C.c_int] * 11
    d.chain_emul_free.argtypes = [C.c_void_p]
    d.chain_emul_seed.argtypes = [C.c_void_p]
    d.chain_emul_fuse.restype = C.c_int
    d.chain_emul_fuse.argtypes = [C.c_void_p, C.POINTER(C.c_uint64), C.c_int, C.c_int, C.c_int64]
    d.chain_emul_n_nodes.argtypes = [C.c_void_p]
    d.chain_emul_gfa_queue.restype = c_int_p
    d.chain_emul_gfa_queue.argtypes = [C.c_void_p]
    d.chain_emul_gfa.restype = C.c_int64
    d.chain_emul_gfa.argtypes = [C.c_void_p, C.c_int, c_int_p, C.c_int64]
    return d


def bind_product(lib):
    d = lib.dll
    d.poa_gfa_host_order.restype = C.c_int
    d.poa_gfa_host_order.argtypes = [C.c_void_p, c_int_p]
    d.poa_gfa_record_text.restype = C.c_void_p
    d.poa_gfa_record_text.argtypes = [c_int_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_size_t)]
    d.abpoa_generate_gfa.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    return d


def record_text(d, rec, s) -> bytes:
    n = C.c_size_t(0)
    p = d.poa_gfa_record_text(rec.ctypes.data_as(c_int_p), C.cast(s.ab, C.c_void_p), C.cast(s.abpt, C.c_void_p), C.byref(n))
    try:
        return C.string_at(p, n.value)
    finally:
        from abpoa_b200.capi import libc_free
        libc_free(p)


def drive_gfa(d, product_lib, reference, cfg: PoaConfig, reads, K=12, extra_words=0):
    """Fuse `reads` with the emulated device code and the host graph layer side by side (alignments from the scalar
    oracle); after the last read compare the device record's text with the host writer's and the reference's."""
    pd = bind_product(product_lib)
    A = cfg.m - 1
    n = len(reads)
    W = (n + 63) // 64 + extra_words
    arrs = [np.ascontiguousarray(r, dtype=np.uint8) for r in reads]
    lens = (C.c_int * n)(*[len(a) for a in arrs])
    ptrs = (c_u8_p * n)(*[a.ctypes.data_as(c_u8_p) for a in arrs])
    n_cap = 2 + sum(len(a) for a in arrs)
    hcfg = PoaConfig(**{**cfg.__dict__, "out_msa": True})       # per-edge read sets on the host side
    with PoaSession(hcfg, product_lib) as s:
        a = s.abpt.contents
        ws = (C.c_int * n)(*[(-1 if a.wb < 0 else a.wb + int(np.float32(a.wf) * np.float32(len(x)))) for x in arrs])
        e = d.chain_emul_new(n, lens, ptrs, ws, n_cap, K, A, a.m, a.max_mat, a.min_mis, a.gap_open1, a.gap_ext1,
                             a.gap_open1 + a.gap_ext1, a.gap_open2 + a.gap_ext2, W)
        try:
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
            s.lib.dll.poa_graph_set_fast_order(s.ab.contents.abg, 0)
            nn = s.ab.contents.abg.contents.node_n
            assert d.chain_emul_n_nodes(e) == nn
            # ---- FIFO order: device queue (SRC, then the segments) against the host writer's ----
            host_order = np.zeros(nn, dtype=np.int32)
            n_seg = pd.poa_gfa_host_order(C.cast(s.ab, C.c_void_p), host_order.ctypes.data_as(c_int_p))
            cap = 8 + 4 * nn + 2 * nn * ((n + 63) // 64) + sum(len(x) + 1 for x in arrs)
            rec = np.full(cap + 64, -0x33333334, dtype=np.int32)
            for with_cons in (0, 1):
                a.out_cons = with_cons
                s.lib.abpoa_clean_msa_cons(s.ab)
                s.ab.contents.abg.contents.is_called_cons = 0
                rec[:] = -0x33333334
                words = d.chain_emul_gfa(e, with_cons, rec.ctypes.data_as(c_int_p), cap)
                assert words > 0, f"no GFA record ({words})"
                assert (rec[words:] == -0x33333334).all(), "record written past its size"
                assert rec[0] == n_seg, f"{rec[0]} segments on the device, {n_seg} on the host"
                q = np.ctypeslib.as_array(d.chain_emul_gfa_queue(e), shape=(n_seg + 1,))
                assert q[0] == 0 and np.array_equal(q[1:], host_order[:n_seg]), "FIFO order differs from the host writer's"
                got = record_text(pd, rec, s)
                want = with_file(lambda fp: pd.abpoa_generate_gfa(C.cast(s.ab, C.c_void_p), C.cast(s.abpt, C.c_void_p), fp))
                assert got == want, f"with_cons={with_cons}: device record text differs from abpoa_generate_gfa at byte " \
                                    f"{next((k for k, (x, y) in enumerate(zip(got, want)) if x != y), min(len(got), len(want)))}"
                ref = reference_msa_md5(reference, cfg, reads, bool(with_cons))
                assert md5(want) == ref, f"with_cons={with_cons}: host GFA differs from the reference's"
        finally:
            d.chain_emul_free(e)


@pytest.mark.parametrize("name", CHAIN_CASES)
def test_device_gfa_matches_host_writer(emul, product_lib, reference, name):
    case = CASES[name]
    cfg = PoaConfig(**case["cfg"])
    drive_gfa(emul, product_lib, reference, cfg, case_reads(case), K=32 if cfg.m > 5 else 12)


@pytest.mark.parametrize("gap", ["convex", "affine"])
def test_device_gfa_two_word_read_sets(emul, product_lib, reference, gap):
    """3alleles.fa: 126 reads, so every read set spans two 64-bit words."""
    drive_gfa(emul, product_lib, reference, PoaConfig(**({} if gap == "convex" else AFFINE)), read_fasta(INPUTS / "3alleles.fa"))


@pytest.mark.parametrize("n_reads", [63, 64, 65, 128])
def test_device_gfa_word_edges(emul, product_lib, reference, n_reads):
    """Groups at the edges of a read-set word."""
    drive_gfa(emul, product_lib, reference, PoaConfig(), synth.make_group(7100 + n_reads, n_reads, 120, 0.08))


def test_device_gfa_spare_words(emul, product_lib, reference):
    """W comes from the largest group of a wave; the record keeps only the group's own words per set."""
    drive_gfa(emul, product_lib, reference, PoaConfig(), synth.make_group(7200, 9, 300, 0.10), extra_words=2)
