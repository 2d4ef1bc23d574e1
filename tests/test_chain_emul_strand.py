"""CPU suite: ambiguous-strand alignment (-s) on the chain engine's graph code.

The device-side graph code (abpoa_b200/csrc/poa_chain.cuh) is compiled for the host and driven read by read next to the
product's host graph layer.  Both strands of every read are aligned by the scalar oracle; the strand is picked as the
alignment warp picks it (chain_weak_hit, then the reverse complement only if it scores strictly more), the host graph
fuses the winning bases and the device code reads them through the slot's strand bytes (chain_read_base).  After every
read every graph array and the next job blob must agree; after the last read the strands must be the reference's
(abpoa_msa), and the device's -r 1 / -r 2 rows and -r 3 / -r 4 GFA record, printed with the device's strands, must be
the reference's text (md5s in tests/golden/reference_runs_strand.json, see tests/strand_reference.py)."""
import ctypes as C
import subprocess
from pathlib import Path

import numpy as np
import pytest

from abpoa_b200 import capi, synth
from abpoa_b200.aligner import PoaConfig, PoaSession
from abpoa_b200.batch import fnv1a_words
from abpoa_b200.capi import c_int_p, c_u8_p
from cases import AFFINE
from gfa_reference import md5, with_file
from mf_reference import set_outputs, with_n
from oracle_binding import oracle_align
from strand_reference import names_of, reference_group, reference_group_md5, revcomp, strand_cfg, strand_mix, strand_reference
from test_chain_emul_gfa import bind_product, record_text

HERE = Path(__file__).resolve().parent
ROOT = HERE.parent
SO = HERE / "emul" / "libchain_emul_strand.so"


@pytest.fixture(scope="module")
def reference():
    ref = strand_reference()
    yield ref
    ref.save()


@pytest.fixture(scope="module")
def emul():
    """tests/emul/chain_emul_strand.cpp (chain_emul.cpp + the -s exports) compiled for the host."""
    srcs = [HERE / "emul" / "chain_emul_strand.cpp", HERE / "emul" / "chain_emul.cpp", ROOT / "abpoa_b200" / "csrc" / "poa_chain.cuh"]
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
    d.chain_emul_msa.restype = C.c_int
    d.chain_emul_msa.argtypes = [C.c_void_p, C.c_int, c_u8_p, C.c_int64]
    d.chain_emul_gfa.restype = C.c_int64
    d.chain_emul_gfa.argtypes = [C.c_void_p, C.c_int, c_int_p, C.c_int64]
    d.chain_emul_layout_check.restype = C.c_int
    d.chain_emul_layout_check.argtypes = [C.c_int] * 8
    return d


def arr(d, e, which, n):
    return np.ctypeslib.as_array(d.chain_emul_array(e, which), shape=(n,)).copy()


def host_weak_hit(score, qlen, node_n, max_mat):
    """The host's expression (poa_msa.c, reference src/abpoa_align.c:323-325) in IEEE double, as C evaluates it."""
    return score < min(qlen, node_n - 2) * max_mat * .3333


def device_cigar(s, al):
    """The alignment as the kernel leaves it in jd.cigar: backtrack order, DP rows instead of node ids."""
    g = s.ab.contents.abg.contents
    row_of = np.ctypeslib.as_array(g.node_id_to_index, shape=(g.node_n,)).copy()
    cig = al.cigar[::-1].copy()
    is_ins = (cig & np.uint64(0xf)) == np.uint64(1)
    rows = row_of[(cig >> np.uint64(34)).astype(np.int64) % len(row_of)].astype(np.uint64)
    return np.ascontiguousarray(np.where(is_ins, cig, (rows << np.uint64(34)) | (cig & np.uint64(0x3ffffffff))), dtype=np.uint64)


def compare_graphs(d, e, s, i, K, A, next_read, blob_buf):
    """Every graph array of the device code against the host graph, and the job blob for the next (forward) read."""
    g = s.ab.contents.abg.contents
    if not g.is_topological_sorted:
        s.lib.abpoa_topological_sort(s.ab.contents.abg, s.abpt)
    sig = s.graph_signature()
    nn = sig["node_n"]
    assert d.chain_emul_n_nodes(e) == nn, f"read {i}: node_n"
    assert list(np.ctypeslib.as_array(d.chain_emul_bases(e), shape=(nn,))[2:]) == sig["bases"], f"read {i}: bases"
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
    if next_read is None:
        return
    nb = s.lib.dll.poa_debug_blob(s.ab, s.abpt, next_read.ctypes.data_as(c_u8_p), len(next_read), blob_buf.ctypes.data_as(c_u8_p), len(blob_buf))
    assert nb > 0
    got = np.ctypeslib.as_array(d.chain_emul_blob(e), shape=(nb,))
    want = blob_buf[:nb]
    hdr = want[:68].view(np.int32)
    n_rows, off_rm, off_pred, off_qs, nbytes = int(hdr[0]), int(hdr[4]), int(hdr[5]), int(hdr[8]), int(hdr[13])
    n_pred = int(want[off_rm + 8 * n_rows: off_rm + 8 * n_rows + 4].view(np.int32)[0])
    for name_, a, b in (("header", 0, 68), ("rowmeta", off_rm, off_rm + 8 * (n_rows + 1)), ("pred", off_pred, off_pred + 4 * n_pred), ("query", off_qs, nbytes)):
        assert np.array_equal(got[a:b], want[a:b]), f"read {i}: job blob for read {i + 1}: section {name_} differs at byte {a + int(np.argmax(got[a:b] != want[a:b]))}"


def set_names(s, n, is_rc):
    """Names r0, r1, ... (as strand_reference.group_text hands them to abpoa_msa) and the strands, on the host handle."""
    abs_ = s.ab.contents.abs.contents
    abs_.n_seq = n
    for i, nm in enumerate(names_of(n)):
        b = nm.encode()
        buf = capi.libc_realloc(None, len(b) + 1)
        C.memmove(buf, b + b"\0", len(b) + 1)
        abs_.name[i].s = C.cast(buf, C.c_char_p)
        abs_.name[i].l = len(b)
        abs_.name[i].m = len(b) + 1
        abs_.is_rc[i] = int(is_rc[i])


def device_text(d, pd, e, s, n, nn, W, bases, r) -> bytes:
    """The -r r text of the device's results after the last read, printed by the product's writers."""
    set_outputs(s.lib, s.abpt, r)
    if r in (3, 4):
        cap = 8 + 4 * nn + 2 * nn * W + bases + n
        rec = np.full(cap + 64, -0x33333334, dtype=np.int32)
        assert d.chain_emul_gfa(e, int(r == 4), rec.ctypes.data_as(c_int_p), cap) > 0, "no GFA record"
        return record_text(pd, rec, s)
    with_cons = int(r == 2)
    s.lib.abpoa_clean_msa_cons(s.ab)
    if with_cons:                                   # as the engine installs them: the consensus first (-r 1 has none)
        out = np.zeros(nn + 1, dtype=np.int32)
        ln = d.chain_emul_consensus(e, out.ctypes.data_as(c_int_p), nn)
        base = np.ascontiguousarray(out[1:1 + ln] & 0xff, dtype=np.uint8)
        cov = np.ascontiguousarray(out[1:1 + ln] >> 8, dtype=np.int32)
        pd.poa_cons_install.argtypes = [C.c_void_p, C.c_int, C.c_int, c_u8_p, c_int_p]
        pd.poa_cons_install(C.cast(s.ab, C.c_void_p), n, ln, base.ctypes.data_as(c_u8_p), cov.ctypes.data_as(c_int_p))
    pd.poa_msa_install.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, c_u8_p]
    rows = np.zeros((n + 1) * nn, dtype=np.uint8)
    msa_len = d.chain_emul_msa(e, with_cons, rows.ctypes.data_as(c_u8_p), len(rows))
    assert msa_len > 0, f"no MSA ({msa_len})"
    pd.poa_msa_install(C.cast(s.ab, C.c_void_p), n, n + with_cons, msa_len, rows.ctypes.data_as(c_u8_p))
    return with_file(lambda fp: s.lib.abpoa_output(s.ab, s.abpt, fp))


def drive_strand(d, product_lib, reference, cfg: PoaConfig, reads, K=12):
    """Fuse `reads` with the emulated device code and the host graph layer side by side, each read on the strand the
    alignment warp would pick; returns the strand bytes (bit 0 flipped, bit 1 the reverse complement was aligned)."""
    pd = bind_product(product_lib)
    A = cfg.m - 1
    n = len(reads)
    W = (n + 63) // 64
    arrs = [np.ascontiguousarray(x, dtype=np.uint8) for x in reads]
    lens = (C.c_int * n)(*[len(x) for x in arrs])
    ptrs = (c_u8_p * n)(*[x.ctypes.data_as(c_u8_p) for x in arrs])
    n_cap = 2 + sum(len(x) for x in arrs)
    read_rc = np.full(n, 0xcd, dtype=np.uint8)
    hcfg = PoaConfig(**{**cfg.__dict__, "out_msa": True})       # read ids on the host side
    with PoaSession(hcfg, product_lib) as s:
        a = s.abpt.contents
        ws = (C.c_int * n)(*[(-1 if a.wb < 0 else a.wb + int(np.float32(a.wf) * np.float32(len(x)))) for x in arrs])
        e = d.chain_emul_new(n, lens, ptrs, ws, n_cap, K, A, a.m, a.max_mat, a.min_mis, a.gap_open1, a.gap_ext1,
                             a.gap_open1 + a.gap_ext1, a.gap_open2 + a.gap_ext2, W)
        d.chain_emul_set_read_rc(e, read_rc.ctypes.data_as(c_u8_p))
        try:
            s.reset(max(len(x) for x in arrs))
            s.lib.dll.poa_graph_set_fast_order(s.ab.contents.abg, 1)
            s.lib.dll.poa_debug_blob.restype = C.c_int
            s.lib.dll.poa_debug_blob.argtypes = [C.c_void_p, C.c_void_p, c_u8_p, C.c_int, c_u8_p, C.c_int]
            blob_buf = np.zeros(64 + 16 * n_cap * 6 + max(len(x) for x in arrs) + 256, dtype=np.uint8)
            tot_cells = 0
            for i, x in enumerate(arrs):
                if i == 0:
                    _, res = oracle_align(s, x)
                    s.add(x, res, n)
                    d.chain_emul_seed(e)
                    assert read_rc[0] == 0, "the seed must clear read 0's strand byte"
                else:
                    node_n = s.ab.contents.abg.contents.node_n
                    al, res = oracle_align(s, x)
                    weak = d.chain_emul_weak_hit(al.best_score, len(x), node_n, a.max_mat)
                    assert bool(weak) == host_weak_hit(al.best_score, len(x), node_n, a.max_mat)
                    seq, flag, cells = x, 0, al.cells
                    if weak:
                        y = revcomp(x)
                        al2, res2 = oracle_align(s, y)
                        cells += al2.cells
                        if al2.best_score > al.best_score:            # a tie keeps the forward strand
                            if res.n_cigar > 0:
                                capi.libc_free(res.graph_cigar)
                            seq, al, res, flag = y, al2, res2, 3
                        else:
                            if res2.n_cigar > 0:
                                capi.libc_free(res2.graph_cigar)
                            flag = 2
                    dev = device_cigar(s, al)
                    read_rc[i] = flag
                    tot_cells += cells
                    s.add(seq, res, n)
                    failed = d.chain_emul_fuse(e, dev.ctypes.data_as(C.POINTER(C.c_uint64)), len(dev), al.best_score, cells)
                    assert failed == 0, f"read {i}: device chain gave up with flags {failed:#x}"
                    assert arr(d, e, 12, n)[i] == al.best_score and arr(d, e, 13, n)[i] == len(al.cigar)
                    assert int(np.ctypeslib.as_array(d.chain_emul_hashes(e), shape=(n,))[i]) == fnv1a_words(al.cigar), f"read {i}: CIGAR hash"
                compare_graphs(d, e, s, i, K, A, arrs[i + 1] if i + 1 < n else None, blob_buf)
            assert d.chain_emul_cells(e) == tot_cells
            s.lib.dll.poa_graph_set_fast_order(s.ab.contents.abg, 0)
            g = s.ab.contents.abg.contents
            g.is_topological_sorted = 0
            s.lib.abpoa_topological_sort(s.ab.contents.abg, s.abpt)

            # ---- the strands are the reference's ----
            is_rc = [int(f & 1) for f in read_rc]
            assert is_rc == reference_group(reference, cfg, reads)["is_rc"], "strands differ from the reference's abpoa_msa"

            # ---- the device's MSA rows and GFA record, printed with the device's strands, are the reference's text ----
            set_names(s, n, is_rc)
            for r in (1, 2, 3, 4):
                got = device_text(d, pd, e, s, n, g.node_n, W, sum(len(x) for x in arrs), r)
                assert md5(got) == reference_group_md5(reference, cfg, reads, r), f"-s -r {r}: device output differs from the reference's"
            return read_rc.copy()
        finally:
            d.chain_emul_free(e)


@pytest.mark.parametrize("gap", ["convex", "affine"])
@pytest.mark.parametrize("seed", [0, 1])
def test_strand_mix(emul, product_lib, reference, gap, seed):
    """Every third read arrives reverse-complemented: those, and only those, are flipped."""
    cfg = strand_cfg(PoaConfig(**({} if gap == "convex" else AFFINE)))
    reads = strand_mix(9900 + 10 * seed + (gap == "affine"), 10, 300 + 100 * seed)
    flags = drive_strand(emul, product_lib, reference, cfg, reads)
    assert [int(f & 1) for f in flags] == [int(i % 3 == 1) for i in range(len(reads))]


def test_reads_with_n(emul, product_lib, reference):
    """Code 4 (N) stays 4 in the reverse complement."""
    reads = with_n(strand_mix(9920, 9, 250), 9921, 4, 0.03)
    flags = drive_strand(emul, product_lib, reference, strand_cfg(), reads)
    assert sum(f & 1 for f in flags) >= 2


def test_amino_acids(emul, product_lib, reference):
    """-c: the complement rule is applied unchanged (codes 0..3 become 3..0, every other code 4)."""
    cfg = strand_cfg(PoaConfig(**synth.WORKLOADS["aa_blosum62_2k"].cfg.__dict__))
    reads = strand_mix(9930, 7, 200, 0.08, m=27)
    drive_strand(emul, product_lib, reference, cfg, reads, K=32)


def test_unrelated_reads(emul, product_lib, reference):
    """Random reads: both strands are weak, and some weak reads keep their forward alignment."""
    rng = np.random.default_rng(9940)
    reads = [rng.integers(0, 4, size=int(rng.integers(150, 260))).astype(np.uint8) for _ in range(8)]
    flags = drive_strand(emul, product_lib, reference, strand_cfg(), reads)
    assert all(f & 2 for f in flags[1:]), "every read of unrelated sequence is a weak hit"
    assert any(f == 2 for f in flags[1:]), "no weak read kept its forward alignment"


def test_no_flipped_read(emul, product_lib, reference):
    flags = drive_strand(emul, product_lib, reference, strand_cfg(), synth.make_group(9950, 8, 300, 0.05))
    assert not any(flags), "a read of a same-strand group was retried or flipped"


@pytest.mark.parametrize("max_mat", [1, 2, 3, 5])
@pytest.mark.parametrize("qlen,node_n", [(120, 400), (2999, 3003), (400, 122), (3003, 2999)])
def test_weak_hit_boundaries(emul, qlen, node_n, max_mat):
    """The shared predicate against the host expression at the threshold, one below and one above it, with qlen below
    and above node_n - 2."""
    thr = min(qlen, node_n - 2) * max_mat * .3333
    for score in {int(np.floor(thr)) - 1, int(np.floor(thr)), int(np.ceil(thr)), int(np.ceil(thr)) + 1, round(thr)}:
        assert bool(emul.chain_emul_weak_hit(score, qlen, node_n, max_mat)) == host_weak_hit(score, qlen, node_n, max_mat), (score, thr)
    # lim * max_mat = 10000: the double product lands next to the integer 3333
    lim = 10000 // max_mat
    thr = lim * max_mat * .3333
    s = round(thr)
    for q, nn in ((lim, lim + 100), (lim + 100, lim + 2)):
        for score in (s - 1, s, s + 1):
            assert bool(emul.chain_emul_weak_hit(score, q, nn, max_mat)) == host_weak_hit(score, q, nn, max_mat), (score, thr)


@pytest.mark.parametrize("n_reads,qmax,W,record", [(2, 100, 0, 0), (50, 10000, 1, 1), (130, 777, 3, 0), (7, 33, 0, 1)])
def test_slot_layout_without_strand_unchanged(emul, n_reads, qmax, W, record):
    """A run without -s lays out its slot exactly as before; -s adds the strand bytes, the second CIGAR buffer and the
    second result behind it."""
    n_cap = qmax * 2 + 64
    assert emul.chain_emul_layout_check(n_cap, qmax, n_reads, 12, 4, 5, W, record) == 0
    assert emul.chain_emul_layout_check(n_cap, qmax, n_reads, 24, 26, 27, W, record) == 0
