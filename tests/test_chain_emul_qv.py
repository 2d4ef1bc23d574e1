"""CPU suite: quality weights (-Q) on the chain engine's graph code.

The device-side graph code (abpoa_b200/csrc/poa_chain.cuh) is compiled for the host and driven read by read next to the
product's host graph layer, with every alignment from the scalar oracle.  The host graph gets each read's weights (on
the read's strand, reversed for a reverse-complemented read under -s); the device code reads them from the slot's weight
bytes (chain_read_weight).  After every read the edge lists with their weights and order, the spliced order, n_read and
the next job blob must agree; after the last read the device's consensus and coverage must be the host's, and the
device's -r 0 / -r 2 / -r 4 text must be the reference's (md5s in tests/golden/reference_runs_qv.json, see
tests/qv_reference.py)."""
import ctypes as C
import subprocess
from pathlib import Path

import numpy as np
import pytest

from abpoa_b200 import capi, synth
from abpoa_b200.aligner import PoaConfig, PoaSession
from abpoa_b200.batch import fnv1a_words
from abpoa_b200.capi import c_int_p, c_u8_p
from cases import AFFINE, CASES, case_reads, case_weights
from gfa_reference import md5, with_file
from helpers import INPUTS, read_fasta
from mf_reference import set_outputs
from oracle_binding import oracle_align
from qv_reference import qv_cfg, qv_reference, quality_weights, reference_group, reference_group_md5, unit_filled
from strand_reference import revcomp, strand_mix
from test_chain_emul_gfa import bind_product
from test_chain_emul_strand import arr, compare_graphs, device_cigar, device_text, host_weak_hit

HERE = Path(__file__).resolve().parent
ROOT = HERE.parent
SO = HERE / "emul" / "libchain_emul_qv.so"


@pytest.fixture(scope="module")
def reference():
    ref = qv_reference()
    yield ref
    ref.save()


@pytest.fixture(scope="module")
def emul():
    """tests/emul/chain_emul_qv.cpp (chain_emul_strand.cpp + the -Q exports) compiled for the host."""
    srcs = [HERE / "emul" / "chain_emul_qv.cpp", HERE / "emul" / "chain_emul_strand.cpp", HERE / "emul" / "chain_emul.cpp",
            ROOT / "abpoa_b200" / "csrc" / "poa_chain.cuh"]
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
    d.chain_emul_set_read_qw.argtypes = [C.c_void_p, c_u8_p]
    d.chain_emul_msa.restype = C.c_int
    d.chain_emul_msa.argtypes = [C.c_void_p, C.c_int, c_u8_p, C.c_int64]
    d.chain_emul_gfa.restype = C.c_int64
    d.chain_emul_gfa.argtypes = [C.c_void_p, C.c_int, c_int_p, C.c_int64]
    d.chain_emul_reads_layout_check.restype = C.c_int
    d.chain_emul_reads_layout_check.argtypes = [C.c_int, C.c_int64]
    d.chain_emul_layout_check.restype = C.c_int
    d.chain_emul_layout_check.argtypes = [C.c_int] * 8
    return d


def set_strands(s, n, is_rc):
    """The reads' strands on the host handle, reads unnamed (as abpoa_msa prints them without names)."""
    abs_ = s.ab.contents.abs.contents
    abs_.n_seq = n
    for i in range(n):
        abs_.name[i].l = 0
        abs_.is_rc[i] = int(is_rc[i])


def consensus_text(d, pd, e, s, n, nn) -> bytes:
    """-r 0: the device's consensus record installed as the engine installs it, printed by the product's writer."""
    set_outputs(s.lib, s.abpt, 0)
    s.lib.abpoa_clean_msa_cons(s.ab)
    out = np.zeros(nn + 1, dtype=np.int32)
    ln = d.chain_emul_consensus(e, out.ctypes.data_as(c_int_p), nn)
    base = np.ascontiguousarray(out[1:1 + ln] & 0xff, dtype=np.uint8)
    cov = np.ascontiguousarray(out[1:1 + ln] >> 8, dtype=np.int32)
    pd.poa_cons_install.argtypes = [C.c_void_p, C.c_int, C.c_int, c_u8_p, c_int_p]
    pd.poa_cons_install(C.cast(s.ab, C.c_void_p), n, ln, base.ctypes.data_as(c_u8_p), cov.ctypes.data_as(c_int_p))
    return with_file(lambda fp: s.lib.abpoa_output(s.ab, s.abpt, fp))


def drive_qv(d, product_lib, reference, cfg: PoaConfig, reads, weights, K=12):
    """Fuse `reads` with their `weights` (per read an int array 0..255, or None) with the emulated device code and the host
    graph layer side by side; with cfg.amb_strand each read on the strand the alignment warp would pick.  Returns the
    strand bytes."""
    pd = bind_product(product_lib)
    A = cfg.m - 1
    n = len(reads)
    W = (n + 63) // 64
    arrs = [np.ascontiguousarray(x, dtype=np.uint8) for x in reads]
    full = unit_filled(arrs, weights)
    lens = (C.c_int * n)(*[len(x) for x in arrs])
    ptrs = (c_u8_p * n)(*[x.ctypes.data_as(c_u8_p) for x in arrs])
    n_cap = 2 + sum(len(x) for x in arrs)
    read_rc = np.full(n, 0xcd, dtype=np.uint8)
    read_qw = np.ascontiguousarray(np.concatenate(full).astype(np.uint8))      # at the reads' offsets, forward strand
    hcfg = PoaConfig(**{**cfg.__dict__, "out_msa": True})       # read ids on the host side
    with PoaSession(hcfg, product_lib) as s:
        a = s.abpt.contents
        ws = (C.c_int * n)(*[(-1 if a.wb < 0 else a.wb + int(np.float32(a.wf) * np.float32(len(x)))) for x in arrs])
        e = d.chain_emul_new(n, lens, ptrs, ws, n_cap, K, A, a.m, a.max_mat, a.min_mis, a.gap_open1, a.gap_ext1,
                             a.gap_open1 + a.gap_ext1, a.gap_open2 + a.gap_ext2, W)
        if cfg.amb_strand:
            d.chain_emul_set_read_rc(e, read_rc.ctypes.data_as(c_u8_p))
        d.chain_emul_set_read_qw(e, read_qw.ctypes.data_as(c_u8_p))
        try:
            s.reset(max(len(x) for x in arrs))
            s.lib.dll.poa_graph_set_fast_order(s.ab.contents.abg, 1)
            s.lib.dll.poa_debug_blob.restype = C.c_int
            s.lib.dll.poa_debug_blob.argtypes = [C.c_void_p, C.c_void_p, c_u8_p, C.c_int, c_u8_p, C.c_int]
            blob_buf = np.zeros(64 + 16 * n_cap * 6 + max(len(x) for x in arrs) + 256, dtype=np.uint8)
            tot_cells = 0
            for i, x in enumerate(arrs):
                w = weights[i]
                if i == 0:
                    _, res = oracle_align(s, x)
                    s.add(x, res, n, w)
                    d.chain_emul_seed(e)
                else:
                    node_n = s.ab.contents.abg.contents.node_n
                    al, res = oracle_align(s, x)
                    seq, flag, cells = x, 0, al.cells
                    if cfg.amb_strand and d.chain_emul_weak_hit(al.best_score, len(x), node_n, a.max_mat):
                        assert host_weak_hit(al.best_score, len(x), node_n, a.max_mat)
                        y = revcomp(x)
                        al2, res2 = oracle_align(s, y)
                        cells += al2.cells
                        if al2.best_score > al.best_score:
                            if res.n_cigar > 0:
                                capi.libc_free(res.graph_cigar)
                            seq, al, res, flag = y, al2, res2, 3
                            w = None if w is None else np.ascontiguousarray(np.asarray(w)[::-1])     # weights flip with the read
                        else:
                            if res2.n_cigar > 0:
                                capi.libc_free(res2.graph_cigar)
                            flag = 2
                    dev = device_cigar(s, al)
                    read_rc[i] = flag
                    tot_cells += cells
                    s.add(seq, res, n, w)
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

            # ---- consensus and coverage: the device's record against the host's heaviest bundling on the same graph ----
            out = np.zeros(g.node_n + 1, dtype=np.int32)
            ln = d.chain_emul_consensus(e, out.ctypes.data_as(c_int_p), g.node_n)
            set_outputs(s.lib, s.abpt, 0)
            s.lib.abpoa_clean_msa_cons(s.ab)
            g.is_called_cons = 0
            s.lib.abpoa_generate_consensus(s.ab, s.abpt)
            assert ln == len(s.consensus()[0]), "consensus length"
            assert np.array_equal(out[1:1 + ln] & 0xff, s.consensus()[0]), "consensus bases"
            assert np.array_equal(out[1:1 + ln] >> 8, s.consensus_cov()[0]), "coverage (n_read, not weights)"

            # ---- the device's -r 0 / -r 2 / -r 4 text, printed with the device's strands, is the reference's ----
            is_rc = [int(f & 1) for f in read_rc] if cfg.amb_strand else [0] * n
            if cfg.amb_strand:
                assert is_rc == reference_group(reference, cfg, reads, weights)["is_rc"], "strands differ from the reference's abpoa_msa"
            set_strands(s, n, is_rc)
            assert md5(consensus_text(d, pd, e, s, n, g.node_n)) == reference_group_md5(reference, cfg, reads, weights, 0), "-r 0"
            for r in (2, 4):
                got = device_text(d, pd, e, s, n, g.node_n, W, sum(len(x) for x in arrs), r)
                assert md5(got) == reference_group_md5(reference, cfg, reads, weights, r), f"-Q -r {r}: device output differs from the reference's"
            return read_rc.copy()
        finally:
            d.chain_emul_free(e)


def test_syn_qv_weights(emul, product_lib, reference):
    c = CASES["syn_qv_weights"]
    reads = case_reads(c)
    drive_qv(emul, product_lib, reference, qv_cfg(), reads, case_weights(c, reads))


def test_heter_fq(emul, product_lib, reference):
    """The reference's FASTQ input with its own qualities (weight = quality character - 32)."""
    path = INPUTS / "heter.fq"
    reads = read_fasta(path)
    lines = path.read_text().splitlines()
    weights = [np.frombuffer(lines[i + 3].encode(), dtype=np.uint8).astype(np.int32) - 32 for i in range(0, len(lines) - 3, 4)]
    assert [len(w) for w in weights] == [len(r) for r in reads]
    drive_qv(emul, product_lib, reference, qv_cfg(), reads, weights)


@pytest.mark.parametrize("seed", [0, 1])
def test_weights_0_and_255(emul, product_lib, reference, seed):
    """The ends of a weight byte: zero-weight edges (kept, ordered last) and 255s that add up past a byte."""
    reads = synth.make_group(9700 + seed, 9, 400, 0.08)
    weights = quality_weights(9710 + seed, reads)
    rng = np.random.default_rng(9720 + seed)
    for w in weights:
        u = rng.random(len(w))
        w[u < 0.25] = 0
        w[u > 0.75] = 255
    drive_qv(emul, product_lib, reference, qv_cfg(), reads, weights)


def test_reads_without_weights(emul, product_lib, reference):
    """A read without weights (NULL) weighs 1 per base, next to reads that have them."""
    reads = synth.make_group(9730, 8, 500, 0.06)
    weights = [None if i % 3 == 1 else w for i, w in enumerate(quality_weights(9731, reads))]
    drive_qv(emul, product_lib, reference, qv_cfg(), reads, weights)


@pytest.mark.parametrize("gap", ["convex", "affine"])
def test_strand_flipped_reads(emul, product_lib, reference, gap):
    """-s: a reverse-complemented read's weights are reversed with it."""
    cfg = qv_cfg(PoaConfig(**({} if gap == "convex" else AFFINE)), amb_strand=True)
    reads = strand_mix(9740 + (gap == "affine"), 10, 350)
    flags = drive_qv(emul, product_lib, reference, cfg, reads, quality_weights(9745, reads))
    assert [int(f & 1) for f in flags[1:]] == [int(i % 3 == 1) for i in range(1, len(reads))]


def test_amino_acids(emul, product_lib, reference):
    cfg = qv_cfg(PoaConfig(**synth.WORKLOADS["aa_blosum62_2k"].cfg.__dict__))
    reads = synth.make_group(9750, 7, 300, 0.08, m=27)
    drive_qv(emul, product_lib, reference, cfg, reads, quality_weights(9751, reads), K=32)


def test_weights_change_the_graph(emul, product_lib, reference):
    """The inputs above test something: with weights the consensus text differs from the unit-weight run's."""
    c = CASES["syn_qv_weights"]
    reads = case_reads(c)
    weights = case_weights(c, reads)
    for w in weights:
        w[: len(w) // 2] = 1
        w[len(w) // 2:] = 40 * (np.arange(len(w) - len(w) // 2) % 2)
    with_w = reference_group_md5(reference, qv_cfg(), reads, weights, 4)
    unit = reference_group_md5(reference, qv_cfg(), reads, [None] * len(reads), 4)
    assert with_w != unit
    drive_qv(emul, product_lib, reference, qv_cfg(), reads, weights)


@pytest.mark.parametrize("n_reads,bases", [(2, 100), (50, 500_000), (130, 777), (7, 33)])
def test_reads_layout_without_weights_unchanged(emul, n_reads, bases):
    """A run without -Q weights lays out its reads exactly as before; -Q adds one byte per base behind them.  The group's
    own region does not change either way."""
    assert emul.chain_emul_reads_layout_check(n_reads, bases) == 0
    assert emul.chain_emul_layout_check(2 * bases // n_reads + 64, bases // n_reads, n_reads, 12, 4, 5, 1, 1) == 0
