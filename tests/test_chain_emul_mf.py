"""CPU suite: the most-frequent-base consensus (-a 1).

The chain engine's vote (abpoa_b200/csrc/poa_chain.cuh: chain_mf_consensus) is compiled for the host and built read by
read next to the product's host graph layer, from the scalar oracle's alignments.  After the last read:
  - every aligned set is one column with pairwise distinct bases (what lets one thread per set vote it);
  - the device record (bases, coverage) and its path equal the host's most_frequent (poa_cons.c), node for node;
  - the -r 2 consensus row (chain_msa_rows) and the -r 4 GFA text (chain_gfa_record) equal the host writers';
  - the host's -r 2, -r 4 and -r 5 text equals the unmodified reference's (md5s in tests/golden/reference_runs_mf.json,
    see tests/mf_reference.py)."""
import ctypes as C
import subprocess
from pathlib import Path

import numpy as np
import pytest

from abpoa_b200 import synth
from abpoa_b200.aligner import PoaConfig, PoaSession
from abpoa_b200.capi import c_int_p, c_u8_p
from cases import AFFINE, CASES, case_reads
from gfa_reference import md5, with_file
from helpers import INPUTS, read_fasta
from mf_reference import mf_cfg, mf_reference, reference_group_md5, set_outputs, with_n
from oracle_binding import oracle_align
from test_chain_emul import CHAIN_CASES
from test_chain_emul_gfa import bind_product, record_text

HERE = Path(__file__).resolve().parent
ROOT = HERE.parent
SO = HERE / "emul" / "libchain_emul_mf.so"


@pytest.fixture(scope="module")
def reference():
    ref = mf_reference()
    yield ref
    ref.save()


@pytest.fixture(scope="module")
def emul():
    """tests/emul/chain_emul_mf.cpp (chain_emul.cpp + the -a 1 exports) compiled for the host."""
    srcs = [HERE / "emul" / "chain_emul_mf.cpp", HERE / "emul" / "chain_emul.cpp", ROOT / "abpoa_b200" / "csrc" / "poa_chain.cuh"]
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
    d.chain_emul_mf.restype = C.c_int
    d.chain_emul_mf.argtypes = [C.c_void_p, c_int_p, C.c_int]
    d.chain_emul_cons_path.restype = C.c_int
    d.chain_emul_cons_path.argtypes = [C.c_void_p, c_int_p, C.c_int]
    d.chain_emul_mf_check_columns.restype = C.c_int
    d.chain_emul_mf_check_columns.argtypes = [C.c_void_p]
    d.chain_emul_mf_msa.restype = C.c_int
    d.chain_emul_mf_msa.argtypes = [C.c_void_p, c_u8_p, C.c_int64]
    d.chain_emul_mf_gfa.restype = C.c_int64
    d.chain_emul_mf_gfa.argtypes = [C.c_void_p, c_int_p, C.c_int64]
    return d


def host_output(s, r: int) -> bytes:
    """abpoa_output of the host graph with the -r r outputs (what abpoa_msa prints for a group without names)."""
    set_outputs(s.lib, s.abpt, r)
    s.lib.abpoa_clean_msa_cons(s.ab)
    s.ab.contents.abg.contents.is_called_cons = 0
    return with_file(lambda fp: s.lib.abpoa_output(s.ab, s.abpt, fp))


def host_consensus(s):
    """(bases, coverage, node ids) of the host's -a 1 consensus."""
    set_outputs(s.lib, s.abpt, 0)
    s.generate()
    abc = s.ab.contents.abc.contents
    assert abc.n_cons == 1
    n = abc.cons_len[0]
    return (np.ctypeslib.as_array(abc.cons_base[0], shape=(n,)).copy(), np.ctypeslib.as_array(abc.cons_cov[0], shape=(n,)).copy(),
            np.ctypeslib.as_array(abc.cons_node_ids[0], shape=(n,)).copy() if n else np.zeros(0, dtype=np.int32))


def drive_mf(d, product_lib, reference, cfg: PoaConfig, reads, K=12):
    """Fuse `reads` with the emulated device code and the host graph layer side by side (alignments from the scalar
    oracle); after the last read compare the device's -a 1 consensus with the host's and the host's with the reference's."""
    pd = bind_product(product_lib)
    cfg = mf_cfg(cfg, out_msa=True)
    A = cfg.m - 1
    n = len(reads)
    W = (n + 63) // 64
    arrs = [np.ascontiguousarray(x, dtype=np.uint8) for x in reads]
    lens = (C.c_int * n)(*[len(x) for x in arrs])
    ptrs = (c_u8_p * n)(*[x.ctypes.data_as(c_u8_p) for x in arrs])
    n_cap = 2 + sum(len(x) for x in arrs)
    with PoaSession(cfg, product_lib) as s:
        a = s.abpt.contents
        ws = (C.c_int * n)(*[(-1 if a.wb < 0 else a.wb + int(np.float32(a.wf) * np.float32(len(x)))) for x in arrs])
        e = d.chain_emul_new(n, lens, ptrs, ws, n_cap, K, A, a.m, a.max_mat, a.min_mis, a.gap_open1, a.gap_ext1,
                             a.gap_open1 + a.gap_ext1, a.gap_open2 + a.gap_ext2, W)
        try:
            s.reset(max(len(x) for x in arrs))
            s.lib.dll.poa_graph_set_fast_order(s.ab.contents.abg, 1)
            for i, x in enumerate(arrs):
                al, res = oracle_align(s, x)
                if i == 0:
                    s.add(x, res, n)
                    d.chain_emul_seed(e)
                else:
                    g = s.ab.contents.abg.contents
                    row_of = np.ctypeslib.as_array(g.node_id_to_index, shape=(g.node_n,)).copy()
                    cig = al.cigar[::-1].copy()                  # backtrack order, DP rows instead of node ids
                    is_ins = (cig & np.uint64(0xf)) == np.uint64(1)
                    rows = row_of[(cig >> np.uint64(34)).astype(np.int64) % len(row_of)].astype(np.uint64)
                    dev = np.ascontiguousarray(np.where(is_ins, cig, (rows << np.uint64(34)) | (cig & np.uint64(0x3ffffffff))), dtype=np.uint64)
                    s.add(x, res, n)
                    failed = d.chain_emul_fuse(e, dev.ctypes.data_as(C.POINTER(C.c_uint64)), len(dev), al.best_score, al.cells)
                    assert failed == 0, f"read {i}: device chain gave up with flags {failed:#x}"
            s.lib.dll.poa_graph_set_fast_order(s.ab.contents.abg, 0)
            nn = s.ab.contents.abg.contents.node_n
            assert d.chain_emul_n_nodes(e) == nn

            # ---- the record and its path ----
            want_b, want_c, want_ids = host_consensus(s)
            out = np.full(nn + 8, -0x33333334, dtype=np.int32)
            ln = d.chain_emul_mf(e, out.ctypes.data_as(c_int_p), nn)
            assert (bad := d.chain_emul_mf_check_columns(e)) == 0, f"node {bad}: an aligned set is not one column of distinct bases"
            assert ln == len(want_b), f"consensus length {ln}, host {len(want_b)}"
            assert (out[1 + ln:] == -0x33333334).all(), "record written past its length"
            assert np.array_equal(out[1:1 + ln] & 0xff, want_b), "consensus bases differ from the host's"
            assert np.array_equal(out[1:1 + ln] >> 8, want_c), "consensus coverage differs from the host's"
            ids = np.zeros(nn, dtype=np.int32)
            assert d.chain_emul_cons_path(e, ids.ctypes.data_as(c_int_p), nn) == ln
            assert np.array_equal(ids[:ln], want_ids), "consensus path differs from the host's node ids"

            # ---- -r 2: the consensus row ----
            set_outputs(s.lib, s.abpt, 2)
            s.generate()
            want_rows = s.msa_rows()
            buf = np.full((n + 1) * nn, 0xee, dtype=np.uint8)
            msa_len = d.chain_emul_mf_msa(e, buf.ctypes.data_as(c_u8_p), len(buf))
            assert msa_len == len(want_rows[0]) and len(want_rows) == n + 1
            for k, w in enumerate(want_rows):
                row = buf[k * msa_len: (k + 1) * msa_len]
                assert np.array_equal(row, w), f"MSA row {k} differs at column {int(np.argmax(row != w))}"

            # ---- -r 4: the GFA text, consensus path included ----
            cap = 8 + 4 * nn + 2 * nn * W + sum(len(x) + 1 for x in arrs)
            rec = np.full(cap + 64, -0x33333334, dtype=np.int32)
            words = d.chain_emul_mf_gfa(e, rec.ctypes.data_as(c_int_p), cap)
            assert words > 0, f"no GFA record ({words})"
            got_gfa = record_text(pd, rec, s)
            want_gfa = host_output(s, 4)
            assert got_gfa == want_gfa, f"GFA text differs from abpoa_generate_gfa at byte " \
                                        f"{next((k for k, (x, y) in enumerate(zip(got_gfa, want_gfa)) if x != y), min(len(got_gfa), len(want_gfa)))}"

            # ---- the host against the reference ----
            for r in (2, 4, 5):
                assert md5(host_output(s, r)) == reference_group_md5(reference, cfg, reads, r), f"-a 1 -r {r}: host output differs from the reference's"
        finally:
            d.chain_emul_free(e)


@pytest.mark.parametrize("name", CHAIN_CASES)
def test_device_mf_matches_host(emul, product_lib, reference, name):
    case = CASES[name]
    cfg = PoaConfig(**case["cfg"])
    drive_mf(emul, product_lib, reference, cfg, case_reads(case), K=32 if cfg.m > 5 else 12)


@pytest.mark.parametrize("gap", ["convex", "affine"])
def test_device_mf_3alleles(emul, product_lib, reference, gap):
    """3alleles.fa: 126 reads, three alleles."""
    drive_mf(emul, product_lib, reference, PoaConfig(**({} if gap == "convex" else AFFINE)), read_fasta(INPUTS / "3alleles.fa"))


@pytest.mark.parametrize("n_reads", [63, 64, 65, 128])
def test_device_mf_word_edges(emul, product_lib, reference, n_reads):
    drive_mf(emul, product_lib, reference, PoaConfig(), synth.make_group(7300 + n_reads, n_reads, 120, 0.08))


@pytest.mark.parametrize("frac", [0.02, 0.3])
def test_device_mf_reads_with_n(emul, product_lib, reference, frac):
    """Code 4 (N) never wins a column and counts as gap; at 30 % N whole columns are dropped."""
    drive_mf(emul, product_lib, reference, PoaConfig(), with_n(synth.make_group(7400, 9, 200, 0.06), 7401, 4, frac))


def test_device_mf_amino_acids_with_last_code(emul, product_lib, reference):
    """-c: code 26 is the last code, so it never wins."""
    cfg = PoaConfig(**synth.WORKLOADS["aa_blosum62_2k"].cfg.__dict__)
    drive_mf(emul, product_lib, reference, cfg, with_n(synth.make_group(7500, 8, 200, 0.10, m=27), 7501, 26, 0.05), K=32)


@pytest.mark.parametrize("seed", range(3))
def test_device_mf_two_reads(emul, product_lib, reference, seed):
    """Two reads: every mismatch column is a base/base tie (the lower code wins), every indel a base/gap tie (kept)."""
    drive_mf(emul, product_lib, reference, PoaConfig(), synth.make_group(7600 + seed, 2, 150, 0.15))


@pytest.mark.parametrize("n_reads", [4, 9])
def test_device_mf_high_error(emul, product_lib, reference, n_reads):
    """25 % error: many columns where the best base and the gaps are close or equal."""
    drive_mf(emul, product_lib, reference, PoaConfig(), synth.make_group(7700 + n_reads, n_reads, 200, 0.25))
