"""GPU: the pyabpoa-compatible surface (abpoa_b200.aligner.msa_aligner mirrors python/pyabpoa.pyx:93-371) must give
what the reference library gives for the same calls -- the very same driver was run over the reference library
(lib=...), and every field of msa_result is compared with what it returned there (stored by tests/reference_runs.py)."""
import numpy as np
import pytest

from abpoa_b200 import synth
from abpoa_b200.aligner import decode, msa_aligner
from reference_runs import Hasher

pytestmark = pytest.mark.gpu

EXAMPLE = [   # python/example.py, second example
    "CGTCAATCTATCGAAGCATACGCGGGCAGAGCCGAAGACCTCGGCAATCCA",
    "CCACGTCAATCTATCGAAGCATACGCGGCAGCCGAACTCGACCTCGGCAATCAC",
    "CGTCAATCTATCGAAGCATACGCGGCAGAGCCCGGAAGACCTCGGCAATCAC",
    "CGTCAATGCTAGTCGAAGCAGCTGCGGCAGAGCCGAAGACCTCGGCAATCAC",
    "CGTCAATCTATCGAAGCATTCTACGCGGCAGAGCCGACCTCGGCAATCAC",
    "CGTCAATCTAGAAGCATACGCGGCAAGAGCCGAAGACCTCGGCCAATCAC",
    "CGTCAATCTATCGGTAAAGCATACGCTCTGTAGCCGAAGACCTCGGCAATCAC",
    "CGTCAATCTATCTTCAAGCATACGCGGCAGAGCCGAAGACCTCGGCAATC",
    "CGTCAATGGATCGAGTACGCGGCAGAGCCGAAGACCTCGGCAATCAC",
    "CGTCAATCTAATCGAAGCATACGCGGCAGAGCCGTCTACCTCGGCAATCACGT",
]


FIELDS = ("n_seq", "n_cons", "clu_n_seq", "clu_read_ids", "cons_len", "cons_seq", "cons_cov", "cons_qv", "msa_len", "msa_seq")


def digest(res):
    """A hash of every field of an msa_result."""
    return {f: Hasher().add(getattr(res, f)).hex() for f in FIELDS}


def same(a, want):
    got = digest(a)
    for f in FIELDS:
        assert got[f] == want[f], f


@pytest.mark.parametrize("mode", ["g", "l", "e"])
def test_msa_example(product_lib, reference, mode):
    a = msa_aligner(aln_mode=mode, lib=product_lib).msa(EXAMPLE, out_cons=True, out_msa=True)
    b = reference.value("pyabpoa_msa", (mode, EXAMPLE), lambda: digest(msa_aligner(aln_mode=mode, lib=reference.lib).msa(EXAMPLE, out_cons=True, out_msa=True)))
    same(a, b)
    if mode == "g":
        assert a.cons_seq[0] == "CGTCAATCTATCGAAGCATACGCGGCAGAGCCGAAGACCTCGGCAATCAC"     # SURVEY 8c
        assert a.msa_len == 75


def test_msa_consensus_only_and_qscores(product_lib, reference):
    reads = [decode(r) for r in synth.make_group(6100, 8, 400, 0.06)]
    rng = np.random.default_rng(3)
    qs = [rng.integers(1, 41, size=len(r)).tolist() for r in reads]
    for kw in (dict(), dict(qscores=qs)):
        a = msa_aligner(lib=product_lib).msa(reads, out_cons=True, out_msa=False, **kw)
        b = reference.value("pyabpoa_cons", (reads, kw), lambda: digest(msa_aligner(lib=reference.lib).msa(reads, out_cons=True, out_msa=False, **kw)))
        same(a, b)


def test_incremental_msa_align_add_output(product_lib, reference):
    reads = [decode(r) for r in synth.make_group(6200, 9, 300, 0.05)]

    def run(lib):
        al = msa_aligner(match=3, mismatch=5, gap_open1=5, gap_open2=30, lib=lib)
        al.msa_align(reads[:4], out_cons=True, out_msa=True)
        first = al.msa_output()
        al.msa_add(reads[4:7]).msa_add(reads[7:])
        return first, al.msa_output()
    a = run(product_lib)
    b = reference.value("pyabpoa_incremental", reads, lambda: [digest(x) for x in run(reference.lib)])
    same(a[0], b[0])
    same(a[1], b[1])


def test_amino_acid_score_matrix(product_lib, reference):
    from abpoa_b200.capi import REPO_ROOT
    mtx = str(REPO_ROOT / "abpoa_b200" / "data" / "BLOSUM62.mtx")
    reads = [decode(r, 27) for r in synth.make_group(6300, 6, 250, 0.10, m=27)]
    a = msa_aligner(is_aa=True, score_matrix=mtx, gap_open2=0, gap_ext2=0, lib=product_lib).msa(reads, True, True)
    b = reference.value("pyabpoa_aa", reads, lambda: digest(msa_aligner(is_aa=True, score_matrix=mtx, gap_open2=0, gap_ext2=0, lib=reference.lib).msa(reads, True, True)))
    same(a, b)
