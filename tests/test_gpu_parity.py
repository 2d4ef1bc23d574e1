"""GPU parity: the CUDA path (through the abpoa.h C ABI of libabpoa_b200.so) against the
unmodified reference (AVX2 build) on the same inputs, as stored by tests/reference_runs.py.

Bar: bit-exact -- per-read best_score, every 64-bit graph-CIGAR word, alignment end
points, the number of DP cells, and the final consensus / coverage / RC-MSA.
"""
import numpy as np
import pytest

from abpoa_b200 import synth
from abpoa_b200.aligner import PoaConfig
from abpoa_b200.capi import ABPOA_EXTEND_MODE, ABPOA_LOCAL_MODE
from helpers import INPUTS, read_fasta, run_group
from reference_runs import assert_run_matches

pytestmark = pytest.mark.gpu

AFFINE = dict(gap_open1=4, gap_ext1=2, gap_open2=0, gap_ext2=0)
LINEAR = dict(gap_open1=0, gap_ext1=2, gap_open2=0, gap_ext2=0)


@pytest.mark.parametrize("fname", ["seq.fa", "test.fa", "heter.fa", "3alleles.fa"])
@pytest.mark.parametrize("gap", ["convex", "affine"])
def test_reference_fixtures(product_lib, reference, fname, gap):
    """The reference's own test inputs (test_data/, config 1 of BASELINE.json)."""
    cfg = PoaConfig(**(AFFINE if gap == "affine" else {}))
    reads = read_fasta(INPUTS / fname)
    assert_run_matches(run_group(product_lib, cfg, reads), reference.run(cfg, reads), f"{fname}/{gap}")


@pytest.mark.parametrize("seed", [11, 12, 13])
def test_affine_1k(product_lib, reference, seed):
    w = synth.WORKLOADS["affine_1k"]
    reads = synth.make_group(seed, 20, 1000, 0.05)
    assert_run_matches(run_group(product_lib, w.cfg, reads), reference.run(w.cfg, reads), f"affine_1k/{seed}")


@pytest.mark.parametrize("seed,length,n", [(21, 2000, 12), (22, 3000, 8)])
def test_convex(product_lib, reference, seed, length, n):
    w = synth.WORKLOADS["convex_10k"]
    reads = synth.make_group(seed, n, length, 0.05)
    assert_run_matches(run_group(product_lib, w.cfg, reads), reference.run(w.cfg, reads), f"convex/{seed}")


def test_convex_int32_switch(product_lib, reference):
    """match=20 forces the reference (and us) onto 32-bit scores."""
    cfg = PoaConfig(match=20, mismatch=40, gap_open1=40, gap_ext1=20, gap_open2=240, gap_ext2=10)
    reads = synth.make_group(31, 8, 2000, 0.05)
    assert_run_matches(run_group(product_lib, cfg, reads), reference.run(cfg, reads), "convex/int32")


@pytest.mark.parametrize("gap", ["linear", "affine", "convex"])
def test_local(product_lib, reference, gap):
    kw = LINEAR if gap == "linear" else (AFFINE if gap == "affine" else {})
    cfg = PoaConfig(align_mode=ABPOA_LOCAL_MODE, **kw)
    reads = synth.make_group(41, 8, 700, 0.05)
    assert_run_matches(run_group(product_lib, cfg, reads), reference.run(cfg, reads), f"local/{gap}")


@pytest.mark.parametrize("gap", ["affine", "convex"])
def test_extend(product_lib, reference, gap):
    cfg = PoaConfig(align_mode=ABPOA_EXTEND_MODE, **(AFFINE if gap == "affine" else {}))
    reads = synth.make_group(51, 8, 900, 0.05)
    assert_run_matches(run_group(product_lib, cfg, reads), reference.run(cfg, reads), f"extend/{gap}")


def test_amino_acid_blosum62(product_lib, reference):
    w = synth.WORKLOADS["aa_blosum62_2k"]
    reads = synth.make_group(61, 10, 1200, 0.10, m=27)
    assert_run_matches(run_group(product_lib, w.cfg, reads), reference.run(w.cfg, reads), "aa/blosum62")


def test_unbanded_global(product_lib, reference):
    cfg = PoaConfig(wb=-1, **AFFINE)
    reads = synth.make_group(71, 6, 500, 0.08)
    assert_run_matches(run_group(product_lib, cfg, reads), reference.run(cfg, reads), "unbanded")
