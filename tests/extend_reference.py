"""Reference results for extend-mode (-m 2, with and without z-drop -z) batches, recorded from the reference build
(oracle/_ref) into tests/golden/reference_runs_extend.json, in the format of tests/reference_runs.py; and the inputs the GPU
tests share.

    ABPOA_RECORD_REFERENCE=tests/golden/reference_runs_extend.json python tests/extend_reference.py"""
from __future__ import annotations

import json
import sys
import tempfile
from pathlib import Path

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parent))
sys.path.insert(0, str(HERE))

from abpoa_b200 import synth  # noqa: E402
from abpoa_b200.aligner import PoaConfig  # noqa: E402
from abpoa_b200.capi import ABPOA_EXTEND_MODE  # noqa: E402
from cases import AFFINE  # noqa: E402
from gfa_reference import list_files, reference_cli_md5  # noqa: E402
from qv_reference import fastq_files  # noqa: E402
from reference_runs import Reference  # noqa: E402

STORE_EXT = HERE / "golden" / "reference_runs_extend.json"


def extend_reference() -> Reference:
    ref = Reference()
    ref.stored = json.loads(STORE_EXT.read_text()) if STORE_EXT.exists() else {}
    return ref


def ext_cfg(**kw) -> PoaConfig:
    return PoaConfig(**{"align_mode": ABPOA_EXTEND_MODE, **kw})


def sweep_groups(lo, hi):
    """3-25 % error, 4-8 reads of 150-450 bases"""
    return [synth.make_group(6000 + s, 4 + s % 5, 150 + 37 * (s % 9), [0.03, 0.08, 0.15, 0.25][s % 4]) for s in range(lo, hi)]


def kind_input(kind, out_msa=False):
    out = dict(out_msa=out_msa)
    if kind == "convex":
        return ext_cfg(**out), sweep_groups(0, 16)
    if kind == "affine":
        return ext_cfg(**AFFINE, **out), sweep_groups(16, 32)
    if kind == "convex_zdrop":
        return ext_cfg(zdrop=100, **out), sweep_groups(32, 48)
    if kind == "zdrop_fires":      # a small z-drop at 15-25 % error: alignments stop early and leave long tails inserted
        return ext_cfg(zdrop=10, **out), [synth.make_group(6100 + g, 8, 400 + 50 * g, 0.15 + 0.02 * g) for g in range(6)]
    if kind == "affine_zdrop_error_fan":   # 20-25 % error, 12-16 reads: in-degree >= 2, full aligned sets
        return ext_cfg(zdrop=40, **AFFINE, **out), [synth.make_group(6200 + g, 12 + g, 250 + 40 * g, 0.20 + 0.01 * g) for g in range(5)]
    if kind == "aa":
        aa = synth.WORKLOADS["aa_blosum62_2k"].cfg
        return ext_cfg(m=27, score_matrix=aa.score_matrix, **AFFINE, **out), [synth.make_group(6300 + g, 8, 300, 0.10 + 0.04 * g, m=27) for g in range(4)]
    if kind == "ragged":     # ragged sizes, a 2-read group, a 1-read group and an empty group (both stay off the DP)
        groups = [synth.make_group(6400 + g, n, 120 + 90 * g, 0.06) for g, n in enumerate([2, 9, 3, 14, 5])]
        return ext_cfg(zdrop=50, **out), groups + [synth.make_group(6410, 1, 200, 0.05), []]
    raise KeyError(kind)


KINDS = ["convex", "affine", "convex_zdrop", "zdrop_fires", "affine_zdrop_error_fan", "aa", "ragged"]

# abpoa -l -m 2 [-z N] -r 0..4 on a FASTA list (gfa_reference.list_files) and a FASTQ list (qv_reference.fastq_files)
CLI_LIST_OPTS = [["-m", "2", *z, "-r", str(r)] for z in ([], ["-z", "100"]) for r in range(5)]


def record_all():
    ref = extend_reference()
    assert ref.record_to, "set ABPOA_RECORD_REFERENCE to the store to record into"
    for kind in KINDS:
        cfg, groups = kind_input(kind, out_msa=True)
        ref.batch(cfg, groups, want_msa=True)
    with tempfile.TemporaryDirectory() as d:
        for files in (list_files(Path(d)), fastq_files(Path(d))):
            for opts in CLI_LIST_OPTS:
                reference_cli_md5(ref, [*opts, "-l"], files)
    ref.save()


if __name__ == "__main__":
    record_all()
