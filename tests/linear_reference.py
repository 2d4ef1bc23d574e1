"""Reference results for banded linear-gap (-O 0) batches, recorded from the reference build (oracle/_ref) into
tests/golden/reference_runs_linear.json, in the format of tests/reference_runs.py; and the inputs the GPU tests share.

    ABPOA_RECORD_REFERENCE=tests/golden/reference_runs_linear.json python tests/linear_reference.py"""
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
from cases import LINEAR  # noqa: E402
from gfa_reference import list_files, reference_cli_md5  # noqa: E402
from qv_reference import fastq_files  # noqa: E402
from reference_runs import Reference  # noqa: E402
from score_window import with_last  # noqa: E402

STORE_LIN = HERE / "golden" / "reference_runs_linear.json"


def linear_reference() -> Reference:
    ref = Reference()
    ref.stored = json.loads(STORE_LIN.read_text()) if STORE_LIN.exists() else {}
    return ref


def lin_cfg(**kw) -> PoaConfig:
    return PoaConfig(**{**LINEAR, **kw})


# the shapes of test_linear_banded_lane_exact_sweep (3-25 % error, default and narrow bands), as batches
def sweep_groups(lo, hi):
    return [synth.make_group(5000 + s, 4 + s % 5, 150 + 37 * (s % 9), [0.03, 0.08, 0.15, 0.25][s % 4]) for s in range(lo, hi)]


# the two vector widths: e1 = 20 with a last read of 1637 bases keeps the reference on int16 (pn = 16), 1638 bases makes it
# pick int32 (pn = 8) -- the score-window points bits_linear_1637 / _1638, which the packed kernel's window admits
PN_CFG = dict(gap_open1=0, gap_ext1=20, gap_open2=0, gap_ext2=0)


def kind_input(kind, out_msa=False):
    out = dict(out_msa=out_msa)
    if kind == "sweep":
        return lin_cfg(**out), sweep_groups(0, 24)
    if kind == "sweep_narrow":
        return lin_cfg(wb=7, wf=0.01, **out), sweep_groups(24, 48)
    if kind == "sweep_wide":
        return lin_cfg(wb=12, wf=0.0, **out), sweep_groups(48, 60)
    if kind == "pn16_pn8":
        return PoaConfig(**PN_CFG, **out), [with_last(309, 3, 1000, 1637)(), with_last(309, 3, 1000, 1638)()]
    if kind == "aa":
        return lin_cfg(**{k: v for k, v in synth.WORKLOADS["aa_blosum62_2k"].cfg.__dict__.items()
                          if k not in LINEAR and k != "out_msa"}, **out), [synth.make_group(9800 + g, 8, 300, 0.08, m=27) for g in range(4)]
    if kind == "ragged":     # ragged sizes, a 2-read group, a 1-read group and an empty group (both stay off the DP)
        groups = [synth.make_group(9810 + g, n, 120 + 90 * g, 0.06) for g, n in enumerate([2, 9, 3, 14, 5])]
        return lin_cfg(**out), groups + [synth.make_group(9820, 1, 200, 0.05), []]
    if kind == "error_fan":  # 20-25 % error, 12-16 reads: rows of more than 4 predecessors (at most 16; the chunked
        # predecessor loop of more than 32 is covered cell by cell by tests/test_gpu_chain_linear_planes.py's deletion fan)
        return lin_cfg(**out), [synth.make_group(9840 + g, 12 + g, 250 + 40 * g, 0.20 + 0.01 * g) for g in range(5)]
    raise KeyError(kind)


KINDS = ["sweep", "sweep_narrow", "sweep_wide", "pn16_pn8", "aa", "ragged", "error_fan"]


# abpoa -l -O 0 -r 0..4 on a FASTA list (gfa_reference.list_files) and a FASTQ list (qv_reference.fastq_files)
CLI_LIST_OPTS = [["-O", "0", "-r", str(r)] for r in range(5)]


def record_all():
    ref = linear_reference()
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
