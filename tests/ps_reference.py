"""What the unmodified reference computes with path scores (-G, inc_path_score: every in-edge adds
max(round(ln(edge_w / node_w)), -20) to the DP terms it feeds, reference src/abpoa_graph.c:429-437), stored in
tests/golden/reference_runs_ps.json and keyed as in tests/reference_runs.py, plus the inputs the -G tests share.

Recording: with oracle/_ref/ built (oracle/Makefile),

    ABPOA_RECORD_REFERENCE=tests/golden/reference_runs_ps.json python tests/ps_reference.py

runs the reference library and the reference CLI on every input of tests/test_gpu_ps.py; the CPU file
tests/test_chain_emul_ps.py records its own while it runs under the same variable."""
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
from abpoa_b200.capi import ABPOA_MF  # noqa: E402
from cases import AFFINE  # noqa: E402
from gfa_reference import reference_cli_md5  # noqa: E402
from qv_reference import fastq_files, kind_groups as qv_kind_groups, quality_weights, reference_group, unit_filled  # noqa: E402
from reference_runs import Reference  # noqa: E402
from strand_reference import strand_mix  # noqa: E402

STORE_PS = HERE / "golden" / "reference_runs_ps.json"


def ps_reference() -> Reference:
    ref = Reference()
    ref.stored = json.loads(STORE_PS.read_text()) if STORE_PS.exists() else {}
    return ref


def ps_cfg(cfg: PoaConfig | None = None, **kw) -> PoaConfig:
    return PoaConfig(**{**(cfg or PoaConfig()).__dict__, **kw, "inc_path_score": True})


# ---- inputs shared by the GPU tests and the recording run ----
KINDS = ("convex", "affine", "aa", "mf", "qv", "qv_extreme", "strand", "strand_qv", "fan")


def kind_cfg(kind, out_msa=True):
    """-G alone on convex / affine / amino acids (-c) / -a 1 / -s, with -Q weights, and on high-error groups whose rows
    have many predecessors."""
    out = dict(out_msa=out_msa)
    if kind == "aa":
        return ps_cfg(PoaConfig(**synth.WORKLOADS["aa_blosum62_2k"].cfg.__dict__), **out)
    if kind == "mf":
        return ps_cfg(cons_algrm=ABPOA_MF, **out)
    if kind in ("strand", "strand_qv"):
        return ps_cfg(amb_strand=True, use_qv=kind == "strand_qv", **out)
    if kind == "affine":
        return ps_cfg(PoaConfig(**AFFINE), **out)
    return ps_cfg(use_qv=kind.startswith("qv"), **out)


def kind_groups(kind):
    """(groups, weights): weights None for the kinds without -Q, else per group and read int32 weights."""
    if kind == "qv":
        return qv_kind_groups("convex")
    if kind == "qv_extreme":
        return qv_kind_groups("extreme")
    if kind == "aa":
        return [synth.make_group(9900 + g, 8, 300, 0.08, m=27) for g in range(4)], None
    if kind in ("strand", "strand_qv"):
        groups = [strand_mix(9920 + g, 5 + g % 4, 300 + 60 * (g % 4)) for g in range(6)]
        return groups, ([quality_weights(9930 + gi, g) for gi, g in enumerate(groups)] if kind == "strand_qv" else None)
    if kind == "fan":           # 20-25 % error, 12-16 reads: many rows with more than 4 predecessors
        return [synth.make_group(9940 + g, 12 + g, 250 + 40 * g, 0.20 + 0.01 * g) for g in range(5)], None
    seed = {"convex": 9950, "affine": 9970, "mf": 9990}[kind]
    return [synth.make_group(seed + g, 6 + g % 5, 300 + 50 * (g % 6), 0.04 + 0.01 * (g % 5)) for g in range(8)], None


def group_weights(groups, weights):
    """Per group, the per-read weights the reference is handed (no -Q: None for every read)."""
    return [[None] * len(g) for g in groups] if weights is None else weights


def batch_weights(groups, weights):
    """The weights Reference.batch keys and runs with: None without -Q."""
    return None if weights is None else [unit_filled(g, w) for g, w in zip(groups, weights)]


# abpoa -l on FASTQ files: -G -r 0 and -Q -G -r 2 are in reference_runs_qv.json (qv_reference.CLI_LIST_OPTS)
CLI_LIST_OPTS = [["-G", "-r", "2"], ["-G", "-r", "4"]]


def headline_groups():
    wl = synth.WORKLOADS["convex_10k"]
    return ps_cfg(wl.cfg), wl.groups(4)


def record_all():
    ref = ps_reference()
    assert ref.record_to, "set ABPOA_RECORD_REFERENCE to the store to record into"
    for kind in KINDS:
        groups, weights = kind_groups(kind)
        cfg = kind_cfg(kind)
        for g, w in zip(groups, group_weights(groups, weights)):
            reference_group(ref, cfg, g, w)
        if not kind.startswith("strand"):
            ref.batch(cfg, groups, want_msa=True, weights=batch_weights(groups, weights))
    cfg, groups = headline_groups()
    ref.batch(cfg, groups, want_msa=False)
    with tempfile.TemporaryDirectory() as d:
        files = fastq_files(Path(d))
        for opts in CLI_LIST_OPTS:
            reference_cli_md5(ref, [*opts, "-l"], files)
    ref.save()


if __name__ == "__main__":
    record_all()
