"""What the unmodified reference computes with quality weights (-Q, use_qv: a base's weight is added to the graph edge
that enters it, reference src/abpoa_graph.c:573-593 and :689-774), stored in tests/golden/reference_runs_qv.json and
keyed as in tests/reference_runs.py, plus the inputs the -Q tests share.

Recording: with oracle/_ref/ built (oracle/Makefile),

    ABPOA_RECORD_REFERENCE=tests/golden/reference_runs_qv.json python tests/qv_reference.py

runs the reference library and the reference CLI on every input of tests/test_gpu_qv.py; the CPU file
tests/test_chain_emul_qv.py records its own while it runs under the same variable."""
from __future__ import annotations

import ctypes as C
import json
import sys
import tempfile
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parent))
sys.path.insert(0, str(HERE))

from abpoa_b200 import synth  # noqa: E402
from abpoa_b200.aligner import PoaConfig, PoaSession, decode, make_para  # noqa: E402
from abpoa_b200.capi import ABPOA_MF, c_int_p, c_u8_p  # noqa: E402
from cases import AFFINE  # noqa: E402
from gfa_reference import md5, reference_cli_md5, with_file  # noqa: E402
from helpers import INPUTS  # noqa: E402
from mf_reference import set_outputs, with_n  # noqa: E402
from reference_runs import Hasher, Reference, _cfg_items  # noqa: E402
from strand_reference import strand_mix  # noqa: E402

STORE_QV = HERE / "golden" / "reference_runs_qv.json"


def qv_reference() -> Reference:
    ref = Reference()
    ref.stored = json.loads(STORE_QV.read_text()) if STORE_QV.exists() else {}
    return ref


def qv_cfg(cfg: PoaConfig | None = None, **kw) -> PoaConfig:
    return PoaConfig(**{**(cfg or PoaConfig()).__dict__, **kw, "use_qv": True})


def quality_weights(seed: int, reads, lo: int = 1, hi: int = 40):
    """Deterministic quality-like weights, lo..hi per base (phred + 1 of FASTQ qualities 0..hi - 1)."""
    rng = np.random.default_rng(seed)
    return [rng.integers(lo, hi + 1, size=len(r)).astype(np.int32) for r in reads]


def unit_filled(reads, weights):
    """`weights` with a read's missing (None) weights spelled out as ones: what abpoa_msa and the engines use for it."""
    return [np.ones(len(r), dtype=np.int32) if w is None else np.asarray(w, dtype=np.int32) for r, w in zip(reads, weights)]


def _msa_call(lib, cfg: PoaConfig, reads, weights, r: int | None, fp, names=None):
    p = make_para(lib, cfg)
    if r is not None:
        set_outputs(lib, p, r)
    ab = lib.abpoa_init()
    try:
        n = len(reads)
        arrs = [np.ascontiguousarray(x, dtype=np.uint8) for x in reads]
        ws = [None if w is None else np.ascontiguousarray(w, dtype=np.int32) for w in weights]
        lens = (C.c_int * max(n, 1))(*[len(x) for x in arrs])
        seqs = (c_u8_p * max(n, 1))(*[x.ctypes.data_as(c_u8_p) for x in arrs])
        wp = (c_int_p * max(n, 1))(*[None if w is None else w.ctypes.data_as(c_int_p) for w in ws])
        nm = None if names is None else (C.c_char_p * n)(*[s.encode() for s in names])
        lib.abpoa_msa(ab, p, n, nm, C.cast(lens, c_int_p), seqs, C.cast(wp, C.POINTER(c_int_p)), fp)
        return ab, p
    except BaseException:
        lib.abpoa_free(ab)
        lib.abpoa_free_para(p)
        raise


def group_text(lib, cfg: PoaConfig, reads, weights, r: int) -> bytes:
    """abpoa_msa(..., qual_weights, out_fp) of one group with -r r, reads without names."""
    held = []
    try:
        return with_file(lambda fp: held.append(_msa_call(lib, cfg, reads, weights, r, fp)))
    finally:
        for ab, p in held:
            lib.abpoa_free(ab)
            lib.abpoa_free_para(p)


def group_run(lib, cfg: PoaConfig, reads, weights) -> dict:
    """abpoa_msa over one group with its weights: which reads were flipped (-s), and a digest of the consensus, its
    coverage and the RC-MSA rows (what the batch engine returns for the group)."""
    cfg = PoaConfig(**{**cfg.__dict__, "out_cons": True})
    with PoaSession(cfg, lib) as s:
        ws = [None if w is None else np.ascontiguousarray(w, dtype=np.int32) for w in weights]
        wp = (c_int_p * len(reads))(*[None if w is None else w.ctypes.data_as(c_int_p) for w in ws])
        arrs = [np.ascontiguousarray(x, dtype=np.uint8) for x in reads]
        lens = (C.c_int * len(reads))(*[len(x) for x in arrs])
        seqs = (c_u8_p * len(reads))(*[x.ctypes.data_as(c_u8_p) for x in arrs])
        s.ab.contents.abs.contents.n_seq = 0
        s.lib.abpoa_msa(s.ab, s.abpt, len(reads), None, lens, seqs, C.cast(wp, C.POINTER(c_int_p)), None)
        abs_ = s.ab.contents.abs.contents
        return {"is_rc": [int(abs_.is_rc[i]) for i in range(len(reads))],
                "digest": Hasher().arrays(s.consensus()).arrays(s.consensus_cov()).arrays(s.msa_rows()).hex()}


def result_digest(r) -> str:
    """The digest of group_run for an abpoa_b200.batch.GroupResult."""
    return Hasher().arrays(r.cons).arrays(r.cov).arrays(r.msa).hex()


def reference_group(ref: Reference, cfg: PoaConfig, reads, weights) -> dict:
    return ref.value("qv_group", _cfg_items(cfg), lambda: group_run(ref.lib, cfg, reads, weights), arrays=list(reads) + unit_filled(reads, weights))


def reference_group_md5(ref: Reference, cfg: PoaConfig, reads, weights, r: int) -> str:
    return ref.value("qv_text", (_cfg_items(cfg), r), lambda: md5(group_text(ref.lib, cfg, reads, weights, r)),
                     arrays=list(reads) + unit_filled(reads, weights))


# ---- inputs shared by the GPU tests and the recording run ----
def kind_cfg(kind, out_msa=True):
    """-Q on convex / affine / amino acids (-c) / -a 1 / -s; -Q with a score term for every edge (-G) stays on the launch
    engine and is checked there too."""
    out = dict(out_msa=out_msa)
    if kind == "aa":
        return qv_cfg(PoaConfig(**synth.WORKLOADS["aa_blosum62_2k"].cfg.__dict__), **out)
    if kind == "mf":
        return qv_cfg(cons_algrm=ABPOA_MF, **out)
    if kind == "strand":
        return qv_cfg(amb_strand=True, **out)
    return qv_cfg(PoaConfig(**({} if kind in ("convex", "extreme", "partial") else AFFINE)), **out)


def kind_groups(kind):
    """(groups, weights): per group, per read int32 weights or None (the read has no qualities)."""
    if kind == "aa":
        groups = [synth.make_group(9300 + g, 8, 300, 0.08, m=27) for g in range(4)]
    elif kind == "strand":
        groups = [strand_mix(9320 + g, 5 + g % 4, 300 + 60 * (g % 4)) for g in range(6)]
    else:
        seed = {"convex": 9340, "affine": 9360, "mf": 9380, "extreme": 9400, "partial": 9420}[kind]
        groups = [with_n(synth.make_group(seed + g, 6 + g % 5, 300 + 50 * (g % 6), 0.04 + 0.01 * (g % 5)), seed + 10 + g, 4, 0.005 * (g % 2))
                  for g in range(8)]
    weights = [quality_weights(9500 + gi, g) for gi, g in enumerate(groups)]
    if kind == "extreme":       # the ends of a weight byte: many 0s and 255s
        for gi, ws in enumerate(weights):
            rng = np.random.default_rng(9550 + gi)
            for w in ws:
                u = rng.random(len(w))
                w[u < 0.2] = 0
                w[u > 0.8] = 255
    if kind == "partial":       # some reads without weights (unit weights), and one group without any
        weights = [None if gi == 3 else [None if i % 3 == 2 else w for i, w in enumerate(ws)] for gi, ws in enumerate(weights)]
    return groups, weights


BATCH_KINDS = ("convex", "affine", "aa", "mf", "strand", "extreme", "partial")
TEXT_R = (0, 2, 4)


def group_weights(groups, weights):
    """Per group, the per-read weights the reference is handed (a group without weights: None for every read)."""
    return [[None] * len(g) if ws is None else ws for g, ws in zip(groups, weights)]


def fastq_files(d: Path):
    """FASTQ files of seeded reads with seeded qualities (phred 0..39), one group each, for the CLI's list mode; then
    tests/golden/inputs/heter.fq."""
    files = []
    for g in range(6):
        reads = synth.make_group(9600 + g, 4 + g % 4, 200 + 70 * g, 0.06)
        ws = quality_weights(9650 + g, reads)
        p = d / f"q{g}.fq"
        p.write_text("".join(f"@read{g}_{i}\n{decode(r)}\n+\n{''.join(chr(32 + int(x)) for x in w)}\n" for i, (r, w) in enumerate(zip(reads, ws))))
        files.append(p)
    return files + [INPUTS / "heter.fq"]


CLI_LIST_OPTS = [["-Q", "-r", "0"], ["-Q", "-r", "2"], ["-Q", "-r", "4"], ["-Q", "-a", "1", "-r", "2"], ["-Q", "-s", "-r", "2"], ["-G", "-r", "0"],
                 ["-Q", "-G", "-r", "2"]]


def record_all():
    ref = qv_reference()
    assert ref.record_to, "set ABPOA_RECORD_REFERENCE to the store to record into"
    for kind in BATCH_KINDS:
        groups, weights = kind_groups(kind)
        gw = group_weights(groups, weights)
        cfg = kind_cfg(kind)
        for g, w in zip(groups, gw):
            reference_group(ref, cfg, g, w)
        if kind != "strand":
            ref.batch(cfg, groups, want_msa=True, weights=[unit_filled(g, w) for g, w in zip(groups, gw)])
    with tempfile.TemporaryDirectory() as d:
        files = fastq_files(Path(d))
        for opts in CLI_LIST_OPTS:
            reference_cli_md5(ref, [*opts, "-l"], files)
    ref.save()


if __name__ == "__main__":
    record_all()
