"""What the unmodified reference computes with ambiguous-strand alignment (-s, reference src/abpoa_align.c:322-344),
stored in tests/golden/reference_runs_strand.json and keyed as in tests/reference_runs.py, plus the inputs the -s tests
share.

Recording: with oracle/_ref/ built (oracle/Makefile),

    ABPOA_RECORD_REFERENCE=tests/golden/reference_runs_strand.json python tests/strand_reference.py

runs the reference library and the reference CLI on every input of tests/test_gpu_strand.py; the CPU file
tests/test_chain_emul_strand.py records its own while it runs under the same variable."""
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
from mf_reference import set_outputs, with_n  # noqa: E402
from reference_runs import Hasher, Reference, _cfg_items  # noqa: E402

STORE_STRAND = HERE / "golden" / "reference_runs_strand.json"


def strand_reference() -> Reference:
    ref = Reference()
    ref.stored = json.loads(STORE_STRAND.read_text()) if STORE_STRAND.exists() else {}
    return ref


def strand_cfg(cfg: PoaConfig | None = None, **kw) -> PoaConfig:
    return PoaConfig(**{**(cfg or PoaConfig()).__dict__, **kw, "amb_strand": True})


def revcomp(x) -> np.ndarray:
    """The reverse complement by the reference's rule: code b < 4 becomes 3 - b, every other code 4 (with -c too)."""
    x = np.asarray(x, dtype=np.uint8)
    return np.ascontiguousarray(np.where(x < 4, 3 - x, 4).astype(np.uint8)[::-1])


def strand_mix(seed, n, length, err=0.05, m=5):
    """A synthetic group in which every third read (1, 4, 7, ...) arrives reverse-complemented."""
    return [revcomp(r) if i % 3 == 1 else r for i, r in enumerate(synth.make_group(seed, n, length, err, m=m))]


def names_of(n):
    return [f"r{i}" for i in range(n)]


def group_text(lib, cfg: PoaConfig, reads, r: int) -> bytes:
    """abpoa_msa(..., out_fp) of one group with -r r, reads named r0, r1, ... (so that flipped reads print as
    r<i>_reverse_complement and as reversed '-' P lines)."""
    p = make_para(lib, cfg)
    set_outputs(lib, p, r)
    ab = lib.abpoa_init()
    try:
        n = len(reads)
        arrs = [np.ascontiguousarray(x, dtype=np.uint8) for x in reads]
        lens = (C.c_int * n)(*[len(x) for x in arrs])
        seqs = (c_u8_p * n)(*[x.ctypes.data_as(c_u8_p) for x in arrs])
        nm = (C.c_char_p * n)(*[s.encode() for s in names_of(n)])
        return with_file(lambda fp: lib.abpoa_msa(ab, p, n, nm, C.cast(lens, c_int_p), seqs, None, fp))
    finally:
        lib.abpoa_free(ab)
        lib.abpoa_free_para(p)


def group_run(lib, cfg: PoaConfig, reads) -> dict:
    """abpoa_msa over one group: which reads were flipped, and a digest of the consensus, its coverage and the RC-MSA
    rows (what the batch engine returns for the group)."""
    cfg = PoaConfig(**{**cfg.__dict__, "out_cons": True})
    with PoaSession(cfg, lib) as s:
        s.msa(reads)
        abs_ = s.ab.contents.abs.contents
        return {"is_rc": [int(abs_.is_rc[i]) for i in range(len(reads))],
                "digest": Hasher().arrays(s.consensus()).arrays(s.consensus_cov()).arrays(s.msa_rows()).hex()}


def result_digest(r) -> str:
    """The digest of group_run for an abpoa_b200.batch.GroupResult."""
    return Hasher().arrays(r.cons).arrays(r.cov).arrays(r.msa).hex()


def reference_group(ref: Reference, cfg: PoaConfig, reads) -> dict:
    return ref.value("strand_group", _cfg_items(cfg), lambda: group_run(ref.lib, cfg, reads), arrays=reads)


def reference_group_md5(ref: Reference, cfg: PoaConfig, reads, r: int) -> str:
    return ref.value("strand_text", (_cfg_items(cfg), r), lambda: md5(group_text(ref.lib, cfg, reads, r)), arrays=reads)


# ---- inputs shared by the GPU tests and the recording run ----
def kind_cfg(kind, out_msa=True):
    if kind == "aa":
        return strand_cfg(PoaConfig(**synth.WORKLOADS["aa_blosum62_2k"].cfg.__dict__), out_msa=out_msa)
    if kind == "mf":
        return strand_cfg(out_msa=out_msa, cons_algrm=ABPOA_MF)
    return strand_cfg(PoaConfig(**({} if kind == "convex" else AFFINE)), out_msa=out_msa)


def kind_groups(kind):
    """strand_mix groups: convex / affine / -a 1 with a few N, amino acids (-c) through the same complement rule."""
    if kind == "aa":
        return [strand_mix(9700 + g, 7, 300, 0.08, m=27) for g in range(4)]
    seed = {"convex": 9600, "affine": 9640, "mf": 9680}[kind]
    return [with_n(strand_mix(seed + g, 5 + g % 4, 300 + 60 * (g % 4)), seed + 20 + g, 4, 0.005 * (g % 2)) for g in range(8)]


BATCH_KINDS = ("convex", "affine", "aa", "mf")


def list_files(d: Path):
    """Named FASTA files with flipped reads, one group each, for the CLI's list mode."""
    files = []
    for g in range(6):
        reads = strand_mix(9800 + g, 4 + g % 4, 200 + 70 * g)
        p = d / f"s{g}.fa"
        p.write_text("".join(f">read{g}_{i}\n{decode(r)}\n" for i, r in enumerate(reads)))
        files.append(p)
    return files


CLI_LIST_R = ["0", "1", "2", "3", "4"]


def record_all():
    ref = strand_reference()
    assert ref.record_to, "set ABPOA_RECORD_REFERENCE to the store to record into"
    for kind in BATCH_KINDS:
        cfg = kind_cfg(kind)
        for g in kind_groups(kind):
            reference_group(ref, cfg, g)
    with tempfile.TemporaryDirectory() as d:
        files = list_files(Path(d))
        for r in CLI_LIST_R:
            reference_cli_md5(ref, ["-s", "-r", r, "-l"], files)
    ref.save()


if __name__ == "__main__":
    record_all()
