"""What the unmodified reference prints as GFA (-r 3 / -r 4, reference src/abpoa_output.c:194-294), stored as md5s in
tests/golden/reference_runs_gfa.json and keyed as in tests/reference_runs.py, plus the inputs the GFA tests share.

Recording: with oracle/_ref/ built (oracle/Makefile),

    ABPOA_RECORD_REFERENCE=tests/golden/reference_runs_gfa.json python tests/gfa_reference.py

runs the reference library and the reference CLI on every input of tests/test_gpu_gfa.py (the CPU file
tests/test_chain_emul_gfa.py records its own while it runs under the same variable)."""
from __future__ import annotations

import ctypes as C
import hashlib
import json
import os
import subprocess
import sys
import tempfile
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parent))
sys.path.insert(0, str(HERE))

from abpoa_b200 import synth  # noqa: E402
from abpoa_b200.aligner import PoaConfig, decode, make_para  # noqa: E402
from abpoa_b200.capi import c_int_p, c_u8_p  # noqa: E402
from cases import AFFINE  # noqa: E402
from helpers import INPUTS  # noqa: E402
from reference_runs import Reference, _cfg_items  # noqa: E402

STORE_GFA = HERE / "golden" / "reference_runs_gfa.json"
REF_BIN = HERE.parent / "oracle" / "_ref" / "abpoa_ref"

_libc = C.CDLL(None)
_libc.fopen.restype = C.c_void_p
_libc.fopen.argtypes = [C.c_char_p, C.c_char_p]
_libc.fclose.argtypes = [C.c_void_p]


def gfa_reference() -> Reference:
    ref = Reference()
    ref.stored = json.loads(STORE_GFA.read_text()) if STORE_GFA.exists() else {}
    return ref


def md5(b: bytes) -> str:
    return hashlib.md5(b).hexdigest()


def gfa_para(lib, cfg: PoaConfig, out_cons: bool):
    """abpoa_para_t with out_gfa set before abpoa_post_set_para, as the reference CLI's -r 3 / -r 4 does."""
    p = make_para(lib, PoaConfig(**{**cfg.__dict__, "out_cons": bool(out_cons), "out_msa": False}))
    p.contents.out_gfa = 1
    lib.abpoa_post_set_para(p)
    return p


def with_file(fn) -> bytes:
    """Call fn(FILE *) on a fresh temporary file and return what it wrote."""
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "out.gfa")
        fp = _libc.fopen(path.encode(), b"w")
        assert fp, "fopen failed"
        try:
            fn(fp)
        finally:
            _libc.fclose(fp)
        return Path(path).read_bytes()


def msa_text(lib, cfg: PoaConfig, reads, out_cons: bool) -> bytes:
    """abpoa_msa(..., out_fp) of one group with -r 3 (out_cons False) or -r 4, reads without names."""
    p = gfa_para(lib, cfg, out_cons)
    ab = lib.abpoa_init()
    try:
        n = len(reads)
        arrs = [np.ascontiguousarray(r, dtype=np.uint8) for r in reads]
        lens = (C.c_int * max(n, 1))(*[len(a) for a in arrs])
        seqs = (c_u8_p * max(n, 1))(*[a.ctypes.data_as(c_u8_p) for a in arrs])
        return with_file(lambda fp: lib.abpoa_msa(ab, p, n, None, C.cast(lens, c_int_p), seqs, None, fp))
    finally:
        lib.abpoa_free(ab)
        lib.abpoa_free_para(p)


def reference_msa_md5(ref: Reference, cfg: PoaConfig, reads, out_cons: bool) -> str:
    return ref.value("gfa_msa", (_cfg_items(cfg), bool(out_cons)), lambda: md5(msa_text(ref.lib, cfg, reads, out_cons)), arrays=reads)


def reference_batch_md5(ref: Reference, cfg: PoaConfig, groups, out_cons: bool) -> str:
    """md5 of the groups' GFA one after the other (what abpoa_gpu_msa_batch_write prints without names)."""
    arrays = [np.asarray(r) for g in groups for r in g]
    material = (_cfg_items(cfg), bool(out_cons), [len(g) for g in groups])
    return ref.value("gfa_batch", material, lambda: md5(b"".join(msa_text(ref.lib, cfg, g, out_cons) for g in groups)), arrays=arrays)


def reference_cli_md5(ref: Reference, args, files) -> str:
    """md5 of the reference CLI's stdout for `args` followed by the files (single file) or by `-l <list>` (list mode)."""
    inputs = [hashlib.sha1(Path(p).read_bytes()).hexdigest() for p in files]

    def compute():
        assert REF_BIN.exists(), f"recording needs the reference CLI {REF_BIN} (oracle/Makefile)"
        with tempfile.TemporaryDirectory() as d:
            tail = [str(files[0])]
            if args and args[-1] == "-l":
                lst = Path(d) / "list.txt"
                lst.write_text("".join(f"{p}\n" for p in files))
                tail = [str(lst)]
            return md5(subprocess.run([str(REF_BIN), *args, *tail], capture_output=True, check=True).stdout)
    return ref.value("gfa_cli", (list(args), inputs), compute)


# ---- inputs shared by the GPU tests and the recording run ----
CLI_SINGLE = [
    (["-r3"], "seq.fa"), (["-r4"], "seq.fa"), (["-r3"], "test.fa"), (["-r4"], "test.fa"),
    (["-r3"], "heter.fq"), (["-r4"], "heter.fq"), (["-r3"], "3alleles.fa"), (["-r4"], "3alleles.fa"),
    (["-s", "-r3"], "heter.fa"), (["-m", "1", "-r4"], "seq.fa"),
]
CLI_LIST_OPTS = [["-r3"], ["-r4"], ["-m", "1", "-r3"], ["-Q", "-r4"]]


def list_files(d: Path):
    """The file set of test_cli.py::test_cli_list_mode_matches_reference_binary, written under d."""
    files = []
    for g in range(7):
        reads = synth.make_group(7000 + g, 4 + g % 4, 150 + 60 * g, 0.06)
        p = d / f"g{g}.fa"
        p.write_text("".join(f">read{g}_{i} len={len(r)}\n{decode(r)}\n" for i, r in enumerate(reads)))
        files.append(p)
    return files + [INPUTS / "seq.fa", INPUTS / "heter.fq"]


def aa_file(d: Path):
    """An amino-acid group as FASTA (for -c)."""
    reads = synth.make_group(8700, 8, 300, 0.08, m=27)
    p = d / "aa.fa"
    p.write_text("".join(f">p{i}\n{decode(r, m=27)}\n" for i, r in enumerate(reads)))
    return p


def kind_cfg(kind):
    if kind == "aa":
        return PoaConfig(**synth.WORKLOADS["aa_blosum62_2k"].cfg.__dict__)
    return PoaConfig(**({} if kind == "convex" else AFFINE))


def kind_groups(kind):
    if kind == "aa":
        return [synth.make_group(8600 + g, 10, 400, 0.10, m=27) for g in range(5)]
    seed = 8500 if kind == "convex" else 8550
    return [synth.make_group(seed + g, 6 + g % 5, 300 + 50 * (g % 6), 0.04 + 0.01 * (g % 5)) for g in range(10)]


def word_edge_groups():
    return [synth.make_group(8800 + n, n, 150, 0.06) for n in (64, 65, 130)]


def mixed_groups():
    """Ragged groups, a 2-read group, a 1-read group and an empty group (the last two never reach the chain)."""
    rng = np.random.default_rng(17)
    groups = []
    for g in range(8):
        base = synth.make_group(8300 + g, 3 + 2 * (g % 4), 700, 0.06)
        groups.append([np.ascontiguousarray(r[: int(rng.integers(5, len(r)))]) if i % 3 == 1 else r for i, r in enumerate(base)])
    return groups + [synth.make_group(8320, 2, 400, 0.05), synth.make_group(8321, 1, 90, 0.0), []]


BATCH_INPUTS = {f"{kind}-{r}": (lambda kind=kind: (kind_cfg(kind), kind_groups(kind))) for kind in ("convex", "affine", "aa") for r in ("r3", "r4")}
BATCH_INPUTS.update({f"word-edges-{r}": (lambda: (PoaConfig(), word_edge_groups())) for r in ("r3", "r4")})
BATCH_INPUTS.update({f"mixed-{r}": (lambda: (PoaConfig(), mixed_groups())) for r in ("r3", "r4")})


def record_all():
    ref = gfa_reference()
    assert ref.record_to, "set ABPOA_RECORD_REFERENCE to the store to record into"
    for args, f in CLI_SINGLE:
        reference_cli_md5(ref, args, [INPUTS / f])
    with tempfile.TemporaryDirectory() as d:
        files = list_files(Path(d))
        for opts in CLI_LIST_OPTS:
            reference_cli_md5(ref, [*opts, "-l"], files)
        aa = aa_file(Path(d))
        for r in ("-r3", "-r4"):
            reference_cli_md5(ref, ["-c", r], [aa])
    for name, make in BATCH_INPUTS.items():
        cfg, groups = make()
        reference_batch_md5(ref, cfg, groups, name.endswith("r4"))
    ref.save()


if __name__ == "__main__":
    record_all()
