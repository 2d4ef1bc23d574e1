"""What the unmodified reference computes with the most-frequent-base consensus (-a 1, reference
src/abpoa_output.c:393-451, :549-586), stored in tests/golden/reference_runs_mf.json and keyed as in
tests/reference_runs.py, plus the inputs the -a 1 tests share.

Recording: with oracle/_ref/ built (oracle/Makefile),

    ABPOA_RECORD_REFERENCE=tests/golden/reference_runs_mf.json python tests/mf_reference.py

runs the reference library and the reference CLI on every input of tests/test_gpu_mf.py; the CPU files
tests/test_chain_emul_mf.py and tests/test_host_mf.py record their own while they run under the same variable."""
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
from abpoa_b200 import aligner  # noqa: E402
from abpoa_b200.aligner import PoaConfig, make_para  # noqa: E402
from abpoa_b200.capi import ABPOA_MF, c_int_p, c_u8_p  # noqa: E402
from cases import AFFINE  # noqa: E402
from gfa_reference import aa_file, list_files, md5, reference_cli_md5, with_file  # noqa: E402
from helpers import INPUTS  # noqa: E402
from reference_runs import Reference, _cfg_items  # noqa: E402

STORE_MF = HERE / "golden" / "reference_runs_mf.json"

# -r of the reference CLI -> (out_cons, out_msa, out_gfa, out_fq)
OUT = {0: (1, 0, 0, 0), 1: (0, 1, 0, 0), 2: (1, 1, 0, 0), 3: (0, 0, 1, 0), 4: (1, 0, 1, 0), 5: (1, 0, 0, 1)}


def mf_reference() -> Reference:
    ref = Reference()
    ref.stored = json.loads(STORE_MF.read_text()) if STORE_MF.exists() else {}
    return ref


def mf_cfg(cfg: PoaConfig | None = None, **kw) -> PoaConfig:
    return PoaConfig(**{**(cfg or PoaConfig()).__dict__, **kw, "cons_algrm": ABPOA_MF})


def set_outputs(lib, abpt, r: int):
    """The output fields of `abpt` as the reference CLI's -r sets them, then abpoa_post_set_para again."""
    a = abpt.contents
    a.out_cons, a.out_msa, a.out_gfa, a.out_fq = OUT[r]
    lib.abpoa_post_set_para(abpt)


def group_text(lib, cfg: PoaConfig, reads, r: int, sub_aln: bool = False) -> bytes:
    """abpoa_msa(..., out_fp) of one group with -r r, reads without names."""
    p = make_para(lib, cfg)
    set_outputs(lib, p, r)
    if sub_aln:
        p.contents.sub_aln = 1
    ab = lib.abpoa_init()
    try:
        n = len(reads)
        arrs = [np.ascontiguousarray(x, dtype=np.uint8) for x in reads]
        lens = (C.c_int * max(n, 1))(*[len(x) for x in arrs])
        seqs = (c_u8_p * max(n, 1))(*[x.ctypes.data_as(c_u8_p) for x in arrs])
        return with_file(lambda fp: lib.abpoa_msa(ab, p, n, None, C.cast(lens, c_int_p), seqs, None, fp))
    finally:
        lib.abpoa_free(ab)
        lib.abpoa_free_para(p)


def reference_group_md5(ref: Reference, cfg: PoaConfig, reads, r: int) -> str:
    return ref.value("mf_msa", (_cfg_items(cfg), r), lambda: md5(group_text(ref.lib, cfg, reads, r)), arrays=reads)


def reference_batch_md5(ref: Reference, cfg: PoaConfig, groups, r: int) -> str:
    """md5 of the groups' output one after the other (what abpoa_gpu_msa_batch_write prints without names)."""
    arrays = [np.asarray(x) for g in groups for x in g]
    material = (_cfg_items(cfg), r, [len(g) for g in groups])
    return ref.value("mf_batch", material, lambda: md5(b"".join(group_text(ref.lib, cfg, g, r) for g in groups)), arrays=arrays)


def with_n(reads, seed: int, code: int, frac: float = 0.03):
    """`reads` with a fraction of their bases replaced by `code` (N for nucleotides, the last code for amino acids)."""
    rng = np.random.default_rng(seed)
    out = []
    for x in reads:
        y = np.array(x, dtype=np.uint8)
        y[rng.random(len(y)) < frac] = code
        out.append(y)
    return out


# ---- inputs shared by the GPU tests and the recording run ----
CLI_SINGLE = [
    (["-a", "1"], "seq.fa"), (["-a", "1", "-r", "2"], "seq.fa"), (["-a", "1", "-r", "4"], "seq.fa"), (["-a", "1", "-r", "5"], "seq.fa"),
    (["-a", "1"], "test.fa"), (["-a", "1", "-r", "2"], "heter.fa"), (["-a", "1"], "3alleles.fa"), (["-a", "1", "-r", "2"], "3alleles.fa"),
    (["-a", "1", "-s"], "heter.fa"), (["-a", "1", "-m", "1"], "seq.fa"), (["-a", "1", "-Q"], "heter.fq"),
]
CLI_LIST_OPTS = [["-a", "1"], ["-a", "1", "-r", "2"], ["-a", "1", "-m", "1"], ["-a", "1", "-Q"], ["-a", "1", "-r", "4"]]


def kind_cfg(kind, r):
    out = dict(out_cons=True, out_msa=r == 2)
    if kind == "aa":
        return mf_cfg(PoaConfig(**synth.WORKLOADS["aa_blosum62_2k"].cfg.__dict__), **out)
    return mf_cfg(PoaConfig(**({} if kind == "convex" else AFFINE)), **out)


def kind_groups(kind):
    """Convex / affine groups with some N (code 4), amino-acid groups with some code 26."""
    if kind == "aa":
        return [with_n(synth.make_group(9100 + g, 10, 400, 0.10, m=27), 9150 + g, 26) for g in range(5)]
    seed = 9000 if kind == "convex" else 9050
    return [with_n(synth.make_group(seed + g, 6 + g % 5, 300 + 50 * (g % 6), 0.04 + 0.01 * (g % 5)), seed + 20 + g, 4, 0.01 * (g % 3))
            for g in range(10)]


def word_edge_groups():
    return [synth.make_group(9200 + n, n, 150, 0.06) for n in (64, 65, 130)]


def mixed_groups():
    """Ragged groups, 2-read groups, 25 % error groups, a 1-read group and an empty group (the last two never reach the
    chain)."""
    rng = np.random.default_rng(19)
    groups = []
    for g in range(8):
        base = synth.make_group(9300 + g, 3 + 2 * (g % 4), 700, 0.06)
        groups.append([np.ascontiguousarray(x[: int(rng.integers(5, len(x)))]) if i % 3 == 1 else x for i, x in enumerate(base)])
    return groups + [synth.make_group(9320, 2, 400, 0.05), synth.make_group(9322, 2, 300, 0.25), synth.make_group(9323, 12, 300, 0.25),
                     synth.make_group(9321, 1, 90, 0.0), []]


# batches checked against Reference.batch digests (-r 0 / -r 2)
BATCH_INPUTS = {f"{kind}-r{r}": (lambda kind=kind, r=r: (kind_cfg(kind, r), kind_groups(kind))) for kind in ("convex", "affine", "aa") for r in (0, 2)}
BATCH_INPUTS.update({f"word-edges-r{r}": (lambda r=r: (mf_cfg(out_msa=r == 2), word_edge_groups())) for r in (0, 2)})
BATCH_INPUTS.update({f"mixed-r{r}": (lambda r=r: (mf_cfg(out_msa=r == 2), mixed_groups())) for r in (0, 2)})
# batches whose -r 4 GFA text is checked against the reference's md5
GFA_INPUTS = {"convex": lambda: (kind_cfg("convex", 0), kind_groups("convex")), "aa": lambda: (kind_cfg("aa", 0), kind_groups("aa")),
              "mixed": lambda: (mf_cfg(), mixed_groups())}


def subgraph_inputs():
    """The reads and windows of test_gpu_cases.py::test_subgraph_alignment's loop (the reference's sub_example.c)."""
    rng = np.random.default_rng(78)
    full = synth.make_group(9400, 4, 400, 0.06)
    reads, windows = list(full), [(0, 1)] * len(full)
    t = full[0]
    for _ in range(6):
        a = int(rng.integers(10, 150)); b = int(rng.integers(250, 390))
        piece = t[a:b].copy()
        piece[::17] = (piece[::17] + 1) % 4
        reads.append(piece)
        windows.append((2 + a, 2 + b - 1))
    return reads, windows


def subgraph_walk_mf(lib, reads, windows) -> str:
    """test_gpu_cases.subgraph_walk with -a 1 -r 2 and sub_aln = 1, as the reference's sub_example.c sets them."""
    from test_gpu_cases import subgraph_walk
    plain = aligner.make_para

    def with_sub_aln(lib_, cfg_):
        p = plain(lib_, cfg_)
        p.contents.sub_aln = 1
        return p
    aligner.make_para = with_sub_aln
    try:
        return subgraph_walk(lib, mf_cfg(out_msa=True), reads, windows)
    finally:
        aligner.make_para = plain


def reference_subgraph_walk(ref: Reference) -> str:
    reads, windows = subgraph_inputs()
    return ref.value("mf_subgraph_walk", windows, lambda: subgraph_walk_mf(ref.lib, reads, windows), reads)


def pyabpoa_digest(lib):
    """Every field of msa_aligner(cons_algrm="MF").msa of the pyabpoa example, with and without the MSA."""
    from abpoa_b200.aligner import msa_aligner
    from test_gpu_pyabpoa import EXAMPLE, digest
    return [digest(msa_aligner(cons_algrm="MF", lib=lib).msa(EXAMPLE, out_cons=True, out_msa=m)) for m in (False, True)]


def reference_pyabpoa(ref: Reference):
    return ref.value("mf_pyabpoa", "example", lambda: pyabpoa_digest(ref.lib))


def record_all():
    ref = mf_reference()
    assert ref.record_to, "set ABPOA_RECORD_REFERENCE to the store to record into"
    for args, f in CLI_SINGLE:
        reference_cli_md5(ref, args, [INPUTS / f])
    with tempfile.TemporaryDirectory() as d:
        files = list_files(Path(d))
        for opts in CLI_LIST_OPTS:
            reference_cli_md5(ref, [*opts, "-l"], files)
        aa = aa_file(Path(d))
        for r in ("0", "2"):
            reference_cli_md5(ref, ["-a", "1", "-c", "-r", r], [aa])
    for name, make in BATCH_INPUTS.items():
        cfg, groups = make()
        ref.batch(cfg, groups, want_msa=cfg.out_msa)
    for make in GFA_INPUTS.values():
        cfg, groups = make()
        reference_batch_md5(ref, cfg, groups, 4)
    reference_subgraph_walk(ref)
    reference_pyabpoa(ref)
    ref.save()


if __name__ == "__main__":
    record_all()
