"""Shared test helpers (pure Python, no alignment logic)."""
from __future__ import annotations

from pathlib import Path

import numpy as np

from abpoa_b200.aligner import PoaConfig, PoaSession, encode

INPUTS = Path(__file__).resolve().parent / "golden" / "inputs"


def read_fasta(path: Path, m: int = 5) -> list[np.ndarray]:
    seqs, cur = [], []
    lines = Path(path).read_text().splitlines()
    is_fq = lines and lines[0].startswith("@")
    if is_fq:
        return [encode(lines[i + 1], m) for i in range(0, len(lines) - 1, 4)]
    for ln in lines:
        if ln.startswith(">"):
            if cur:
                seqs.append(encode("".join(cur), m))
            cur = []
        elif ln.strip():
            cur.append(ln.strip())
    if cur:
        seqs.append(encode("".join(cur), m))
    return seqs


def deletion_fan(seed=7, n=40, flank=220):
    """Reads that delete 1..n-1 bases in front of the same template position: that node collects one
    in-edge per read (> 32 predecessors: the chunked predecessor loops of the DP and of the backtrace)."""
    rng = np.random.default_rng(seed)
    t = rng.integers(0, 4, size=2 * flank).astype(np.uint8)
    return [t] + [np.concatenate([t[: flank - k], t[flank:]]) for k in range(1, n)]


def run_group(lib, cfg: PoaConfig, reads, want_msa: bool = True, use_oracle: bool = False, fast_order: bool = False, weights=None):
    """Progressive POA of one group through `lib`; returns per-read records + consensus (+ MSA).

    use_oracle=True: the graph / consensus / MSA code of `lib` is driven, but every
    alignment comes from the scalar oracle (oracle/libpoa_oracle.so).  That is how the
    CPU-only suite exercises the product's host layer without a GPU -- a test harness
    arrangement, not a product path."""
    cfg = PoaConfig(**{**cfg.__dict__, "out_msa": want_msa})
    with PoaSession(cfg, lib) as s:
        if use_oracle:
            from oracle_binding import oracle_align
            s.reset(max((len(r) for r in reads), default=1024))
            if fast_order:      # what the batch engine does per handle: spliced topological order between reads
                s.lib.dll.poa_graph_set_fast_order(s.ab.contents.abg, 1)
            alns = []
            for i, r in enumerate(reads):
                a, res = oracle_align(s, r)
                alns.append(a)
                s.add(r, res, len(reads), weights[i] if weights is not None else None)
            if fast_order:      # ... and the reference's Kahn order again before consensus / MSA
                import ctypes as C
                spl, fb = C.c_int64(0), C.c_int64(0)
                s.lib.dll.poa_graph_order_stats(s.ab.contents.abg, C.byref(spl), C.byref(fb))
                s.order_stats = (spl.value, fb.value)
                s.lib.dll.poa_graph_set_fast_order(s.ab.contents.abg, 0)
                g = s.ab.contents.abg.contents
                if g.node_n > 2:
                    g.is_topological_sorted = 0
                    s.lib.abpoa_topological_sort(s.ab.contents.abg, s.abpt)
        else:
            alns = s.run_reads(reads, weights=weights)
        s.generate()
        return {
            "order_stats": getattr(s, "order_stats", None),
            "alns": alns,
            "cons": s.consensus(),
            "cov": s.consensus_cov(),
            "msa": s.msa_rows(),
        }


def group_digest(r, m: int = 5):
    """Same shape as the entries of tests/golden/golden.json."""
    import hashlib

    from abpoa_b200.aligner import decode

    def sha(a):
        return hashlib.sha1(a.tobytes()).hexdigest()
    return {
        "alns": [{"aligned": a.aligned, "score": a.best_score, "cells": a.cells, "n_cigar": int(len(a.cigar)), "cigar_sha1": sha(a.cigar),
                  "ends": [a.node_s, a.node_e, a.query_s, a.query_e]} for a in r["alns"]],
        "cons": [decode(c, m) for c in r["cons"]],
        "cov_sha1": [sha(c) for c in r["cov"]],
        "msa_sha1": [sha(x) for x in r["msa"]],
        "msa_len": int(len(r["msa"][0])) if r["msa"] else 0,
    }


def assert_digest_equal(got, want, tag=""):
    assert len(got["alns"]) == len(want["alns"]), tag
    for i, (x, y) in enumerate(zip(got["alns"], want["alns"])):
        assert x == y, f"{tag} read {i}: {x} != {y}"
    for k in ("cons", "cov_sha1", "msa_len", "msa_sha1"):
        assert got[k] == want[k], f"{tag}: {k} differs"
