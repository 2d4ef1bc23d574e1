"""What the unmodified reference (abPOA v1.5.6) computes on the inputs of the parity tests, stored as digests.

The parity tests compare the product against these digests, so they need no build of the reference.  The
digests live in tests/golden/reference_runs.json, keyed by a hash of everything that determines the result
(configuration, reads, weights, options).  A group digest is "cells:unaligned:reads[:ends]":

  cells      DP cells of all alignments of the group
  unaligned  indices of the reads the reference did not align (comma-separated)
  reads      hash of (index, best score, graph-CIGAR length, FNV-1a of the graph-CIGAR words) of every aligned read,
             then of the consensus, coverage and RC-MSA rows -- what the batch engine reports per group
  ends       hash of (index, DP cells, node_s, node_e, query_s, query_e) of every aligned read (single-group runs only)

Recording: with ABPOA_RECORD_REFERENCE=<file> and the reference built under oracle/_ref/ (oracle/Makefile), every
lookup runs the reference instead, the tests compare against that run, and the digests are merged into <file> when
the session ends.
"""
from __future__ import annotations

import hashlib
import json
import os
from pathlib import Path

import numpy as np

from abpoa_b200.batch import fnv1a_words

STORE = Path(__file__).resolve().parent / "golden" / "reference_runs.json"
REFERENCE_LIB = Path(__file__).resolve().parent.parent / "oracle" / "_ref" / "libabpoa_ref.so"
HASH_HEX = 10


class Hasher:
    def __init__(self):
        self.h = hashlib.sha1()

    def add(self, *items):
        for x in items:
            self.h.update(repr(x).encode())
        return self

    def arrays(self, xs):
        self.add(len(xs))
        for x in xs:
            a = np.asarray(x, dtype=np.int64)
            self.add(a.size)
            self.h.update(a.tobytes())
        return self

    def hex(self, n=HASH_HEX):
        return self.h.hexdigest()[:n]


def _cfg_items(cfg):
    d = dict(cfg.__dict__)
    if d.get("score_matrix"):
        d["score_matrix"] = Path(d["score_matrix"]).name        # where the checkout lies is not part of the input
    return sorted(d.items())


def _group_key(h: Hasher, reads, weights):
    h.arrays(reads)
    h.add(weights is None)
    if weights is not None:
        h.arrays(weights)


def run_digest(r, with_ends=True) -> str:
    """Digest of a helpers.run_group result (either side)."""
    alns = r["alns"]
    aligned = [i for i, a in enumerate(alns) if a.aligned]
    reads = Hasher()
    for i in aligned:
        a = alns[i]
        reads.add((i, int(a.best_score), len(a.cigar), fnv1a_words(a.cigar)))
    reads.arrays(r["cons"]).arrays(r["cov"]).arrays(r["msa"])
    out = [str(sum(int(a.cells) for a in alns)), ",".join(str(i) for i, a in enumerate(alns) if not a.aligned), reads.hex()]
    if with_ends:
        ends = Hasher()
        for i in aligned:
            a = alns[i]
            ends.add((i, int(a.cells), a.node_s, a.node_e, a.query_s, a.query_e))
        out.append(ends.hex())
    return ":".join(out)


def batch_digest(r, n_reads: int, unaligned: str, msa=True) -> str:
    """Digest of an abpoa_b200.batch.GroupResult (run with record_reads=True) in the form of the reference's, given
    which reads the reference aligned."""
    skip = {int(i) for i in unaligned.split(",") if i}
    reads = Hasher()
    for i in range(n_reads):
        if i not in skip:
            reads.add((i, int(r.read_best_score[i]), int(r.read_n_cigar[i]), int(r.read_cigar_hash[i])))
    reads.arrays(r.cons).arrays(r.cov).arrays(r.msa if msa else [])
    return ":".join([str(int(r.dp_cells)), unaligned, reads.hex()])


def assert_run_matches(got_run, want: str, tag=""):
    """A product helpers.run_group result against the reference's digest: aligned reads, scores, graph-CIGARs, end
    points, DP cells, consensus, coverage and RC-MSA."""
    got = run_digest(got_run).split(":")
    want = want.split(":")
    assert got[1] == want[1], f"{tag}: unaligned reads {got[1]!r}, reference {want[1]!r}"
    assert got[0] == want[0], f"{tag}: DP cells {got[0]}, reference {want[0]}"
    assert got[2] == want[2], f"{tag}: scores / graph-CIGARs / consensus / coverage / RC-MSA differ from the reference"
    assert got[3] == want[3], f"{tag}: end points or per-read DP cells differ from the reference"


def assert_batch_matches(got, groups, want: list[str], tag="", msa=True):
    """Batch-engine results against the reference's digests, group by group."""
    assert len(got) == len(want) == len(groups)
    for gi, (r, g, w) in enumerate(zip(got, groups, want)):
        w_cells, unaligned, _ = w.split(":")
        assert r.dp_cells == int(w_cells), f"{tag} group {gi}: DP cells {r.dp_cells}, reference {w_cells}"
        assert batch_digest(r, len(g), unaligned, msa) == w, \
            f"{tag} group {gi}: per-read scores / CIGAR lengths / CIGAR hashes, consensus, coverage or RC-MSA differ from the reference"


def _batch_worker(args):
    cfg_kw, reads, want_msa, weights = args
    from abpoa_b200 import capi
    from abpoa_b200.aligner import PoaConfig
    from helpers import run_group
    r = run_group(capi.load_library(REFERENCE_LIB), PoaConfig(**cfg_kw), reads, want_msa=want_msa, weights=weights)
    return run_digest(r, with_ends=False)


class Reference:
    """Stored reference results; live ones while recording."""

    def __init__(self):
        self.record_to = os.environ.get("ABPOA_RECORD_REFERENCE")
        self.stored = json.loads(STORE.read_text()) if STORE.exists() else {}
        self.recorded: dict = {}
        self._lib = None

    @property
    def lib(self):
        """The live reference library (recording only)."""
        if self._lib is None:
            from abpoa_b200 import capi
            assert REFERENCE_LIB.exists(), f"recording needs the reference build {REFERENCE_LIB} (oracle/Makefile)"
            self._lib = capi.load_library(REFERENCE_LIB)
        return self._lib

    def value(self, kind: str, material, compute, arrays=()):
        """The stored value for (kind, material, arrays); while recording, compute() runs the reference and its (JSON)
        result is stored.  `material` is anything with an exact repr, `arrays` a list of integer arrays (reads)."""
        return self._lookup(f"{kind}:{Hasher().add(kind, material).arrays(arrays).hex(16)}", compute)

    def _lookup(self, key, compute):
        if self.record_to:
            if key not in self.recorded:
                self.recorded[key] = compute()
            return self.recorded[key]
        assert key in self.stored, f"no stored reference result {key} in {STORE.name}: record it (see tests/reference_runs.py)"
        return self.stored[key]

    def run(self, cfg, reads, want_msa=True, weights=None) -> str:
        """Digest of helpers.run_group(reference, cfg, reads, want_msa, weights)."""
        h = Hasher().add("run", _cfg_items(cfg), bool(want_msa))
        _group_key(h, reads, weights)

        def compute():
            from helpers import run_group
            return run_digest(run_group(self.lib, cfg, reads, want_msa=want_msa, weights=weights))
        return self._lookup(f"run:{h.hex(16)}", compute)

    def batch(self, cfg, groups, want_msa=False, weights=None) -> list[str]:
        """Per-group digests (without end points) of the reference's run of every group."""
        h = Hasher().add("batch", _cfg_items(cfg), bool(want_msa), len(groups))
        for gi, g in enumerate(groups):
            _group_key(h, g, weights[gi] if weights else None)

        def compute():
            jobs = [(dict(cfg.__dict__), g, want_msa, weights[gi] if weights else None) for gi, g in enumerate(groups)]
            if sum(len(r) for g in groups for r in g) < 2_000_000:
                return [_batch_worker(j) for j in jobs]
            import multiprocessing as mp       # the reference is single-threaded: 10 kbp groups in parallel processes
            with mp.get_context("spawn").Pool(min(os.cpu_count() or 4, len(jobs))) as pool:
                return pool.map(_batch_worker, jobs)
        return self._lookup(f"batch:{h.hex(16)}", compute)

    def save(self):
        if not self.record_to or not self.recorded:
            return
        out = Path(self.record_to)
        merged = json.loads(out.read_text()) if out.exists() else {}
        merged.update(self.recorded)
        out.write_text(json.dumps(dict(sorted(merged.items())), indent=0) + "\n")
