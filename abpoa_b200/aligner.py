"""Host-side mirror of the reference's Python interface (python/pyabpoa.pyx:9-371).

``msa_aligner`` / ``msa_result`` keep pyabpoa's names, arguments and result fields, but the
calls go through the abpoa.h C ABI of a shared object -- by default the GPU library
(``libabpoa_b200.so``), whose alignments run in CUDA kernels.  Passing ``lib=`` lets the test
suite run the very same driver over ``oracle/_ref/libabpoa_ref.so`` (the unmodified
reference) to compare results; the product path never does that.

``PoaSession`` is the finer-grained driver used by parity tests and the benchmark: it steps
one read at a time (``abpoa_align_sequence_to_graph`` + ``abpoa_add_graph_alignment``, the
loop of reference src/abpoa_align.c:312-352 and pyabpoa.pyx:189-209) and records the best
score, the full graph-CIGAR, and the number of DP cells of every alignment.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field
from typing import Iterable, Sequence

import numpy as np

from . import capi
from .capi import (ABPOA_AFFINE_GAP, ABPOA_CONVEX_GAP, ABPOA_EXTEND_MODE, ABPOA_GLOBAL_MODE, ABPOA_HB,
                   ABPOA_LINEAR_GAP, ABPOA_LOCAL_MODE, ABPOA_MF, PoaLibrary, abpoa_res_t, c_int_p, c_u8_p)

NT_ORDER = "ACGTN"
AA_ORDER = "ACGTNBDEFHIJKLMOPQRSUVWXYZ*"


def encode(seq: str | bytes | np.ndarray, m: int = 5) -> np.ndarray:
    """Residue letters -> codes 0..m-1 (tables of reference src/abpoa_seq.c:15-95)."""
    if isinstance(seq, np.ndarray):
        return np.ascontiguousarray(seq, dtype=np.uint8)
    if isinstance(seq, str):
        seq = seq.encode()
    lut = np.full(256, m - 1, dtype=np.uint8)
    if m == 5:
        for ch, v in zip("ACGTUN", (0, 1, 2, 3, 3, 4)):
            lut[ord(ch)] = v
            lut[ord(ch.lower())] = v
    else:
        for v, ch in enumerate(AA_ORDER[:26]):
            lut[ord(ch)] = v
            lut[ord(ch.lower())] = v
    return lut[np.frombuffer(seq, dtype=np.uint8)]


def decode(codes: Iterable[int], m: int = 5) -> str:
    order = NT_ORDER if m == 5 else AA_ORDER
    return "".join(order[c] if c < len(order) else "-" for c in codes)


@dataclass
class PoaConfig:
    """The subset of abpoa_para_t a caller normally sets (CLI flags of reference src/abpoa.c:172-236)."""
    align_mode: int = ABPOA_GLOBAL_MODE
    m: int = 5
    match: int = 2
    mismatch: int = 4
    score_matrix: str | None = None
    gap_open1: int = 4
    gap_open2: int = 24
    gap_ext1: int = 2
    gap_ext2: int = 1
    wb: int = 10
    wf: float = 0.01
    zdrop: int = -1
    out_cons: bool = True
    out_msa: bool = False
    amb_strand: bool = False
    inc_path_score: bool = False
    put_gap_on_right: bool = False
    put_gap_at_end: bool = False
    use_qv: bool = False
    cons_algrm: int = ABPOA_HB
    max_n_cons: int = 1
    min_freq: float = 0.25


def make_para(lib: PoaLibrary, cfg: PoaConfig):
    """abpoa_init_para + field assignment + abpoa_post_set_para, as every reference caller does."""
    p = lib.abpoa_init_para()
    a = p.contents
    a.align_mode = cfg.align_mode
    if cfg.m != a.m:
        a.m = cfg.m
        a.mat = C.cast(capi.libc_realloc(a.mat, cfg.m * cfg.m * 4), c_int_p)
    a.match, a.mismatch = cfg.match, cfg.mismatch
    a.gap_open1, a.gap_open2, a.gap_ext1, a.gap_ext2 = cfg.gap_open1, cfg.gap_open2, cfg.gap_ext1, cfg.gap_ext2
    a.wb, a.wf = cfg.wb, cfg.wf
    a.zdrop = cfg.zdrop
    a.out_cons, a.out_msa = int(cfg.out_cons), int(cfg.out_msa)
    a.amb_strand = int(cfg.amb_strand)
    a.inc_path_score = int(cfg.inc_path_score)
    a.put_gap_on_right, a.put_gap_at_end = int(cfg.put_gap_on_right), int(cfg.put_gap_at_end)
    a.use_qv = int(cfg.use_qv)
    a.cons_algrm, a.max_n_cons, a.min_freq = cfg.cons_algrm, cfg.max_n_cons, cfg.min_freq
    if cfg.score_matrix:
        a.use_score_matrix = 1
        # the library frees mat_fn with free(): hand it a malloc'ed copy
        raw = str(cfg.score_matrix).encode() + b"\0"
        buf = capi.libc_realloc(None, len(raw))
        C.memmove(buf, raw, len(raw))
        C.cast(C.byref(a, abpoa_para_mat_fn_offset()), C.POINTER(C.c_void_p))[0] = buf
    lib.abpoa_post_set_para(p)
    return p


def abpoa_para_mat_fn_offset() -> int:
    return capi.abpoa_para_t.mat_fn.offset


@dataclass
class ReadAlignment:
    """What one abpoa_align_sequence_to_graph call produced."""
    aligned: bool                    # False for the first read of a group (empty graph, no DP)
    best_score: int = 0
    cigar: np.ndarray = field(default_factory=lambda: np.zeros(0, dtype=np.uint64))
    node_s: int = 0
    node_e: int = 0
    query_s: int = 0
    query_e: int = 0
    cells: int = 0                   # sum over DP rows of dp_end - dp_beg + 1
    rows: int = 0


class PoaSession:
    """One abpoa_t handle + one abpoa_para_t on a given library."""

    def __init__(self, cfg: PoaConfig | None = None, lib: PoaLibrary | None = None):
        self.lib = lib if lib is not None else capi.product()
        self.cfg = cfg or PoaConfig()
        self.abpt = make_para(self.lib, self.cfg)
        self.ab = self.lib.abpoa_init()
        self.n_seq = 0
        self._keep = []

    def close(self):
        if self.ab:
            self.lib.abpoa_free(self.ab)
            self.lib.abpoa_free_para(self.abpt)
            self.ab = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    # ---- per-read stepping -------------------------------------------------------------
    def reset(self, qlen: int = 1024):
        self.lib.abpoa_reset(self.ab, self.abpt, qlen)
        self.n_seq = 0

    def align(self, codes: np.ndarray, count_cells: bool = True) -> tuple[ReadAlignment, abpoa_res_t]:
        codes = np.ascontiguousarray(codes, dtype=np.uint8)
        res = abpoa_res_t()
        res.n_cigar = 0
        res.graph_cigar = None
        res.n_aln_bases = res.n_matched_bases = 0
        rc = self.lib.abpoa_align_sequence_to_graph(self.ab, self.abpt, codes.ctypes.data_as(c_u8_p), len(codes), C.byref(res))
        if rc < 0:
            return ReadAlignment(aligned=False), res
        cig = np.ctypeslib.as_array(res.graph_cigar, shape=(res.n_cigar,)).copy() if res.n_cigar > 0 else np.zeros(0, dtype=np.uint64)
        out = ReadAlignment(True, int(res.best_score), cig, res.node_s, res.node_e, res.query_s, res.query_e)
        if count_cells:
            g = self.ab.contents.abg.contents
            abm = self.ab.contents.abm.contents
            rows = g.node_n - 1                  # DP rows 0 .. gn-2 (SURVEY 8d)
            beg = np.ctypeslib.as_array(abm.dp_beg, shape=(rows,))
            end = np.ctypeslib.as_array(abm.dp_end, shape=(rows,))
            out.cells = int((end.astype(np.int64) - beg + 1).sum())
            out.rows = rows
        return out, res

    def add(self, codes: np.ndarray, res: abpoa_res_t, tot_n_seq: int, weights: np.ndarray | None = None):
        codes = np.ascontiguousarray(codes, dtype=np.uint8)
        wp = None
        if weights is not None:
            weights = np.ascontiguousarray(weights, dtype=np.int32)
            wp = weights.ctypes.data_as(c_int_p)
        self.lib.abpoa_add_graph_alignment(self.ab, self.abpt, codes.ctypes.data_as(c_u8_p), wp, len(codes), None, res,
                                           self.n_seq, tot_n_seq, 1)
        if res.n_cigar > 0:
            capi.libc_free(res.graph_cigar)
        self.n_seq += 1
        self.ab.contents.abs.contents.n_seq = self.n_seq     # as pyabpoa.pyx:243 does

    def run_reads(self, reads: Sequence[np.ndarray], count_cells: bool = True, weights: Sequence[np.ndarray] | None = None) -> list[ReadAlignment]:
        """Progressive POA of one group, read by read, recording every alignment.
        weights: per-read base weights (the reference's -Q quality weights), used when cfg.use_qv."""
        self.reset(max((len(r) for r in reads), default=1024))
        out = []
        for i, r in enumerate(reads):
            a, res = self.align(r, count_cells)
            out.append(a)
            self.add(r, res, len(reads), weights[i] if weights is not None else None)
        return out

    # ---- whole-group call ---------------------------------------------------------------
    def msa(self, reads: Sequence[np.ndarray], names: Sequence[str] | None = None):
        """abpoa_msa(ab, abpt, n, names, lens, seqs, NULL, NULL) (reference src/abpoa_align.c:401)."""
        n = len(reads)
        arrs = [np.ascontiguousarray(r, dtype=np.uint8) for r in reads]
        lens = (C.c_int * n)(*[len(a) for a in arrs])
        seqs = (c_u8_p * n)(*[a.ctypes.data_as(c_u8_p) for a in arrs])
        nm = None
        if names is not None:
            nm = (C.c_char_p * n)(*[s.encode() for s in names])
        self.ab.contents.abs.contents.n_seq = 0
        self.lib.abpoa_msa(self.ab, self.abpt, n, nm, lens, seqs, None, None)
        self.n_seq = n

    # ---- results ---------------------------------------------------------------------------
    def generate(self):
        a = self.abpt.contents
        self.lib.abpoa_clean_msa_cons(self.ab)
        self.ab.contents.abg.contents.is_called_cons = 0
        if a.out_msa:
            self.lib.abpoa_generate_rc_msa(self.ab, self.abpt)
        elif a.out_cons:
            self.lib.abpoa_generate_consensus(self.ab, self.abpt)

    def consensus(self) -> list[np.ndarray]:
        abc = self.ab.contents.abc.contents
        return [np.ctypeslib.as_array(abc.cons_base[i], shape=(abc.cons_len[i],)).copy() for i in range(abc.n_cons)]

    def consensus_cov(self) -> list[np.ndarray]:
        abc = self.ab.contents.abc.contents
        return [np.ctypeslib.as_array(abc.cons_cov[i], shape=(abc.cons_len[i],)).copy() for i in range(abc.n_cons)]

    def msa_rows(self) -> list[np.ndarray]:
        abc = self.ab.contents.abc.contents
        if abc.msa_len <= 0:
            return []
        return [np.ctypeslib.as_array(abc.msa_base[i], shape=(abc.msa_len,)).copy() for i in range(abc.n_seq + abc.n_cons)]

    def graph_signature(self) -> dict:
        """Everything that decides the next DP: order, bases, edge lists+weights, remain, aligned sets."""
        g = self.ab.contents.abg.contents
        n = g.node_n
        sig = {
            "node_n": n,
            "index_to_node_id": np.ctypeslib.as_array(g.index_to_node_id, shape=(n,)).copy(),
            "node_id_to_index": np.ctypeslib.as_array(g.node_id_to_index, shape=(n,)).copy(),
        }
        if g.node_id_to_max_remain:
            sig["max_remain"] = np.ctypeslib.as_array(g.node_id_to_max_remain, shape=(n,)).copy()
        bases, ins, outs, alns, nread = [], [], [], [], []
        for i in range(n):
            nd = g.node[i]
            bases.append(nd.base)
            ins.append(tuple((nd.in_id[k], nd.in_edge_weight[k]) for k in range(nd.in_edge_n)))
            outs.append(tuple((nd.out_id[k], nd.out_edge_weight[k]) for k in range(nd.out_edge_n)))
            alns.append(tuple(nd.aligned_node_id[k] for k in range(nd.aligned_node_n)))
            nread.append((nd.n_read, nd.n_span_read))
        sig.update(bases=bases[2:], in_edges=ins, out_edges=outs, aligned=alns, n_read=nread)
        return sig


# ---------------------------------------------------------------------------------------------
# pyabpoa-compatible surface
# ---------------------------------------------------------------------------------------------
class msa_result:
    """Fields of pyabpoa.msa_result (python/pyabpoa.pyx:9-75)."""

    def __init__(self, n_seq, n_cons, clu_n_seq, clu_read_ids, cons_len, cons_seq, cons_cov, cons_qv, msa_len, msa_seq):
        self.n_seq, self.n_cons = n_seq, n_cons
        self.clu_n_seq, self.clu_read_ids = clu_n_seq, clu_read_ids
        self.cons_len, self.cons_seq, self.cons_cov, self.cons_qv = cons_len, cons_seq, cons_cov, cons_qv
        self.msa_len, self.msa_seq = msa_len, msa_seq

    def print_msa(self):
        if not self.msa_seq:
            return
        for i, s in enumerate(self.msa_seq):
            if i < self.n_seq:
                print(f">Seq_{i + 1}")
            else:
                cid = ""
                if self.n_cons > 1:
                    cid = f'_{i - self.n_seq + 1} {",".join(map(str, self.clu_read_ids[i - self.n_seq]))}'
                print(f">Consensus_sequence{cid}")
            print(s)


class msa_aligner:
    """pyabpoa.msa_aligner (python/pyabpoa.pyx:93-371) over the GPU library: same constructor arguments, same
    methods (msa, msa_align, msa_add, msa_output), same result fields.  One handle lives as long as the object,
    so msa_align / msa_add / msa_output build a graph incrementally exactly as the Cython class does."""

    def __init__(self, aln_mode="g", is_aa=False, match=2, mismatch=4, score_matrix="", gap_open1=4, gap_open2=24,
                 gap_ext1=2, gap_ext2=1, extra_b=10, extra_f=0.01, cons_algrm="HB", lib: PoaLibrary | None = None):
        modes = {"g": ABPOA_GLOBAL_MODE, "l": ABPOA_LOCAL_MODE, "e": ABPOA_EXTEND_MODE}
        if aln_mode not in modes:
            raise Exception(f"Unknown align mode: {aln_mode}")
        algs = {"HB": ABPOA_HB, "MF": ABPOA_MF}
        if cons_algrm.upper() not in algs:
            raise Exception(f"Unknown conseneus calling mode: {cons_algrm}")
        if isinstance(score_matrix, bytes):
            score_matrix = score_matrix.decode()
        self.m = 27 if is_aa else 5
        self._cfg = PoaConfig(align_mode=modes[aln_mode], m=self.m, match=match, mismatch=mismatch,
                              score_matrix=score_matrix or None, gap_open1=gap_open1, gap_open2=gap_open2,
                              gap_ext1=gap_ext1, gap_ext2=gap_ext2, wb=extra_b, wf=extra_f,
                              cons_algrm=algs[cons_algrm.upper()])
        self._s = PoaSession(self._cfg, lib)          # abpoa_init + parameters, freed with the object

    def __del__(self):
        s = getattr(self, "_s", None)
        if s is not None:
            s.close()

    def __bool__(self):
        return self._s.ab is not None

    # ---- helpers ------------------------------------------------------------------------------
    def _set_outputs(self, out_cons, out_msa, max_n_cons, min_freq, use_qv):
        if max_n_cons < 1 or max_n_cons > 2:
            raise Exception("Error: max number of consensus sequences should be 1 or 2.")
        a = self._s.abpt.contents
        a.out_cons, a.out_msa = int(bool(out_cons)), int(bool(out_msa))
        a.max_n_cons, a.min_freq = max_n_cons, min_freq
        a.use_qv = int(use_qv)
        self._s.lib.abpoa_post_set_para(self._s.abpt)

    def _add_sequences(self, seqs, qscores, exist_n, tot_n):
        """pyabpoa.pyx:176-209: align + fuse, read by read."""
        if qscores is not None and len(qscores) != len(seqs):
            raise ValueError("qscores must contain one entry per input sequence.")
        s = self._s
        for i, seq in enumerate(seqs):
            codes = encode(seq, self.m)
            weights = None
            if qscores is not None:
                if len(qscores[i]) != len(codes):
                    raise ValueError("Each qscore array must have the same length as its sequence.")
                weights = np.asarray([int(q) for q in qscores[i]], dtype=np.int32)
                if (weights < 0).any():
                    raise ValueError("Qscores must be non-negative integers.")
            _, res = s.align(codes, count_cells=False)
            wp = weights.ctypes.data_as(c_int_p) if weights is not None else None
            s.lib.abpoa_add_graph_alignment(s.ab, s.abpt, codes.ctypes.data_as(c_u8_p), wp, len(codes), None, res, exist_n + i, tot_n, 1)
            if res.n_cigar > 0:
                capi.libc_free(res.graph_cigar)

    def _result(self, tot_n):
        s = self._s
        a = s.abpt.contents
        if a.out_msa:
            s.lib.abpoa_generate_rc_msa(s.ab, s.abpt)
        elif a.out_cons:
            s.lib.abpoa_generate_consensus(s.ab, s.abpt)
        abc = s.ab.contents.abc.contents
        n_cons = abc.n_cons
        cons = s.consensus()
        covs = s.consensus_cov()
        clu_n = [abc.clu_n_seq[i] for i in range(n_cons)]
        clu_ids = [[abc.clu_read_ids[i][j] for j in range(clu_n[i])] for i in range(n_cons)]
        qv = ["".join(chr(abc.cons_phred_score[i][j]) for j in range(abc.cons_len[i])) if abc.cons_phred_score else "" for i in range(n_cons)]
        rows = s.msa_rows()
        return msa_result(tot_n, n_cons, clu_n, clu_ids, [len(c) for c in cons], [decode(c, self.m) for c in cons],
                          [list(map(int, c)) for c in covs], qv, int(abc.msa_len), [decode(r, self.m) for r in rows])

    # ---- pyabpoa methods -------------------------------------------------------------------------
    def msa_align(self, seqs, out_cons, out_msa, max_n_cons=1, min_freq=0.25, incr_fn=b"", qscores=None):
        if incr_fn:
            raise NotImplementedError("restoring a graph from a GFA / MSA file is outside the hot-path scope")
        self._set_outputs(out_cons, out_msa, max_n_cons, min_freq, qscores is not None)
        s = self._s
        s.lib.abpoa_reset(s.ab, s.abpt, len(seqs[0]))
        abs_ = s.ab.contents.abs.contents
        abs_.n_seq += len(seqs)
        self._add_sequences(seqs, qscores, 0, len(seqs))
        return self

    def msa_add(self, new_seqs, qscores=None):
        if isinstance(new_seqs, str):
            raise TypeError('Expected a list of strings. If you want to add a single sequence, pass it as a list: ["ACGT..."]')
        s = self._s
        abs_ = s.ab.contents.abs.contents
        exist_n = abs_.n_seq
        if exist_n == 0:
            raise Exception("Error: no existing sequences in the graph. Please run msa() or msa_align() first.")
        abs_.n_seq += len(new_seqs)
        if qscores is not None:
            s.abpt.contents.use_qv = 1
        self._add_sequences(new_seqs, qscores, exist_n, exist_n + len(new_seqs))
        return self

    def msa_output(self):
        return self._result(self._s.ab.contents.abs.contents.n_seq)

    def msa(self, seqs, out_cons, out_msa, max_n_cons=1, min_freq=0.25, out_pog=b"", incr_fn=b"", qscores=None):
        if out_pog:
            raise NotImplementedError("graph plotting is outside the hot-path scope")
        self.msa_align(seqs, out_cons, out_msa, max_n_cons, min_freq, incr_fn, qscores)
        return self._result(len(seqs))
