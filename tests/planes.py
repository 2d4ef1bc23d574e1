"""Cell-by-cell comparison of the DP planes a CUDA kernel stored with the scalar oracle's (oracle/poa_oracle.c).

The product aligns read by read through abpoa.h on the GPU; a second session on the same graph gets every alignment
from the oracle, whose row callback hands over each computed row in 32 bits with a true minus infinity.  After each
alignment the whole DP state of the product is fetched in one copy (poa_debug_fetch_planes) and compared row by row:

  band         (beg, end) of every row the oracle computed
  arg-max      first / last column of the row maximum (rowinfo.left / right), which the band of later rows follows;
               compared where the oracle computes it (banded, or not global mode) and the row has a finite maximum
  finite cell  every plane cell the oracle holds a finite value for: exact equality
  -inf cell    every cell the oracle holds minus infinity for: at or below the floor of the kernel that ran (FLOOR)

No tolerance: any exception is a named rule below, with the backtrace code that never reads the cell.

poa_debug_last_run tells which kernel produced the accepted result (after any redo), so a test written for one kernel
cannot pass on another one.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field

import numpy as np

from abpoa_b200 import capi
from abpoa_b200.aligner import PoaSession, ReadAlignment
from abpoa_b200.capi import ABPOA_GLOBAL_MODE, ABPOA_LINEAR_GAP, ABPOA_LOCAL_MODE, abpoa_res_t, c_u8_p

PLANE_NAMES = ("H", "E1", "E2", "F1", "F2")       # the oracle's plane order (row_cb arguments)
KERNELS = {15: "packed", 16: "generic-int16", 32: "generic-int32"}

# Minus infinity as each kernel stores it.  Cells the oracle holds -inf for may sit a little above the rail: the kernels
# add scores to -inf operands (a match on the diagonal of a -inf cell) and clamp only from below; the suite sees them
# within a few units of it.  For the packed kernel the margin also separates them from real cells: a job it accepts has
# every row maximum >= -14000 and max_band * e + oe <= 15000 (its run-time guard), which keeps real cells above about
# -14000 - 15000 = -29000 = NEGP + INF_MARGIN.  The generic int16 kernel widens -32768 on load, the int32 one uses
# POA_NEG32 = -2^29.
NEGP = -30000
POA_NEG32 = -(1 << 29)
INF_MARGIN = 1000
FLOOR = {15: NEGP + INF_MARGIN, 16: -32768 + INF_MARGIN, 32: POA_NEG32 // 2}
ORACLE_NINF = (-(1 << 31)) // 4                    # NINF of poa_oracle.c; addinf() keeps everything <= NINF / 2 at -inf


def _bind(lib):
    d = lib.dll
    if not getattr(d, "_planes_bound", False):
        d.poa_debug_fetch_planes.restype = C.c_int64
        d.poa_debug_fetch_planes.argtypes = [capi.abpoa_t_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64]
        d.poa_debug_last_run.restype = C.c_int
        d.poa_debug_last_run.argtypes = [capi.abpoa_t_p, C.c_void_p]
        d.poa_debug_chain_replay.restype = C.c_int64
        d.poa_debug_chain_replay.argtypes = [capi.abpoa_t_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                             C.c_int64, C.c_void_p, C.c_int64, C.c_void_p]
        d._planes_bound = True
    return d


@dataclass
class RunInfo:
    """How one alignment ran (poa_debug_last_run), plus what its planes showed."""
    kernel: int
    lean: bool
    tma: bool
    ring_rows: int
    ring_cells: int
    n_rows: int
    n_planes: int
    retries: int
    widest_groups: int = 0         # 8-cell groups of the widest computed row (a ring slot holds ring_cells / 8)
    min_finite: int = 0            # lowest finite oracle cell (how close real scores came to the kernel's floor)
    max_inf: int = ORACLE_NINF     # highest product value in a cell the oracle holds -inf for
    min_row_max: int = 1 << 30     # lowest and highest oracle row maximum (rows > 0) and widest row (cells):
    max_row_max: int = -(1 << 30)  # what the packed kernel's run-time guard watches
    max_band: int = 0

    @property
    def name(self):
        return KERNELS.get(self.kernel, str(self.kernel))


def last_run(session: PoaSession) -> RunInfo:
    out = np.zeros(8, dtype=np.int32)
    assert _bind(session.lib).poa_debug_last_run(session.ab, out.ctypes.data) == 0, "no alignment on this handle yet"
    return RunInfo(int(out[0]), bool(out[1]), bool(out[2]), int(out[3]), int(out[4]), int(out[5]), int(out[6]), int(out[7]))


def fetch_planes(session: PoaSession, info: RunInfo):
    """(rowinfo [n_rows, 4], rowoff [n_rows], slab) of the last alignment, one copy each."""
    d = _bind(session.lib)
    rowinfo = np.zeros((info.n_rows, 4), dtype=np.int32)
    rowoff = np.zeros(info.n_rows, dtype=np.uint32)
    need = d.poa_debug_fetch_planes(session.ab, None, None, None, 0)
    assert need >= 0, "poa_debug_fetch_planes: no single alignment to fetch"
    slab = np.zeros(max(int(need), 16), dtype=np.uint8)
    got = d.poa_debug_fetch_planes(session.ab, rowinfo.ctypes.data, rowoff.ctypes.data, slab.ctypes.data, len(slab))
    assert got == need
    return rowinfo, rowoff, slab[:need].view(np.int32 if info.kernel == 32 else np.int16)


@dataclass
class ChainReplay:
    """The last alignment replayed on the chain engine's job function (poa_debug_chain_replay): compact row layout
    (H, E1 (, E2)), then every row's F planes and insertion-step decision bytes rebuilt by the backtrace's recompute."""
    status: int
    best_score: int
    ends: tuple                    # (node_s, node_e, query_s, query_e), as abpoa_res_t holds them
    n_ops: int
    cells: int
    max_band: int
    plane_units_used: int
    ring_rows: int
    ring_cells: int
    buf_cells: int                 # decision-byte buffer of the recompute (cells)
    windows: int                   # fb_recompute calls of the dump, all rows
    max_windows: int               # ... of the row with the most
    cigar: np.ndarray              # graph-CIGAR (node ids)
    rowinfo: np.ndarray            # [n_rows, 4] beg, end, left, right
    rowoff: np.ndarray             # [n_rows] slab offset of each row (8-cell units)
    slab: np.ndarray               # int16: H, E1 (, E2) of each row, ngrp * 8 cells each
    fslab: np.ndarray              # int16: F1 (, F2) of each row at the same offsets
    fbits: np.ndarray              # uint8: decision byte of cell j of a row at rowoff * 8 + j - 8 (beg >> 3)


def chain_replay(session: PoaSession, info: RunInfo, qlen: int, ring_rows: int = 0, ring_cells: int = 0, buf_cells: int = 0) -> ChainReplay:
    """Replay the last alignment of `session` with ring geometry (ring_rows, ring_cells) (0, 0: the chain's pick) and a
    recompute buffer of buf_cells cells (0: the chain's, the ring; -1: a whole row)."""
    d = _bind(session.lib)
    out = np.zeros(16, dtype=np.int64)
    need = d.poa_debug_chain_replay(session.ab, ring_rows, ring_cells, buf_cells, None, None, None, None, None, 0, None, 0, out.ctypes.data)
    assert need > 0, f"poa_debug_chain_replay refused the last alignment ({need})"
    rowinfo = np.zeros((info.n_rows, 4), dtype=np.int32)
    rowoff = np.zeros(info.n_rows, dtype=np.uint32)
    slab = np.zeros(need // 2, dtype=np.int16)
    fslab = np.zeros(need // 2, dtype=np.int16)
    fbits = np.zeros(need // 2, dtype=np.uint8)
    cig = np.zeros(qlen + info.n_rows + 8, dtype=np.uint64)
    used = d.poa_debug_chain_replay(session.ab, ring_rows, ring_cells, buf_cells, rowinfo.ctypes.data, rowoff.ctypes.data, slab.ctypes.data,
                                    fslab.ctypes.data, fbits.ctypes.data, need, cig.ctypes.data, len(cig), out.ctypes.data)
    assert used >= 0, f"poa_debug_chain_replay: geometry ({ring_rows}, {ring_cells}) / buffer {buf_cells} rejected ({used})"
    o = [int(x) for x in out]
    return ChainReplay(o[0], o[1], (o[4], o[2], o[5], o[3]), o[6], o[7], o[8], o[9], o[10], o[11], o[12], o[13], o[14], cig[:o[6]].copy(),
                       rowinfo, rowoff, slab, fslab, fbits)


def decision_bytes(h: np.ndarray, fs: list, gaps: list) -> np.ndarray:
    """The insertion-step decision byte of every cell of one row's band (RowLayout in poa_kernels.cu) from the row's H and F
    planes over the band: for F plane k with penalties (oe_k, e_k), bits 3k .. 3k+2 are
      FB_A  H[j] == F_k[j],   FB_B  H[j-1] - oe_k == F_k[j],   FB_C  F_k[j-1] - e_k == F_k[j]
    with B and C 0 at the band's first cell.  In int64, so no value wraps."""
    h = np.asarray(h, dtype=np.int64)
    out = np.zeros(len(h), dtype=np.uint8)
    for k, (f, (oe, e)) in enumerate(zip(fs, gaps)):
        f = np.asarray(f, dtype=np.int64)
        a = h == f
        b = np.zeros(len(h), dtype=bool); c = np.zeros(len(h), dtype=bool)
        b[1:] = h[:-1] - oe == f[1:]
        c[1:] = f[:-1] - e == f[1:]
        out |= ((a * 1 | b * 2 | c * 4) << (3 * k)).astype(np.uint8)
    return out


def oracle_rows_of(align):
    """Run `align(row_cb)` and collect the oracle's rows: {row: (beg, end, [H, E1, E2, F1, F2] or None each)}."""
    rows = {}

    def cb(user, row, beg, end, h, e1, e2, f1, f2):
        wd = end - beg + 1
        rows[row] = (beg, end, [np.ctypeslib.as_array(p, shape=(wd,)).copy() if p and wd > 0 else None for p in (h, e1, e2, f1, f2)])
    out = align(cb)
    return out, rows


def score_bits(abpt, qlen: int, n_rows: int) -> int:
    """The reference's int16 / int32 choice (poa_score_bits in poa_flat.c, reference src/abpoa_align_simd.c:1293-1303)."""
    a = abpt.contents
    max_score = max(qlen * a.max_mat, max(qlen, n_rows) * a.gap_ext1 + a.gap_open1)
    return 16 if max_score <= 32767 - a.min_mis - (a.gap_open1 + a.gap_ext1) - (a.gap_open2 + a.gap_ext2) else 32


# product plane k holds oracle plane PLANE_ORDER[n_planes][k] (five-plane layout of each gap mode)
PLANE_ORDER = {1: (0,), 3: (0, 1, 3), 5: (0, 1, 2, 3, 4)}


def compare_planes(session: PoaSession, rows: dict, info: RunInfo, qlen: int, tag: str = "", order=None, planes=None) -> list[str]:
    """Every rule of the module docstring on the last alignment of `session`; returns the violations (at most one per
    row and plane, each naming row, plane and column), [] when the planes match.
    order: the oracle plane (index into PLANE_NAMES) of each plane a row stores, in storage order; default PLANE_ORDER of
    the kernel's plane count.  planes: (rowinfo, rowoff, slab) to check instead of fetch_planes(session, info), e.g. the
    compact slab (H, E1 (, E2)) or the recomputed F slab (F1 (, F2)) of the chain's job function (ChainReplay)."""
    cfg = session.cfg
    # storage granule of a row (log2 cells): the 8-cell group, except banded linear-gap rows outside local mode on the
    # generic kernel ("lgx"), which are stored in whole reference vectors of pn = 16 / 8 cells around the band
    lgx = info.kernel != 15 and session.abpt.contents.gap_mode == ABPOA_LINEAR_GAP and cfg.align_mode != ABPOA_LOCAL_MODE and cfg.wb >= 0
    xs = (4 if score_bits(session.abpt, qlen, info.n_rows) == 16 else 3) if lgx else 3
    rowinfo, rowoff, slab = fetch_planes(session, info) if planes is None else planes
    floor = FLOOR[info.kernel]
    order = PLANE_ORDER[info.n_planes] if order is None else tuple(order)
    n_planes = len(order)
    with_argmax = cfg.wb >= 0 or cfg.align_mode != ABPOA_GLOBAL_MODE
    bad = []
    for row in sorted(rows):
        beg, end, pl = rows[row]
        pb, pe, pleft, pright = (int(x) for x in rowinfo[row])
        if (pb, pe) != (beg, end):
            bad.append(f"{tag} row {row}: band ({pb},{pe}), oracle ({beg},{end})")
            continue
        if end < beg:
            continue
        h = pl[0]
        info.max_band = max(info.max_band, end - beg + 1)
        if row > 0:
            info.min_row_max = min(info.min_row_max, int(h.max()))
            info.max_row_max = max(info.max_row_max, int(h.max()))
        # row 0 is no arg-max row: its successors get the fixed hint column 1 (the oracle's first-row block), which the
        # product keeps as left = right = 0
        if row > 0 and with_argmax and h.max() > ORACLE_NINF // 2:
            arg = np.flatnonzero(h == h.max())
            want = (beg + int(arg[0]), beg + int(arg[-1]))
            if (pleft, pright) != want:
                bad.append(f"{tag} row {row}: arg-max (left, right) ({pleft},{pright}), oracle {want}")
        g0 = ((beg >> xs) << xs) >> 3
        ngrp = (((((end >> xs) + 1) << xs) - 1) >> 3) - g0 + 1
        info.widest_groups = max(info.widest_groups, ngrp)
        base = int(rowoff[row]) * 8
        stored = slab[base: base + n_planes * ngrp * 8].astype(np.int64).reshape(n_planes, ngrp * 8)
        lo = beg - g0 * 8
        for k, pi in enumerate(order):
            want = pl[pi]
            if want is None:
                continue
            got = stored[k, lo: lo + end - beg + 1]
            finite = want > ORACLE_NINF // 2
            if finite.any():
                info.min_finite = min(info.min_finite, int(want[finite].min()))
            if (~finite).any():
                info.max_inf = max(info.max_inf, int(got[~finite].max()))
            diff = np.flatnonzero((finite & (got != want)) | (~finite & (got > floor)))
            if len(diff):
                j = int(diff[0])
                w = int(want[j]) if finite[j] else "-inf"
                bad.append(f"{tag} row {row} plane {PLANE_NAMES[pi]} column {beg + j}: {info.name} kernel {int(got[j])}, oracle {w} "
                           f"(band {beg}..{end}, {len(diff)} cells differ)")
    return bad


@dataclass
class PlanesRun:
    runs: list = field(default_factory=list)        # RunInfo per aligned read
    alns: list = field(default_factory=list)        # product ReadAlignment per read
    oracle: list = field(default_factory=list)      # oracle ReadAlignment per read


def _align_sub(session, r, beg_id, end_id):
    d = session.lib.dll
    res = abpoa_res_t()
    rc = d.abpoa_align_sequence_to_subgraph(session.ab, session.abpt, beg_id, end_id, r.ctypes.data_as(c_u8_p), len(r), C.byref(res))
    if rc < 0:
        return ReadAlignment(aligned=False), res
    cig = np.ctypeslib.as_array(res.graph_cigar, shape=(res.n_cigar,)).copy() if res.n_cigar > 0 else np.zeros(0, dtype=np.uint64)
    return ReadAlignment(True, int(res.best_score), cig, res.node_s, res.node_e, res.query_s, res.query_e), res


def _add_sub(session, r, res, beg_id, end_id, i, n):
    session.lib.dll.abpoa_add_subgraph_alignment(session.ab, session.abpt, beg_id, end_id, r.ctypes.data_as(c_u8_p), None, len(r), None,
                                                 res, i, n, 0)
    if res.n_cigar > 0:
        capi.libc_free(res.graph_cigar)


def run_planes(cfg, reads, lib=None, windows=None, tag: str = "", check=None, after=None) -> PlanesRun:
    """Progressive alignment of `reads` on the GPU with every DP plane compared to the oracle's after every read.
    windows: per read (inc_beg, inc_end) node-id windows for sub-graph alignment (abpoa_subgraph_nodes), or None.
    check(i, RunInfo): called after every aligned read (assert the kernel variant here).
    after(session, oracle rows, RunInfo, oracle ReadAlignment): called after check, before the read joins the graph (more
    checks on the same alignment, e.g. a replay of it with chain_replay).
    Raises AssertionError naming the first read / row / plane / column that differs."""
    from oracle_binding import oracle_align
    lib = lib or capi.product()
    reads = [np.ascontiguousarray(r, dtype=np.uint8) for r in reads]
    out = PlanesRun()
    with PoaSession(cfg, lib) as gpu, PoaSession(cfg, lib) as cpu:       # cpu: host graph only, alignments from the oracle
        gpu.reset(max(len(r) for r in reads)); cpu.reset(max(len(r) for r in reads))
        if windows is not None:
            gpu.ab.contents.abs.contents.n_seq = cpu.ab.contents.abs.contents.n_seq = len(reads)
        for i, r in enumerate(reads):
            t = f"{tag} read {i} (qlen {len(r)})"
            eb, ee = C.c_int(0), C.c_int(1)
            if windows is not None and i:
                lib.dll.abpoa_subgraph_nodes(gpu.ab, gpu.abpt, windows[i][0], windows[i][1], C.byref(eb), C.byref(ee))
            if windows is None:
                (o, ores), rows = oracle_rows_of(lambda cb: oracle_align(cpu, r, row_cb=cb))
                a, res = gpu.align(r, count_cells=False)
            else:
                (o, ores), rows = oracle_rows_of(lambda cb: oracle_align(cpu, r, row_cb=cb, beg_node_id=eb.value, end_node_id=ee.value))
                a, res = _align_sub(gpu, r, eb.value, ee.value)
            out.alns.append(a); out.oracle.append(o)
            assert a.aligned == o.aligned, t
            if a.aligned:
                info = last_run(gpu)
                bad = compare_planes(gpu, rows, info, len(r), t)
                assert not bad, f"DP planes differ from the oracle ({len(bad)} rows / planes):\n  " + "\n  ".join(bad[:12])
                assert a.best_score == o.best_score, f"{t}: score {a.best_score}, oracle {o.best_score}"
                assert np.array_equal(a.cigar, o.cigar), f"{t}: graph-CIGAR differs from the oracle"
                assert (a.node_s, a.node_e, a.query_s, a.query_e) == (o.node_s, o.node_e, o.query_s, o.query_e), f"{t}: end points"
                out.runs.append(info)
                if check is not None:
                    check(i, info)
                if after is not None:
                    after(gpu, rows, info, o)
            if windows is None:
                gpu.add(r, res, len(reads)); cpu.add(r, ores, len(reads))
            else:
                _add_sub(gpu, r, res, eb.value, ee.value, i, len(reads)); _add_sub(cpu, r, ores, eb.value, ee.value, i, len(reads))
    return out
