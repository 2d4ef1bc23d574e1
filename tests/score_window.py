"""Scoring and shape points on both sides of every threshold that decides the score width (shared by
tests/test_score_window.py's CPU and GPU parts).

Thresholds (what each point sits next to):
  poa_p16_ok (poa_flat.c)    qlen * max_mat <= 28000, 2 * w * e + oe <= 12000, e <= 100, mismatch <= 1000: packed kernel admitted
  packed-kernel guard        a row maximum below -14000 / above 29000, or max_band * e + oe > 15000: POA_ST_RANGE, redo
  poa_score_bits             the reference's int16 / int32 switch (src/abpoa_align_simd.c:1293-1303); also sets pn, the
                             vector width that rounds the band's left edge
  the reference's inf_min    INT16_MIN + max(min_mis, oe1, oe2) + 512 * max(e1, e2) (src/abpoa_align_simd.c:1295): its int16
                             "minus infinity", which with large gap extensions lies above real scores

Every point is built from fixed seeds.  `reference_sound` says where the reference's int16 floor cannot have touched a real
score, i.e. where the reference's result is the true optimum and the library must reproduce it exactly.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

from abpoa_b200 import synth
from abpoa_b200.aligner import PoaConfig
from abpoa_b200.capi import ABPOA_LINEAR_GAP, ABPOA_LOCAL_MODE
from planes import ORACLE_NINF, score_bits

# A real (oracle-finite) cell closer than this to the reference's inf_min makes a point unsound.  Found from the sweep
# below: every point whose smallest headroom (finite cell - inf_min) exceeds it agrees with the oracle, the closest at
# 2050; every disagreeing point has real cells below inf_min (headroom -2338 and lower), and between -144 and 1024 the
# reference may still agree.  1024 leaves room on the sound side for the reference's -inf cells, which start at inf_min
# and move by whole scores per row (up by a match on a diagonal), so a real cell that close may lose to one of them.
SOUND_MARGIN = 1024


def affine(e, **kw):
    return dict(gap_open1=2 * e, gap_ext1=e, gap_open2=0, gap_ext2=0, **kw)


def convex(e, **kw):
    return dict(gap_open1=2 * e, gap_ext1=e, gap_open2=12 * e, gap_ext2=max(1, e // 2), **kw)


def ragged600(seed=950):
    """6 reads of 600 bp, reads 1-2 cut to 40 bp: long end gaps, real scores far below zero."""
    short = synth.make_group(seed, 6, 600, 0.05)
    return [short[0]] + [np.ascontiguousarray(r[:40]) for r in short[1:3]] + list(short[3:])


def group(seed, n, length, err=0.05):
    return lambda: synth.make_group(seed, n, length, err)


def with_last(seed, n, length, last_len, err=0.05):
    """n - 1 reads of `length`, then one of exactly `last_len` bases (the read whose qlen sits on the edge).  The reads are
    drawn longer than needed and cut: synth.make_group's indels make a read's length differ from the template's."""
    def make():
        g = synth.make_group(seed, n, max(length, last_len) + 200, err)
        out = [np.ascontiguousarray(r[:length]) for r in g[:-1]] + [np.ascontiguousarray(g[-1][:last_len])]
        assert [len(r) for r in out] == [length] * (n - 1) + [last_len]
        return out
    return make


# (name, PoaConfig kwargs, reads builder, which side: "in" / "out" of the edge named first in `name`)
POINTS = [
    # poa_p16_ok: qlen * max_mat = 28000 / 28020 (one query base more)
    ("p16_qlen_28000", dict(match=20, mismatch=40, **affine(20)), with_last(301, 4, 1300, 1400), "in"),
    ("p16_qlen_28020", dict(match=20, mismatch=40, **affine(20)), with_last(301, 4, 1300, 1401), "out"),
    # poa_p16_ok: 2 * w * e + oe = 12000 / 12001 (w = wb with wf = 0)
    ("p16_band_12000", dict(gap_open1=993, gap_ext1=3, gap_open2=0, gap_ext2=0, wb=1834, wf=0.0), group(302, 5, 500), "in"),
    ("p16_band_12001", dict(gap_open1=994, gap_ext1=3, gap_open2=0, gap_ext2=0, wb=1834, wf=0.0), group(302, 5, 500), "out"),
    # poa_p16_ok: e = 100 / 101 (oe = 300 / 303)
    ("p16_e_100", affine(100), group(303, 5, 400), "in"),
    ("p16_e_101", affine(101), group(303, 5, 400), "out"),
    # poa_p16_ok: mismatch = 1000 / 1001
    ("p16_mis_1000", dict(mismatch=1000), group(304, 5, 500, 0.08), "in"),
    ("p16_mis_1001", dict(mismatch=1001), group(304, 5, 500, 0.08), "out"),
    # packed-kernel guard: global row maxima around -14000 (40 bp reads against a 600-node graph: -13920 at e = 25,
    # -14480 at e = 26)
    ("guard_lo_e25", affine(25), ragged600, "in"),
    ("guard_lo_e26", affine(26), ragged600, "out"),
    # packed-kernel guard: local maximum near +28000 (the highest qlen * max_mat poa_p16_ok admits, so the +29000 side of
    # the guard cannot be reached by an admitted job)
    ("guard_hi_local", dict(match=20, mismatch=40, align_mode=ABPOA_LOCAL_MODE, **affine(20)), with_last(305, 3, 1400, 1400, 0.01), "in"),
    # packed-kernel guard: max_band * e + oe around 15000 (a read twice the graph's length makes rows ~910 cells wide:
    # 14592 at e = 16, 15504 at e = 17)
    ("guard_band_e16", dict(wb=100, wf=0.0, **affine(16)), lambda: synth.make_group(306, 3, 700, 0.05) + [synth.make_group(307, 1, 1400, 0.05)[0]], "in"),
    ("guard_band_e17", dict(wb=100, wf=0.0, **affine(17)), lambda: synth.make_group(306, 3, 700, 0.05) + [synth.make_group(307, 1, 1400, 0.05)[0]], "out"),
    # poa_score_bits: len * e1 + o1 against 32767 - min_mis - oe1 - oe2, +-1 on qlen (affine: 1633 / 1634)
    ("bits_affine_1633", affine(20), with_last(308, 3, 1000, 1633), "in"),
    ("bits_affine_1634", affine(20), with_last(308, 3, 1000, 1634), "out"),
    # ... banded linear gaps (the "lgx" path, where pn decides the vector-granular band): 1637 / 1638
    ("bits_linear_1637", dict(gap_open1=0, gap_ext1=20, gap_open2=0, gap_ext2=0), with_last(309, 3, 1000, 1637), "in"),
    ("bits_linear_1638", dict(gap_open1=0, gap_ext1=20, gap_open2=0, gap_ext2=0), with_last(309, 3, 1000, 1638), "out"),
]
# the reference's inf_min region: affine and convex, e = 24 .. 64, ragged groups
for _e in (24, 28, 30, 32, 36, 40, 64):
    POINTS.append((f"infmin_affine_e{_e}", affine(_e), ragged600, "in"))
for _e in (24, 32, 40, 64):
    POINTS.append((f"infmin_convex_e{_e}", convex(_e), ragged600, "in"))
POINTS.append(("infmin_affine_e64_g400", affine(64), group(900, 6, 400, 0.10), "in"))
POINTS.append(("infmin_convex_e64_g400", convex(64), group(900, 6, 400, 0.10), "in"))

# where the reference's int16 floor is known to have won over a real score (differs from the true optimum, or exits)
REFERENCE_WRONG = ["infmin_affine_e32", "infmin_affine_e36", "infmin_affine_e40", "infmin_affine_e64_g400", "infmin_convex_e64_g400"]

BY_NAME = {p[0]: p for p in POINTS}


def guard_margin(name: str, cfg: PoaConfig, alns: list[Aln]) -> tuple[int, int, int] | None:
    """(value, low, high): the quantity a guard point's name says it sits next to, and the range it must lie in."""
    packed = [a for a in alns if a.packed]
    if name.startswith("guard_lo_"):
        v = min(a.min_row_max for a in packed)
        return (v, -14000, -13000) if BY_NAME[name][3] == "in" else (v, -15000, -14001)
    if name.startswith("guard_band_"):
        e = max(cfg.gap_ext1, cfg.gap_ext2); oe = max(cfg.gap_open1 + cfg.gap_ext1, cfg.gap_open2 + cfg.gap_ext2)
        v = max(a.max_band * e + oe for a in packed)
        return (v, 14000, 15000) if BY_NAME[name][3] == "in" else (v, 15001, 16000)
    if name.startswith("guard_hi_"):
        return (max(a.max_row_max for a in packed), 26000, 28000)
    return None


def point(name):
    _, kw, make, _ = BY_NAME[name]
    return PoaConfig(**kw), make()


def inf_min(cfg: PoaConfig) -> int:
    """The reference's int16 minus infinity for cfg (src/abpoa_align_simd.c:1295); mismatch is min_mis with the default matrix."""
    oe1, oe2 = cfg.gap_open1 + cfg.gap_ext1, cfg.gap_open2 + cfg.gap_ext2
    return -32768 + max(cfg.mismatch, oe1, oe2) + 512 * max(cfg.gap_ext1, cfg.gap_ext2)


@dataclass
class Aln:
    """What the oracle shows about one alignment of a point, and what the library's thresholds make of it."""
    qlen: int
    n_rows: int
    bits: int                 # the reference's score width (poa_score_bits)
    packed: bool              # admitted to the packed int16x2 kernel (packed_admits)
    min_row_max: int          # lowest row maximum (rows > 0) ...
    max_row_max: int          # ... and highest: what the packed kernel's guard watches
    max_band: int             # widest computed row (cells)
    min_cell: int             # lowest finite cell of any plane
    guard: bool               # the packed kernel's run-time guard fires (guard_fires)


def packed_admits(abpt, qlen: int, n_rows: int) -> bool:
    """use_p16_for (poa_cuda.cu) with poa_p16_ok (poa_flat.c) in Python: may the packed int16x2 kernel take this job?"""
    a = abpt.contents
    if a.gap_mode == ABPOA_LINEAR_GAP and a.align_mode != ABPOA_LOCAL_MODE and a.wb >= 0:
        return False                                           # banded linear gaps: the generic kernel's "lgx" rows
    oe1, oe2 = a.gap_open1 + a.gap_ext1, a.gap_open2 + a.gap_ext2
    emax, oemax = max(a.gap_ext1, a.gap_ext2), max(oe1, oe2)
    if a.max_mat <= 0 or qlen * a.max_mat > 28000:
        return False
    if a.min_mis > 1000 or a.max_mat > 1000 or oemax > 1000 or emax > 100:
        return False
    if a.wb < 0:
        return a.align_mode == ABPOA_LOCAL_MODE or max(qlen, n_rows) * a.gap_ext1 + a.gap_open1 <= 26000
    w = a.wb + int(np.float32(a.wf) * np.float32(qlen))          # the C float product of poa_band_halfwidth
    return 2 * w * emax + oemax <= 12000


def guard_fires(abpt, min_row_max: int, max_row_max: int, max_band: int) -> bool:
    """The packed kernel's run-time guard (end of p16_run_job in poa_kernels.cu): POA_ST_RANGE when a row maximum leaves
    [-14000, 29000] or, banded outside local mode, max_band * e + oe > 15000.  (Its third test, best score <= NEGP + 2000,
    implies the first.)"""
    a = abpt.contents
    if min_row_max < -14000 or max_row_max > 29000:
        return True
    emax, oemax = max(a.gap_ext1, a.gap_ext2), max(a.gap_open1 + a.gap_ext1, a.gap_open2 + a.gap_ext2)
    return a.wb >= 0 and a.align_mode != ABPOA_LOCAL_MODE and max_band * emax + oemax > 15000


def profile(cfg: PoaConfig, reads, lib) -> list[Aln]:
    """Progressive alignment of `reads` by the oracle on `lib`'s host graph; one Aln per aligned read."""
    from abpoa_b200.aligner import PoaSession
    from oracle_binding import oracle_align
    out = []
    with PoaSession(cfg, lib) as s:
        s.reset(max(len(r) for r in reads))
        for r in reads:
            rows = {}

            def cb(user, row, beg, end, h, e1, e2, f1, f2):
                wd = end - beg + 1
                if wd > 0:
                    rows[row] = (wd, [np.ctypeslib.as_array(p, shape=(wd,)).copy() for p in (h, e1, e2, f1, f2) if p])
            n_rows = s.ab.contents.abg.contents.node_n
            o, res = oracle_align(s, r, row_cb=cb)
            if o.aligned:
                maxima = [int(pl[0].max()) for row, (wd, pl) in rows.items() if row > 0]
                cells = np.concatenate([p for wd, pl in rows.values() for p in pl])
                lo, hi, band = min(maxima), max(maxima), max(wd for wd, pl in rows.values())
                out.append(Aln(len(r), n_rows, score_bits(s.abpt, len(r), n_rows), packed_admits(s.abpt, len(r), n_rows), lo, hi, band,
                               int(cells[cells > ORACLE_NINF // 2].min()), guard_fires(s.abpt, lo, hi, band)))
            s.add(r, res, len(reads))
    return out


def edge_side(name: str, alns: list[Aln]) -> str | None:
    """Which side of its edge a point actually sits on ("in" / "out"), from what the oracle shows; None for inf_min points.
      p16_*   the edge read (the last one) is admitted to the packed kernel
      guard_* no admitted alignment makes the packed kernel's guard fire
      bits_*  the edge read gets the reference's int16 width"""
    if name.startswith("p16_"):
        return "in" if alns[-1].packed else "out"
    if name.startswith("guard_"):
        return "out" if any(a.packed and a.guard for a in alns) else "in"
    if name.startswith("bits_"):
        return "in" if alns[-1].bits == 16 else "out"
    return None


def headroom(cfg: PoaConfig, alns: list[Aln]) -> int | None:
    """Smallest (finite oracle cell - inf_min) over every alignment the reference runs in int16; None if it runs none in int16."""
    h = [a.min_cell - inf_min(cfg) for a in alns if a.bits == 16]
    return min(h) if h else None


def reference_sound(cfg: PoaConfig, alns: list[Aln]) -> bool:
    """The reference takes int32 for every alignment, or no finite cell in a computed band comes within SOUND_MARGIN of its
    int16 inf_min: then the reference's result is the true optimum."""
    h = headroom(cfg, alns)
    return h is None or h > SOUND_MARGIN
