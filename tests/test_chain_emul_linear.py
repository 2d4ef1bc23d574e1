"""CPU suite: the device graph code with linear gaps (-O 0), and the chain's plane estimate for linear-gap rows.

1. tests/test_chain_emul.py's drive(): the device-side graph code (poa_chain.cuh) compiled for the host, read by read next
   to the product's host graph layer; every next job blob must equal poa_blob_fill's byte for byte, header included, so
   also its vector width pn.  Inputs: the banded linear-gap sweep's shapes with default and narrow (wb / wf) bands, amino
   acids, and the score-window points whose last read makes the reference pick 16 lanes (1637 bases) or 8 lanes (1638).
2. On the scalar oracle: a linear-gap row is stored in whole vectors of pn cells around its band, up to 2 (pn - 1) cells
   more than the band.  For every row of every alignment of the sweep shapes, the stored extent (from the oracle's band,
   the reference's lg_vector_row rows) must fit chain_flatten's per-row estimate for the job
   ((2w + 1 + drift + 64 + POA_LG_ROW_CELLS(pn) + 7) / 8 + 2 groups), so the common path never needs a PLANE_OVF re-run."""
import ctypes as C

import numpy as np
import pytest

import score_window as sw
from abpoa_b200 import synth
from abpoa_b200.aligner import PoaConfig, PoaSession
from abpoa_b200.capi import c_u8_p
from cases import LINEAR
from oracle_binding import oracle_align
from test_chain_emul import drive, emul  # noqa: F401  (emul: the module's fixture)

E20 = dict(gap_open1=0, gap_ext1=20, gap_open2=0, gap_ext2=0)
AA = {k: v for k, v in synth.WORKLOADS["aa_blosum62_2k"].cfg.__dict__.items() if k not in LINEAR}


def sweep(lo, hi):
    return [(synth.make_group(5000 + s, 4 + s % 5, 150 + 37 * (s % 9), [0.03, 0.08, 0.15, 0.25][s % 4]),
             dict(LINEAR) if s % 2 == 0 else dict(LINEAR, wb=6 + s % 7, wf=0.01)) for s in range(lo, hi)]


EMUL_CASES = {
    "sweep_default_band": lambda: sweep(0, 1)[0],
    "sweep_narrow_band": lambda: sweep(1, 2)[0],
    "sweep_25pct": lambda: sweep(3, 4)[0],
    "sweep_narrow_long": lambda: sweep(7, 8)[0],
    "amino_acids": lambda: (synth.make_group(9800, 8, 300, 0.08, m=27), dict(LINEAR, **AA)),
    "pn16_1637": lambda: (sw.with_last(309, 3, 1000, 1637)(), dict(E20)),
    "pn8_1638": lambda: (sw.with_last(309, 3, 1000, 1638)(), dict(E20)),
}


@pytest.mark.parametrize("name", list(EMUL_CASES))
def test_device_graph_code_linear(emul, product_lib, name):  # noqa: F811
    reads, cfg_kw = EMUL_CASES[name]()
    cfg = PoaConfig(**cfg_kw)
    drive(emul, product_lib, cfg, reads, K=32 if cfg.m > 5 else 12)


def test_pn_widths_of_the_score_window_points(product_lib):
    """The two points give the job blob of their last read pn = 16 and pn = 8."""
    for last, pn in ((1637, 16), (1638, 8)):
        reads = sw.with_last(309, 3, 1000, last)()
        with PoaSession(PoaConfig(**E20), product_lib) as s:
            s.reset(max(len(r) for r in reads))
            for r in reads[:-1]:
                _, res = oracle_align(s, r)
                s.add(r, res, len(reads))
            assert blob_header(s, reads[-1])["pn"] == pn, f"last read of {last} bases"


def blob_header(s, r):
    d = s.lib.dll
    d.poa_debug_blob.restype = C.c_int
    d.poa_debug_blob.argtypes = [C.c_void_p, C.c_void_p, c_u8_p, C.c_int, c_u8_p, C.c_int]
    g = s.ab.contents.abg.contents
    buf = np.zeros(64 + 16 * (g.node_n + 2) * 6 + len(r) + 256, dtype=np.uint8)
    nb = d.poa_debug_blob(s.ab, s.abpt, r.ctypes.data_as(c_u8_p), len(r), buf.ctypes.data_as(c_u8_p), len(buf))
    assert nb > 0
    hdr = buf[:68].view(np.int32)
    off_rm = int(hdr[4])
    return dict(qlen=int(hdr[1]), w=int(hdr[2]), pn=int(hdr[14]), rem0=int(buf[off_rm + 4: off_rm + 8].view(np.int32)[0]) >> 8)


POA_LG_ROW_CELLS = lambda pn: 2 * (pn - 1)  # noqa: E731  (poa_chain.cuh)


def per_row_estimate(h):
    """chain_flatten's plane estimate of one row (8-cell groups, one plane) for a linear-gap job."""
    drift = abs(h["qlen"] - h["rem0"])
    per_row = (2 * h["w"] + 1 + drift + 64 + POA_LG_ROW_CELLS(h["pn"]) + 7) // 8 + 2
    return min(per_row, (h["qlen"] + 1 + 7) // 8 + 1)


@pytest.mark.parametrize("lo", [0, 20, 40])
def test_plane_estimate_covers_stored_lgx_rows(product_lib, lo):
    n_rows = widest = 0
    for reads, cfg_kw in sweep(lo, lo + 20) + [(sw.with_last(309, 3, 1000, 1638)(), dict(E20))]:
        reads = [np.ascontiguousarray(r, dtype=np.uint8) for r in reads]
        with PoaSession(PoaConfig(**cfg_kw), product_lib) as s:
            s.reset(max(len(r) for r in reads))
            for i, r in enumerate(reads):
                if i:
                    h = blob_header(s, r)
                    xs = 4 if h["pn"] == 16 else 3
                    bands = []
                    o, res = oracle_align(s, r, row_cb=lambda user, row, beg, end, *p: bands.append((beg, end)))
                    est = per_row_estimate(h)
                    for beg, end in bands:
                        if end < beg:
                            continue
                        ngrp = (((((end >> xs) + 1) << xs) - 1) >> 3) - (((beg >> xs) << xs) >> 3) + 1
                        widest = max(widest, ngrp)
                        n_rows += 1
                        assert ngrp <= est, f"read {i}: a row stores {ngrp} groups (band {beg}..{end}, pn {h['pn']}), estimate {est}"
                else:
                    o, res = oracle_align(s, r)
                s.add(r, res, len(reads))
    assert n_rows > 1000 and widest > 8
