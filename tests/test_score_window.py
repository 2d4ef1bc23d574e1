"""The int16 score window on both sides of every edge (tests/score_window.py).

CPU: the oracle against the reference's stored result at every point.  Where `reference_sound` holds they must agree;
where the reference's int16 minus infinity (inf_min) beat a real score they must not (or the reference exits).  The
library's contract there is the oracle's: the exact optimum (INTEGRATION.md, "Differences from the reference").

GPU: the library at every point -- scores, graph-CIGARs, end points and every DP cell equal to the oracle's
(tests/planes.py); equal to the reference's digest where the reference is sound; the kernel that produced each accepted
result is the one the thresholds call for, and a packed-kernel result whose run the guard should have stopped is never
accepted.  Then the chain engine on both schedules.

Recording the reference's results (ABPOA_RECORD_REFERENCE, tests/reference_runs.py) runs it in a child process per
point, because at some points it calls exit(); those are stored as "aborts".
"""
from __future__ import annotations

import subprocess
import sys
from pathlib import Path

import pytest

import score_window as sw
from helpers import run_group
from reference_runs import _cfg_items, assert_run_matches, run_digest

NAMES = [p[0] for p in sw.POINTS]
HERE = Path(__file__).resolve().parent

_CHILD = """
import sys
sys.path[:0] = [{root!r}, {tests!r}]
from abpoa_b200 import capi
from helpers import run_group
from reference_runs import REFERENCE_LIB, run_digest
import score_window as sw
cfg, reads = sw.point({name!r})
print("DIGEST " + run_digest(run_group(capi.load_library(REFERENCE_LIB), cfg, reads)), flush=True)
"""


def reference_outcome(reference, name):
    """The reference's run digest at point `name`, or "aborts" when the reference exits there."""
    cfg, reads = sw.point(name)

    def compute():
        p = subprocess.run([sys.executable, "-c", _CHILD.format(root=str(HERE.parent), tests=str(HERE), name=name)],
                           capture_output=True, text=True, timeout=600)
        got = [ln.split()[1] for ln in p.stdout.splitlines() if ln.startswith("DIGEST ")]
        return got[0] if p.returncode == 0 and got else "aborts"
    return reference.value("score_window", _cfg_items(cfg), compute, reads)


@pytest.mark.parametrize("name", NAMES)
def test_oracle_vs_reference(product_lib, reference, name):
    cfg, reads = sw.point(name)
    want = reference_outcome(reference, name)
    got = run_digest(run_group(product_lib, cfg, reads, use_oracle=True))
    sound = sw.reference_sound(cfg, sw.profile(cfg, reads, product_lib))
    if name in sw.REFERENCE_WRONG:
        assert not sound, f"{name}: listed as a point where the reference's inf_min wins, but reference_sound holds"
        assert want == "aborts" or want != got, f"{name}: the reference now agrees with the oracle"
    elif sound:
        assert want != "aborts", f"{name}: the reference exits on a sound point"
        assert got == want, f"{name}: oracle and reference disagree on a point where the reference is sound"


@pytest.mark.parametrize("name", [n for n in NAMES if not n.startswith("infmin_")])
def test_point_sits_on_its_side(product_lib, name):
    """Each edge point lies on the side of its threshold its label says (poa_p16_ok for the edge read, the packed
    kernel's guard over all admitted alignments, poa_score_bits for the edge read), and a guard point lies near the
    threshold, not merely on one side of it."""
    cfg, reads = sw.point(name)
    alns = sw.profile(cfg, reads, product_lib)
    assert sw.edge_side(name, alns) == sw.BY_NAME[name][3], \
        f"{name}: sits on the {sw.edge_side(name, alns)!r} side, labelled {sw.BY_NAME[name][3]!r}: {alns}"
    m = sw.guard_margin(name, cfg, alns)
    if m is not None:
        v, lo, hi = m
        assert lo <= v <= hi, f"{name}: guarded quantity {v} is not in [{lo}, {hi}]"


def test_reference_sound_is_not_vacuous(product_lib):
    """The predicate is not trivially true: every point listed in REFERENCE_WRONG has a finite cell within SOUND_MARGIN
    of inf_min (the agreement of every sound point with the reference is test_oracle_vs_reference's job)."""
    for name in sw.REFERENCE_WRONG:
        cfg, reads = sw.point(name)
        h = sw.headroom(cfg, sw.profile(cfg, reads, product_lib))
        assert h is not None and h <= sw.SOUND_MARGIN, f"{name}: headroom {h}"


# ------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_library_on_window(product_lib, reference, name):
    """Every alignment: the accepted kernel is the packed one exactly when the job is admitted and the guard (modelled
    from the oracle's rows) does not fire; otherwise the generic kernel of the reference's width, after a redo if the job
    was admitted.  Planes, scores and CIGARs equal the oracle's; the run equals the reference where that is sound."""
    from abpoa_b200.aligner import PoaSession
    from planes import NEGP, run_planes
    cfg, reads = sw.point(name)
    prev = [0]
    seen = []

    def check(i, info):
        redo = info.retries > prev[0]
        prev[0] = info.retries
        with PoaSession(cfg, product_lib) as s:
            ok = sw.packed_admits(s.abpt, len(reads[i]), info.n_rows)
            bits = sw.score_bits(s.abpt, len(reads[i]), info.n_rows)
            fires = ok and sw.guard_fires(s.abpt, info.min_row_max, info.max_row_max, info.max_band)
        seen.append((info, ok, fires, redo))
        want = 15 if ok and not fires else bits
        assert info.kernel == want, f"{name} read {i}: accepted result from the {info.name} kernel, expected {want} " \
                                    f"(admitted {ok}, guard fires {fires}, reference width {bits})"
        if fires:
            assert redo, f"{name} read {i}: the guard should have fired, but no redo ran"
        if info.kernel == 15:        # the guard's bounds keep every real cell of an accepted job above -29000
            assert info.min_finite > NEGP, f"{name} read {i}: packed-kernel result accepted with a real cell at {info.min_finite}"
    run_planes(cfg, reads, product_lib, tag=name, check=check)
    print(f"[window] {name}: kernels {[x[0].kernel for x in seen]} admitted {[int(x[1]) for x in seen]} "
          f"guard {[int(x[2]) for x in seen]} redo {[int(x[3]) for x in seen]}")
    if name.startswith("guard_"):
        fired = any(x[2] for x in seen)
        assert fired == (sw.BY_NAME[name][3] == "out"), f"{name}: guard fired {fired}"
    want = reference_outcome(reference, name)
    if name not in sw.REFERENCE_WRONG and sw.reference_sound(cfg, sw.profile(cfg, reads, product_lib)):
        assert_run_matches(run_group(product_lib, cfg, reads), want, name)


# sound edge points through the chain engine, and whether the group must stay on the device.  The chain admits a group
# only if poa_p16_ok holds for every read against a graph of 3 x its length (poa_chain.cu), and hands a group back to
# the launch engine when one of its alignments ends in any status but OK -- a RANGE from the guard included.
CHAIN_POINTS = {"p16_qlen_28000": True, "guard_lo_e25": True, "guard_lo_e26": False, "bits_affine_1633": True,
                "guard_band_e16": True, "guard_band_e17": False}


@pytest.mark.gpu
@pytest.mark.parametrize("schedule", ["free-running", "rounds"])
def test_chain_engine_on_window(reference, monkeypatch, schedule):
    """Edge points (all sound), one group per run, through both chain-engine schedules: every group equals the reference;
    a group stays on the chain unless one of its jobs leaves the packed kernel's window, then it is handed back."""
    from abpoa_b200.batch import BatchEngine
    from reference_runs import assert_batch_matches
    if schedule == "rounds":
        monkeypatch.setenv("ABPOA_GPU_CHAIN_ROUNDS", "1")
    else:
        monkeypatch.delenv("ABPOA_GPU_CHAIN_ROUNDS", raising=False)
    for name, on_chain in CHAIN_POINTS.items():
        cfg, reads = sw.point(name)
        with BatchEngine(n_workers=1, groups_per_launch=1) as eng:
            got = eng.run(cfg, [reads], record_reads=True)
            st = eng.stats()
        assert_batch_matches(got, [reads], reference.batch(cfg, [reads]), f"{name} ({schedule})", msa=False)
        print(f"[window-chain] {name} {schedule}: chain_groups={st['chain_groups']} handed_back={st['chain_fallback_groups']}")
        assert st["chain_groups"] + st["chain_fallback_groups"] == 1, f"{name} ({schedule}): the group never reached the chain: {st}"
        assert st["chain_groups"] == int(on_chain), f"{name} ({schedule}): expected {'on the chain' if on_chain else 'handed back'}: {st}"
