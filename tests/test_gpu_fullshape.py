"""GPU parity at the BENCHMARKED sizes (BASELINE.json configs 2-5), product vs the unmodified
reference (stored by tests/reference_runs.py): per-read best score, graph-CIGAR length and FNV-1a
hash of every CIGAR word, DP-cell totals, consensus and coverage.

Small cases cannot reach what these do: 25 k-row graphs, bands wider than one 256-cell pass, scores
close to the packed kernel's int16 window, graphs past the point where the reference itself switches
to int32 (gn > 16 364), 20-pass rows in local mode.
"""
import pytest

from abpoa_b200 import synth
from abpoa_b200.batch import BatchEngine
from reference_runs import assert_batch_matches

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("engine", ["chain", "launch"])
@pytest.mark.parametrize("name,n_groups", [("convex_10k", 4), ("affine_1k", 6), ("local_linear_5k", 1), ("aa_blosum62_2k", 2)])
def test_full_shape(reference, name, n_groups, engine):
    """engine: the engine's own choice, which is the device-resident chain for global/banded/consensus runs (local mode
    always takes the launch engine, and must not touch the chain), or the launch-per-round engine forced."""
    w = synth.WORKLOADS[name]
    groups = w.groups(n_groups, base_seed=4200)
    ref = reference.batch(w.cfg, groups)
    with BatchEngine() as eng:
        got = eng.run(w.cfg, groups, record_reads=True, no_chain=(engine == "launch"))
        st = eng.stats()
    if engine == "chain":
        on_chain = n_groups if w.cfg.align_mode == 0 else 0
        assert st["chain_groups"] == on_chain and st["chain_fallback_groups"] == 0, st
    assert_batch_matches(got, groups, ref, f"{name}/{engine}", msa=False)


def test_full_shape_convex_generic_kernels(reference, monkeypatch):
    """The same 10 kbp x 50 shape with the packed kernel switched off: generic int16 planes while the reference's
    criterion allows (gn <= 16 364), int32 planes beyond -- both instantiations at full size."""
    monkeypatch.setenv("ABPOA_GPU_NO_P16", "1")
    w = synth.WORKLOADS["convex_10k"]
    groups = w.groups(1, base_seed=4300)
    ref = reference.batch(w.cfg, groups)
    with BatchEngine(n_workers=1, groups_per_launch=1) as eng:
        got = eng.run(w.cfg, groups, record_reads=True)
    assert_batch_matches(got, groups, ref, "convex_10k/generic", msa=False)
