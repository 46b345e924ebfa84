"""The kernel matrix of tests/bm_reference.py on the CPU: the oracle's calc_disparity (the reference's sliding double box
sums) against the float64 brute force on every case, so that the two references the GPU tests compare with agree; and the
coverage ledger: every block-matching instantiation the CUDA sources compile is run by some case, or is listed in
bm_reference.UNREACHABLE with the reason no call can select it."""
import numpy as np
import pytest

import bm_reference as bm


@pytest.mark.parametrize("case", bm.CASES, ids=[c.id for c in bm.CASES])
def test_oracle_matches_brute_force(oracle, case):
    left, right = case.inputs()
    ref = bm.brute_calc_disparity(case.cost, left, right, case.search, case.kernel)
    got = oracle.calc_disparity(case.cost, left, right, case.search, case.kernel)
    bad = ~np.all(got == ref, axis=-1)
    assert not bad.any(), f"{case.id}: {int(bad.sum())} of {bad.size} pixels differ"
    assert ref[..., 2].any()


def _norm(family, args):
    return family, tuple(int(a) for a in args)


def test_coverage_ledger():
    compiled = {_norm(*k) for k in bm.compiled_instantiations()}
    assert len(compiled) > 100, "the dispatch switches were not parsed"
    unreachable = {_norm(*k) for k in bm.UNREACHABLE}
    covered = set()
    for case in bm.CASES:
        e = case.expect()
        covered.add(_norm(e.family, e.args))
        if e.merge:
            covered.add(_norm(*e.merge))
        if e.seed:
            covered.add(_norm("k1_fast_abs_kernel", e.seed))
    for _, cost, *_ in bm.VIEW_CASES:
        e = bm.view_expect(cost)
        covered.add(_norm(e.family, e.args))
    assert not unreachable & covered, f"listed as unreachable but run: {sorted(unreachable & covered)}"
    assert compiled - unreachable <= covered, f"compiled but run by no case: {sorted(compiled - unreachable - covered)}"
    assert unreachable <= compiled, f"listed as unreachable but not compiled: {sorted(unreachable - compiled)}"


def test_unreachable_screen_instantiations_are_unreachable():
    """Sq on K1 screen at kx = 3 and 5: over every ky and range, either K1 fast or no exact kernel takes it"""
    for kx in (3, 5):
        for ky in range(1, 42, 2):
            for r in (255, 1024, 2047, 3000, 4095):
                assert not (bm.k1_screen_supported(bm.SQ, kx, ky, 16, 8, 0, r, True)
                            and not bm.k1_fast_supported(bm.SQ, kx, ky, 16, 8, 0, r, True)), (kx, ky, r)


def test_matrix_reaches_every_ring_depth_and_staging_class():
    sd = {(e.args[1], e.geom["sd"]) for e in (c.expect() for c in bm.CASES) if e.family == "k1_screen_kernel"}
    assert sd == {(m, d) for m in (0, 1) for d in (1, 2, 3)}
    cls = {e.geom["cls"] for e in (c.expect() for c in bm.CASES) if e.family == "k1_zone_int_kernel"}
    assert cls == {0, 1, 2}
