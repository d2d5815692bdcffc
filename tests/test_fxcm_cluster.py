"""FXCM on a cluster of two CTAs: the model CTA hands every bit to the mixer CTA through a 4-slot ring (fxcm.cuh).

GPU (-m gpu): bulk calls of sizes that make the ring wrap at every offset, lock-step stretches between bulk calls, three
streams in one batch and a device encoder -> decoder round trip must stay equal to the reference fixtures at tolerance 0;
and so must bulk calls with either CTA of the cluster alone slow, then alone fast, in the jitter build.
"""
import pytest

from harness import GROUPS, awkward_lock_step, batch, cm, code_in_pieces, even, golden, jitter_lib, ppmd_arena, round_trip, \
    run_jitter  # noqa: F401  (cm, jitter_lib, ppmd_arena: fixtures)

PIECES = [1, 3, 4, 5, 17, 129]
FX_GROUPS = ["JG_FX_MODEL", "JG_FX_MIXER"]


def test_fxcm_warp_groups_exist():
    assert all(g in GROUPS for g in FX_GROUPS)


@pytest.mark.gpu
@pytest.mark.parametrize("piece", PIECES)
@pytest.mark.parametrize("name", ["fxwiki", "english"])
def test_bulk_pieces(cm, name, piece):
    g = golden("reach_" + name)
    P = cm.Predictor(g["vocab"])
    try:
        code_in_pieces(P, g, even(0, 512, piece))   # the fixtures' code CRCs cover blocks of 4096 bits
    finally:
        P.close()


@pytest.mark.gpu
def test_lock_step_between_bulk_calls(cm):
    awkward_lock_step(cm, "reach_fxwiki")


@pytest.mark.gpu
def test_three_streams_in_one_batch(cm):
    batch(cm, ["reach_fxwiki", "reach_english", "reach_xml"], 1024)


@pytest.mark.gpu
def test_device_round_trip(cm, port):
    round_trip(cm, port, "reach_fxwiki", 512)


@pytest.mark.gpu
@pytest.mark.timeout(1800)
def test_starve_and_hurry_each_fxcm_cta(jitter_lib):
    jobs = []
    for g in FX_GROUPS:
        for mode in ("starve", "hurry"):
            jobs += [[[mode, 0, g, 0, 0], "bulk", ["reach_" + n, 1024, piece]] for n in ("fxwiki", "english") for piece in (5, 1024)]
    run_jitter(jitter_lib, "fxcm starve / hurry", jobs)
