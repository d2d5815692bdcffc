"""FXCM on a cluster of two CTAs: the model CTA hands every bit to the mixer CTA through a 4-slot ring (fxcm.cuh).

GPU (-m gpu): bulk calls of sizes that make the ring wrap at every offset, lock-step stretches between bulk calls, three
streams in one batch and a device encoder -> decoder round trip must stay equal to the reference fixtures at tolerance 0;
and so must bulk calls with either CTA of the cluster alone slow, then alone fast, in the jitter build.
"""
import pytest

import test_schedule_jitter as jit
from test_call_schedules import _ppmd_arena  # noqa: F401  (autouse: a 512 MB PPMD arena, so three resident streams fit)
from test_schedule_jitter import jitter_lib  # noqa: F401  (the jitter build, a module fixture)

PIECES = [1, 3, 4, 5, 17, 129]
FX_GROUPS = ["JG_FX_MODEL", "JG_FX_MIXER"]


def test_fxcm_warp_groups_exist():
    assert all(g in jit.GROUPS for g in FX_GROUPS)


@pytest.mark.gpu
@pytest.mark.parametrize("piece", PIECES)
@pytest.mark.parametrize("name", ["fxwiki", "english"])
def test_bulk_pieces(name, piece):
    import cmix_b200
    jit._bulk(cmix_b200, name, 512, piece)   # the fixtures' code CRCs cover blocks of 4096 bits


@pytest.mark.gpu
def test_lock_step_between_bulk_calls():
    import cmix_b200
    jit._awkward(cmix_b200, "fxwiki")


@pytest.mark.gpu
def test_three_streams_in_one_batch():
    import cmix_b200
    jit._batch(cmix_b200, ["fxwiki", "english", "xml"], 1024)


@pytest.mark.gpu
def test_device_round_trip(port):
    import cmix_b200
    jit._round_trip(cmix_b200, port, "fxwiki", 512)


@pytest.mark.gpu
@pytest.mark.timeout(1800)
def test_starve_and_hurry_each_fxcm_cta(jitter_lib):  # noqa: F811
    jobs = []
    for g in FX_GROUPS:
        for mode in ("starve", "hurry"):
            jobs += [[[mode, 0, g, 0, 0], "bulk", [n, 1024, piece]] for n in ("fxwiki", "english") for piece in (5, 1024)]
    # _run records its runs in test_schedule_jitter's RAN and FIRED, which that module's last test compares with its own
    # set of runs; these runs are not among them, so they leave both as they found them
    ran, fired = set(jit.RAN), dict(jit.FIRED)
    try:
        jit._run(jitter_lib, "fxcm starve / hurry", jobs)
    finally:
        jit.RAN.clear(); jit.RAN.update(ran)
        jit.FIRED.clear(); jit.FIRED.update(fired)
