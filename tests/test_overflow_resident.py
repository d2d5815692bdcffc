"""The mixers' overflow row with every model resident, against the unmodified reference.

tests/test_mixer_overflow.py replays FXCM, PAQ8 and PPMD, which leaves out the resident models and the device decoder.
tests/golden/overflow_random6k.npz (tools/make_overflow_golden.py) holds the reference's Predict() of every bit of 6000
coded bytes of uniform random data with 15 % spaces, which takes eleven mixers past the 10 000-context cap, and CRCs of
its FXCM and PAQ8 codes per 4096 bits and of its PPMD distribution per byte.

CPU: the host PAQ8 build over the stream (it must not trip PAQ8's image / audio / JPEG gate) against the fixture's CRCs.
GPU (-m gpu, tolerance 0): every model resident in bulk calls whose boundaries fall on the onsets; lock-step across the
first onset; a device encoder -> device decoder round trip over the whole stream."""
import numpy as np
import pytest

from harness import DBG_SEL, LAYER1, N_MIXERS, SEL_PITCH, build_host_tool, cm, code_in_pieces, expect, golden, lock_step, \
    onsets, ppmd_arena, round_trip, run_host_tool  # noqa: F401  (cm, ppmd_arena: fixtures)
from make_overflow_golden import coded_stream

# mixer -> the coded byte at which it meets its 10 001st context (the device's selectors, which equal the reference's)
ONSETS = {4: 2233, 23: 2415, 2: 2439, 3: 2439, 16: 3402, 44: 3402, 19: 3916, 43: 3916, 22: 4042, 45: 4042, 5: 5368}
# bulk calls whose boundaries fall on those onsets; each at most 2000 bytes, so that the debug fetches of the generated
# codes and selectors cover the whole call
PIECES = [1, 127, 129, 1000, 976, 182, 24, 963, 514, 126, 1958]


def _fixture():
    return golden("overflow_random6k")


def test_generator_reproduces_the_fixture():
    g = _fixture()
    assert np.array_equal(coded_stream(), g["stream"])
    assert g["vocab"].sum() == 256 and sum(PIECES) == g["stream"].size


def test_paq8_host_build_passes_the_gate_and_matches(tmp_path):
    g = _fixture()
    p8 = build_host_tool("paq8_check", str(tmp_path), ["-DCENSUS"])
    rc, out, crc = run_host_tool(p8, str(tmp_path), "p8_overflow", g["stream"])[:3]
    assert rc != 3, "overflow_random6k trips PAQ8's image / audio / JPEG gate:\n%s" % out[-2000:]
    assert rc == 0, out[-2000:]
    full = g["stream"].size * 8 // 4096          # the host build writes CRCs of whole 4096-bit blocks only
    bad = np.nonzero(crc != g["crc_p8"][:full])[0]
    assert crc.size == full and bad.size == 0, "PAQ8 codes: %d CRC blocks, expected %d; first differing block %s" % (crc.size, full, bad[:1])


@pytest.mark.gpu
@pytest.mark.timeout(900)
def test_everything_resident_across_the_onsets(cm):
    g = _fixture()
    ends = np.cumsum(PIECES).tolist()
    P = cm.Predictor(g["vocab"])
    sels = []
    try:
        code_in_pieces(P, g, zip([0] + ends[:-1], ends),
                       after=lambda P, a, b: sels.append(P.debug_fetch(DBG_SEL, ((b - a) * 8, SEL_PITCH), np.uint32)[:, :N_MIXERS]))
    finally:
        P.close()
    on = onsets(np.concatenate(sels))
    print("\noverflow_random6k: mixers past the cap at byte %s" % sorted(on.items(), key=lambda kv: (kv[1], kv[0])))
    assert on == ONSETS and any(m in LAYER1 for m in on), on


@pytest.mark.gpu
@pytest.mark.timeout(900)
def test_lock_step_across_the_first_onset(cm):
    g = _fixture()
    lo, hi = 2200, 2260                    # mixer 4 meets its 10 001st context at coded byte 2233
    P = cm.Predictor(g["vocab"])
    try:
        expect("overflow_random6k: bulk [0,%d)" % lo, P.code_bytes(g["stream"][:lo]), g["p"][:lo * 8])
        lock_step(P, g, lo * 8, hi * 8, "overflow_random6k: bulk [0,%d), lock-step [%d,%d)" % (lo, lo, hi))
        expect("overflow_random6k: lock-step then bulk [%d,6000)" % hi, P.code_bytes(g["stream"][hi:]), g["p"][hi * 8:], hi * 8)
    finally:
        P.close()


@pytest.mark.gpu
@pytest.mark.timeout(900)
def test_device_round_trip(cm, port):
    round_trip(cm, port, "overflow_random6k")
