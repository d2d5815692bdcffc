"""The mixers' overflow row with every model resident, against the unmodified reference.

tests/test_mixer_overflow.py replays FXCM, PAQ8 and PPMD, which leaves out the resident models and the device decoder.
tests/golden/overflow_random6k.npz (tools/make_overflow_golden.py) holds the reference's Predict() of every bit of 6000
coded bytes of uniform random data with 15 % spaces, which takes eleven mixers past the 10 000-context cap, and CRCs of
its FXCM and PAQ8 codes per 4096 bits and of its PPMD distribution per byte.

CPU: the host PAQ8 build over the stream (it must not trip PAQ8's image / audio / JPEG gate) against the fixture's CRCs.
GPU (-m gpu, tolerance 0): every model resident in bulk calls whose boundaries fall on the onsets; lock-step across the
first onset; a device encoder -> device decoder round trip over the whole stream."""
import os
import zlib

import numpy as np
import pytest

from conftest import ROOT
from make_overflow_golden import coded_stream
from test_mixer_overflow import DBG_SEL, LAYER1, N_MIXERS, SEL_PITCH, onsets

# mixer -> the coded byte at which it meets its 10 001st context (the device's selectors, which equal the reference's)
ONSETS = {4: 2233, 23: 2415, 2: 2439, 3: 2439, 16: 3402, 44: 3402, 19: 3916, 43: 3916, 22: 4042, 45: 4042, 5: 5368}
# bulk calls whose boundaries fall on those onsets; each at most 2000 bytes, so that the debug fetches of the generated
# codes and selectors cover the whole call
PIECES = [1, 127, 129, 1000, 976, 182, 24, 963, 514, 126, 1958]


def _fixture():
    z = np.load(os.path.join(ROOT, "tests", "golden", "overflow_random6k.npz"))
    return {k: z[k] for k in z.files}


def test_generator_reproduces_the_fixture():
    g = _fixture()
    assert np.array_equal(coded_stream(), g["stream"])
    assert g["vocab"].sum() == 256 and sum(PIECES) == g["stream"].size


def test_paq8_host_build_passes_the_gate_and_matches(tmp_path):
    from test_stress_data import _compile, _host_run
    g = _fixture()
    p8 = _compile(str(tmp_path), "paq8_check", ["-ffp-contract=off"])
    rc, out, crc, _ = _host_run(p8, str(tmp_path), "p8_overflow", g["stream"])
    assert rc != 3, "overflow_random6k trips PAQ8's image / audio / JPEG gate:\n%s" % out[-2000:]
    assert rc == 0, out[-2000:]
    full = g["stream"].size * 8 // 4096          # the host build writes CRCs of whole 4096-bit blocks only
    bad = np.nonzero(crc != g["crc_p8"][:full])[0]
    assert crc.size == full and bad.size == 0, "PAQ8 codes: %d CRC blocks, expected %d; first differing block %s" % (crc.size, full, bad[:1])


@pytest.fixture(autouse=True)
def _ppmd_arena(monkeypatch):
    if "CMIXB200_PPMD_MB" not in os.environ:
        monkeypatch.setenv("CMIXB200_PPMD_MB", "512")


@pytest.fixture(scope="module")
def cm():
    import cmix_b200
    cmix_b200.load_library()
    return cmix_b200


@pytest.mark.gpu
@pytest.mark.timeout(900)
def test_everything_resident_across_the_onsets(cm):
    from test_stress_data import _mismatch_report
    g = _fixture()
    s = g["stream"]
    P = cm.Predictor(g["vocab"])
    ps, exts, sels, ppmd_crc = [], [], [], []
    try:
        off = 0
        for n in PIECES:
            ps.append(P.code_bytes(s[off:off + n]))
            exts.append(P.debug_fetch(10, (n * 8, 2022), np.uint16))
            sels.append(P.debug_fetch(DBG_SEL, (n * 8, SEL_PITCH), np.uint32)[:, :N_MIXERS])
            rows = P.debug_fetch(8, (n, 256), np.float32)
            ppmd_crc += [zlib.crc32(rows[t].tobytes()) for t in range(n)]
            off += n
    finally:
        P.close()
    on = onsets(np.concatenate(sels))
    print("\noverflow_random6k: mixers past the cap at byte %s" % sorted(on.items(), key=lambda kv: (kv[1], kv[0])))
    assert on == ONSETS and any(m in LAYER1 for m in on), on
    ext = np.concatenate(exts)
    crc_fx = np.array([zlib.crc32(np.ascontiguousarray(ext[b:b + 4096, :431]).tobytes()) for b in range(0, ext.shape[0], 4096)], dtype=np.uint32)
    crc_p8 = np.array([zlib.crc32(np.ascontiguousarray(ext[b:b + 4096, 431:]).tobytes()) for b in range(0, ext.shape[0], 4096)], dtype=np.uint32)
    report = _mismatch_report("overflow_random6k", g, np.concatenate(ps), crc_fx, crc_p8, ext[:64], np.array(ppmd_crc, dtype=np.uint32))
    if report:
        pytest.fail(report, pytrace=False)


@pytest.mark.gpu
@pytest.mark.timeout(900)
def test_lock_step_across_the_first_onset(cm):
    from test_call_schedules import _expect, _lock_step
    g = _fixture()
    lo, hi = 2200, 2260                    # mixer 4 meets its 10 001st context at coded byte 2233
    P = cm.Predictor(g["vocab"])
    try:
        _expect("overflow_random6k: bulk [0,%d)" % lo, P.code_bytes(g["stream"][:lo]), g["p"][:lo * 8])
        _lock_step(P, g, lo * 8, hi * 8, "overflow_random6k: bulk [0,%d), lock-step [%d,%d)" % (lo, lo, hi))
        _expect("overflow_random6k: lock-step then bulk [%d,6000)" % hi, P.code_bytes(g["stream"][hi:]), g["p"][hi * 8:], hi * 8)
    finally:
        P.close()


@pytest.mark.gpu
@pytest.mark.timeout(900)
def test_device_round_trip(cm, port):
    from test_call_schedules import _expect, _first_bad_byte, _host_archive
    g = _fixture()
    s, p = g["stream"], g["p"]
    enc = cm.Predictor(g["vocab"])
    try:
        enc.coder_begin(2 * s.size + 64)
        _expect("overflow_random6k: encoder", enc.code_bytes(s), p)
        archive = enc.coder_finish()
    finally:
        enc.close()
    want = _host_archive(port, p, np.unpackbits(s))
    assert archive == want, "overflow_random6k: device archive differs from the host encoder's: %s" % _first_bad_byte(archive, want)
    dec = cm.Predictor(g["vocab"])
    try:
        out = dec.decode_bytes(archive, s.size)
    finally:
        dec.close()
    assert out.tobytes() == s.tobytes(), "overflow_random6k, decoder: %s" % _first_bad_byte(out, s)
