"""Long-run parity (SURVEY §8(d) sizes): 256 KiB of gen_synth text through the complete resident predictor equals the
reference bit for bit - one CRC32 per 4096 coded bits over the float bit patterns of Predict(), checked in order so that a
failure names the first block that differs. The fixture comes from a dump of the unmodified reference
(tools/make_long_golden.py). The run crosses what short fixtures do not reach: >100 PPMD model growth steps per capacity
class, thousands of LSTM BPTT windows, PAQ8/FXCM bucket replacement under load, the mixers' learning-rate decay."""
import os
import zlib

import numpy as np
import pytest

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "long_text256k.npz")


def test_fixture_is_consistent():
    g = np.load(GOLD)
    n = g["stream"].size
    assert n >= 256 * 1024 and n % 512 == 0
    assert g["crc_p"].size == n * 8 // 4096
    assert zlib.crc32(g["p_head"].tobytes()) == int(g["crc_p"][0])
    assert zlib.crc32(g["p_tail"].tobytes()) == int(g["crc_p"][-1])
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
    from gen_synth import synth_text
    # the coded stream is runner.cpp's: a 5-byte block header (NoPreprocess), then the generator's text
    assert synth_text(262144)[:n - 5] == g["stream"][5:].tobytes()


@pytest.mark.gpu
@pytest.mark.timeout(1200)
def test_256k_text_equals_the_reference():
    import cmix_b200
    g = np.load(GOLD)
    stream = g["stream"]
    os.environ.setdefault("CMIXB200_PPMD_MB", "4096")
    P = cmix_b200.Predictor(g["vocab"])
    p = np.empty(stream.size * 8, dtype=np.float32)
    step = 32768
    for lo in range(0, stream.size, step):                       # the stream is ONE predictor; pieces only bound the host buffers
        p[lo * 8:(lo + step) * 8] = P.code_bytes(stream[lo:lo + step])
    P.close()
    crc = np.array([zlib.crc32(p[b:b + 4096].tobytes()) for b in range(0, p.size, 4096)], dtype=np.uint32)
    bad = np.nonzero(crc != g["crc_p"])[0]
    assert bad.size == 0, "first differing block of 4096 bits: %d (byte %d)" % (bad[0], bad[0] * 512)
    np.testing.assert_array_equal(p[-4096:].view(np.uint32), g["p_tail"].view(np.uint32))
    bits = np.unpackbits(stream)
    pd = p.astype(np.float64)
    bpc = float(-np.log2(np.where(bits == 1, pd, 1 - pd).clip(1.0 / 65536, 1)).sum() / stream.size)
    assert abs(bpc - float(g["bpc"][0])) < 1e-9


GOLD_1M = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "long_text1m.npz")


@pytest.mark.gpu
@pytest.mark.timeout(3600)
@pytest.mark.skipif(os.environ.get("CMIXB200_SLOW") != "1" or not os.path.exists(GOLD_1M), reason="1 MiB run: set CMIXB200_SLOW=1")
def test_1m_text_equals_the_reference():
    """Same check over 1 MiB (gen_synth seed 0xE9E80011): 8.4 M coded bits, one CRC per 4 096; run on demand."""
    import cmix_b200
    g = np.load(GOLD_1M)
    stream = g["stream"]
    os.environ.setdefault("CMIXB200_PPMD_MB", "8192")
    P = cmix_b200.Predictor(g["vocab"])
    step = 65536
    bad = []
    for lo in range(0, stream.size, step):
        p = P.code_bytes(stream[lo:lo + step])
        crc = np.array([zlib.crc32(p[b:b + 4096].tobytes()) for b in range(0, p.size, 4096)], dtype=np.uint32)
        want = g["crc_p"][lo * 8 // 4096:(lo + step) * 8 // 4096]
        miss = np.nonzero(crc != want)[0]
        if miss.size:
            bad.append(lo * 8 // 4096 + int(miss[0]))
            break
    P.close()
    assert not bad, "first differing block of 4096 bits: %d" % bad[0]
