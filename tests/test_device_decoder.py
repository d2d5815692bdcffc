"""Decompress direction on the device (SURVEY §8f rank 1, cmixb200_decode_bytes): the arithmetic decoder runs between the
predict and the perceive kernels of every bit, so a stream decodes without the bit visiting the host.
 * archive written by the device ENCODER (coder_begin / code_bytes / coder_finish) -> device decoder gives the bytes back;
 * the same archive through the host-side reference decoder arithmetic (tests/_coder.py restates decoder.cpp) driving the
   lock-step Predict()/Perceive() gives the same bytes: the two decode paths agree bit for bit;
 * the C-ABI exports the symbol (CPU check)."""
import os
import time

import numpy as np
import pytest

from harness import host_decode

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "full_text.npz")


def test_symbol_is_exported():
    from cmix_b200.capi import load_library
    lib = load_library()
    assert hasattr(lib, "cmixb200_decode_bytes")


@pytest.mark.gpu
@pytest.mark.timeout(900)
def test_device_decoder_round_trip():
    import cmix_b200
    os.environ.setdefault("CMIXB200_PPMD_MB", "512")
    g = np.load(GOLD)
    stream = g["stream"][:1536]
    enc = cmix_b200.Predictor(g["vocab"])
    enc.coder_begin(2 * stream.size + 64)
    p_enc = enc.code_bytes(stream)
    archive = enc.coder_finish()
    enc.close()
    np.testing.assert_array_equal(p_enc.view(np.uint32), g["p"][:stream.size * 8].view(np.uint32))   # the encoder side is the reference's

    dec = cmix_b200.Predictor(g["vocab"])
    t0 = time.perf_counter()
    out = dec.decode_bytes(archive, stream.size)
    dt = time.perf_counter() - t0
    dec.close()
    assert out.tobytes() == stream.tobytes()
    print("device decode: %.1f us per bit" % (dt / (stream.size * 8) * 1e6))

    host = cmix_b200.Predictor(g["vocab"])
    n_host = 96
    assert host_decode(host, archive, n_host) == stream[:n_host].tobytes()
    host.close()


@pytest.mark.gpu
@pytest.mark.timeout(900)
def test_device_decoder_continues_a_stream():
    """Two decode calls on one predictor, the second starting where the first stopped, equal one call; a bulk call may follow."""
    import cmix_b200
    os.environ.setdefault("CMIXB200_PPMD_MB", "512")
    g = np.load(GOLD)
    stream = g["stream"][:512]
    enc = cmix_b200.Predictor(g["vocab"])
    enc.coder_begin(2 * stream.size + 64)
    enc.code_bytes(stream)
    archive = enc.coder_finish()
    p_next = enc.code_bytes(g["stream"][512:544])
    enc.close()
    dec = cmix_b200.Predictor(g["vocab"])
    out = dec.decode_bytes(archive, stream.size)
    assert out.tobytes() == stream.tobytes()
    # the decoder's model state after 512 bytes is the encoder's: it predicts the following bytes identically
    np.testing.assert_array_equal(dec.code_bytes(g["stream"][512:544]).view(np.uint32), p_next.view(np.uint32))
    dec.close()
