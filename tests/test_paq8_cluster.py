"""PAQ8 on a cluster of two CTAs: the model CTA hands each bit to the mixer CTA through a ring of P8_RING = 4 slots.

Bulk calls of 1, 2, 3, 4 and 5 bytes end the ring at different fill levels relative to a launch's start, lock-step bits use a
one-slot handover, and every switch must carry the mixer CTA's state (weight-set cache, last prediction, persistent codes)
and the model CTA's state over exactly. Checked against the reference's dumps (tests/golden/full_text.npz: Predict() of
every bit and all 2 022 codes of the first 64 bits) at tolerance 0, after each call: the probabilities, the PAQ8 codes the
bulk kernel wrote per bit and the codes handed to the next Predict() (State::codes after a bulk call). Also: an error
raised by the model CTA (a JPEG header) still reaches the host when the mixer CTA writes back its part of the state."""
import numpy as np
import pytest

from harness import cm, golden  # noqa: F401  (cm: fixture)

pytestmark = pytest.mark.gpu

DBG_EXT_GEN, DBG_EXT_BIT = 10, 11


def _same(what, got, want):
    got, want = np.ascontiguousarray(got), np.ascontiguousarray(want)
    bad = np.argwhere(got != want)
    assert bad.size == 0, "%s: first difference at %s (%d differ)" % (what, bad[0].tolist(), len(bad))


def test_ring_depths_lock_step_and_bulk(cm):
    g = golden("full_text")
    s, first, p_ref = g["stream"], g["first_codes"], g["p"]
    bits = np.unpackbits(s)
    assert first.shape[0] >= 64
    P = cm.Predictor(g["vocab"])
    try:
        t = 0
        for n in (1, 2, 3):                        # bytes 0..5, bulk
            p = P.code_bytes(s[t // 8:t // 8 + n])
            _same("bulk of %d bytes at bit %d: Predict()" % (n, t), p.view(np.uint32), p_ref[t:t + 8 * n].view(np.uint32))
            ext = P.debug_fetch(DBG_EXT_GEN, (8 * n, 2022), np.uint16)
            _same("bulk of %d bytes at bit %d: PAQ8 codes" % (n, t), ext[:, 431:], first[t:t + 8 * n, 431:])
            t += 8 * n
            ext_bit = P.debug_fetch(DBG_EXT_BIT, (2022,), np.uint16)
            _same("codes handed over after the bulk call ending at bit %d" % t, ext_bit[431:], first[t, 431:])
        for _ in range(8):                         # byte 6, lock-step
            assert P.Predict() == p_ref[t], "lock-step bit %d" % t
            P.Perceive(int(bits[t]))
            t += 1
            if t < 64:
                _same("lock-step codes after bit %d" % (t - 1), P.debug_fetch(DBG_EXT_BIT, (2022,), np.uint16)[431:], first[t, 431:])
        p = P.code_bytes(s[7:8])                   # byte 7, bulk after lock-step
        _same("bulk after lock-step: Predict()", p.view(np.uint32), p_ref[56:64].view(np.uint32))
        _same("bulk after lock-step: PAQ8 codes", P.debug_fetch(DBG_EXT_GEN, (8, 2022), np.uint16)[:, 431:], first[56:64, 431:])
        t = 64
        for n in (4, 5, 1, 2, 3, 100):             # the rest of the depths, then a longer call
            p = P.code_bytes(s[t // 8:t // 8 + n])
            _same("bulk of %d bytes at bit %d: Predict()" % (n, t), p.view(np.uint32), p_ref[t:t + 8 * n].view(np.uint32))
            t += 8 * n
    finally:
        P.close()


def test_model_cta_error_reaches_the_host(cm):
    """A JPEG header in the third bulk call: the model CTA raises the sticky error, the mixer CTA owns the rest of the state."""
    g = golden("full_text")
    text = g["stream"][:400].copy()
    jpeg = np.frombuffer(bytes([0xFF, 0xD8, 0xFF, 0xE0, 0x00, 0x10]) + b"JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00", dtype=np.uint8)
    P = cm.Predictor(np.ones(256, dtype=np.uint8))
    try:
        P.code_bytes(text[:100])
        P.code_bytes(text[100:103])
        with pytest.raises(RuntimeError, match="image / audio / JPEG"):
            P.code_bytes(np.concatenate([jpeg, text[103:]]))
        with pytest.raises(RuntimeError, match="image / audio / JPEG"):   # sticky: the next call fails too
            P.code_bytes(text[:5])
    finally:
        P.close()
