"""The complete predictor with every model group resident (SURVEY §8 rows a1-a18): no replayed inputs anywhere.

Fixtures (tools/make_full_golden.py) come from dumps of the unmodified reference: Predictor::Predict() of every bit plus a
CRC32 per 4096 bits over its FXCM codes and over its PAQ8 codes.
CPU (-m "not gpu"): the host build of the PAQ8 model (tools/paq8_check.cpp) against the PAQ8 CRCs.
GPU (-m gpu): bytes in, probabilities out through the C-ABI; must equal the reference's probabilities bit for bit
(tolerance 0; north_star allows 1e-5), bulk and lock-step, and the generated FXCM / PAQ8 codes must match the CRCs."""
import os

import numpy as np
import pytest

from conftest import ROOT
from harness import build_host_tool, cm, code_in_pieces, even, golden, pretrain_buffer, run_host_tool  # noqa: F401  (cm: fixture)


@pytest.fixture(scope="module")
def paq8_check(tmp_path_factory):
    return build_host_tool("paq8_check", str(tmp_path_factory.mktemp("p8")))


@pytest.mark.parametrize("name", ["full_text", "full_bin"])
def test_paq8_host_build_matches_reference_codes(paq8_check, tmp_path, name):
    g = golden(name)
    n = 2048                                           # 4 CRC blocks: ~5 s of CPU per fixture
    r = run_host_tool(paq8_check, str(tmp_path), "d", g["stream"][:n])
    assert r.rc == 0, r.out
    assert np.array_equal(r.crc, g["crc_p8"][:r.crc.size]) and r.crc.size == n * 8 // 4096


def test_paq8_tables_are_the_reference_tables():
    """The hex tables in paq8_host.h against SHA-256 digests of what the reference's own initialisers produce
    (tests/golden/reference_tables.json, written by tools/make_ref_goldens.py)."""
    import hashlib
    import json
    from make_paq8_tables import ours
    want = json.load(open(os.path.join(ROOT, "tests", "golden", "reference_tables.json")))["paq8"]
    assert len(want) == 15
    for name, digest in want.items():
        assert hashlib.sha256(ours(name).encode()).hexdigest() == digest, name


# ------------------------------------------------------------------------------------------------ GPU
def _run_resident(cm, g, dictionary=None, pretrain=None, n=None):
    """Bulk calls of 2048 bytes over the first n bytes (all by default), after Pretrain() over `pretrain`; fails with every
    difference from the fixture. Returns {"p", "crc_fx", "crc_p8"}."""
    P = cm.Predictor(g["vocab"], dictionary_path=dictionary)
    try:
        if pretrain is not None:
            P.pretrain_bytes(pretrain)
        return code_in_pieces(P, g, even(0, g["stream"][:n].size))
    finally:
        P.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["full_text", "full_bin"])
def test_everything_resident_equals_the_reference(cm, name):
    g = golden(name)
    p = _run_resident(cm, g)["p"]
    bits = np.unpackbits(g["stream"])
    bpc = -np.log2(np.where(bits == 1, p, 1 - p).clip(1e-9, 1)).sum() / g["stream"].size
    bpc_ref = -np.log2(np.where(bits == 1, g["p"], 1 - g["p"]).clip(1e-9, 1)).sum() / g["stream"].size
    assert abs(bpc - bpc_ref) <= 0.001                 # north_star: compressed bits per byte within 0.001 of the reference


@pytest.mark.gpu
def test_everything_resident_with_dictionary_and_pretraining(cm, dict_path):
    """cmix -c english.dic in out: WRT code words in the stream, Pretrain() over header + dictionary before the first bit."""
    _run_resident(cm, golden("full_wrt"), dictionary=dict_path, pretrain=pretrain_buffer(dict_path), n=2048)


@pytest.mark.gpu
def test_everything_resident_lock_step(cm):
    """Predict()/Perceive(bit) one bit at a time (the decoder's order), then the bulk kernels mid-stream."""
    g = golden("full_text")
    bits = np.unpackbits(g["stream"])
    P = cm.Predictor(g["vocab"])
    n = 24
    for t in range(n * 8):
        assert P.Predict() == g["p"][t], "bit %d" % t
        P.Perceive(int(bits[t]))
    rest = P.code_bytes(g["stream"][n:512], None, None)
    P.close()
    assert np.array_equal(rest, g["p"][n * 8:512 * 8])


@pytest.mark.gpu
def test_unmodelled_block_fails_loudly(cm):
    """PAQ8's image / audio / JPEG sub-models are not resident: a stream in which its block parser would validate such a header
    must make the call fail (CMIXB200_ERR_UNSUPPORTED), never return different predictions silently."""
    g = golden("full_text")
    text = g["stream"][:700].copy()
    jpeg = np.frombuffer(bytes([0xFF, 0xD8, 0xFF, 0xE0, 0x00, 0x10]) + b"JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00", dtype=np.uint8)
    stream = np.concatenate([text[:300], jpeg, text[300:]])
    P = cm.Predictor(np.ones(256, dtype=np.uint8))
    with pytest.raises(RuntimeError, match="image / audio / JPEG"):
        P.code_bytes(stream, None, None)
    P.close()
