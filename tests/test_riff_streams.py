"""RIFF data through the resident predictor: PAQ8's WAV parser (audioModel, paq8.cpp:5811-5866) decides what leaves the
ordinary models, exactly as the reference's does.

Fixtures tests/golden/near_*.npz and wav_*.npz (tools/make_wav_goldens.py over tools/gen_wav.py) come from dumps of the
unmodified reference, every bit of every stream. Near misses (text that mentions RIFF, AVI, WebP, a non-PCM, a 24-bit and a
badly sized WAV, one of them through the CLI's preprocessor) never reach the reference's audio models and must code
bit-exactly. Real PCM WAV files (8/16 bits, mono/stereo, an 18-byte fmt chunk with a LIST chunk, a data chunk longer than
the stream) reach them on their first sample, coded-stream bit 8192. Whatever the predictor returns for those must equal the
reference; it may stop with CMIXB200_ERR_UNSUPPORTED where it does not model the data, but never before the first sample.
CPU (-m "not gpu"): the host PAQ8 build (tools/paq8_check.cpp) against the reference's PAQ8 code CRCs; the generator.
GPU (-m gpu, tolerance 0): bulk calls, lock-step over a RIFF header, one batch of text and near misses, and the WAV files."""
import re

import numpy as np
import pytest

from gen_wav import ENTRY, STREAMS, coded_stream
from harness import batch, build_host_tool, cm, code_in_pieces, even, expect, golden, lock_step, ppmd_arena, run_host_tools, \
    wav_until_unsupported  # noqa: F401  (cm, ppmd_arena: fixtures)

NEAR = [n for n in STREAMS if n.startswith("near_")]
WAVS = [n for n in STREAMS if n.startswith("wav_")]


# ------------------------------------------------------------------------------------------------ CPU
@pytest.fixture(scope="module")
def host_runs(tmp_path_factory):
    """tools/paq8_check over every fixture, in parallel: HostRun (return code, output, CRCs per 4096 bits it completed)."""
    tmp = str(tmp_path_factory.mktemp("riff"))
    exe = build_host_tool("paq8_check", tmp)
    return run_host_tools({name: (exe, tmp, name, golden(name)["stream"]) for name in NEAR + WAVS})


@pytest.mark.parametrize("name", NEAR)
def test_near_miss_codes_with_the_ordinary_models(host_runs, name):
    rc, out, crc = host_runs[name][:3]
    want = golden(name)["crc_p8"]
    assert rc == 0, "%s: PAQ8's error word is set (image / audio / JPEG gate):\n%s" % (name, out[-2000:])
    bad = np.nonzero(crc != want[:crc.size])[0]
    assert crc.size == want.size and bad.size == 0, "%s: first differing 4096-bit block %s" % (name, bad[:1])


@pytest.mark.parametrize("name", WAVS)
def test_pcm_wav_host_build_never_codes_differently(host_runs, name):
    """Every 4096-bit block the host build completes equals the reference's. If it stops on PAQ8's error word, it stops on
    the first sample or later: the RIFF header and the text before it code with the ordinary models, as in the reference."""
    rc, out, crc = host_runs[name][:3]
    want = golden(name)["crc_p8"]
    assert rc in (0, 3), "%s:\n%s" % (name, out[-2000:])
    bad = np.nonzero(crc != want[:crc.size])[0]
    assert bad.size == 0, "%s: first differing 4096-bit block %d" % (name, bad[0])
    if rc == 0:
        assert crc.size == want.size, name
    else:
        stop = int(re.search(r"UNSUPPORTED after (\d+) bits", out).group(1))
        assert stop >= ENTRY * 8 - 1, "%s: the error word is set at bit %d, before the first sample (bit %d)" % (name, stop, ENTRY * 8)


@pytest.mark.parametrize("name", [n for n in NEAR + WAVS if STREAMS[n][2] == "n"])
def test_generator_reproduces_the_fixture(name):
    assert np.array_equal(coded_stream(name), golden(name)["stream"])


# ------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("name", NEAR)
def test_near_miss_resident_equals_the_reference(cm, name):
    """Bulk calls of 1024 bytes: the RIFF data starts inside the first call and runs on into the next."""
    g = golden(name)
    P = cm.Predictor(g["vocab"])
    try:
        got = code_in_pieces(P, g, even(0, g["stream"].size, 1024))
    finally:
        P.close()
    assert got["crc_p8"].size == g["crc_p8"].size


@pytest.mark.gpu
@pytest.mark.timeout(900)
def test_near_miss_lock_step_over_the_riff_header(cm):
    """Predict()/Perceive(bit) one bit at a time across the header of a WAVE file with a non-PCM format tag, then bulk."""
    g = golden("near_mp3_tag")
    P = cm.Predictor(g["vocab"])
    try:
        expect("near_mp3_tag: bulk [0,580)", P.code_bytes(g["stream"][:580]), g["p"][:580 * 8])
        lock_step(P, g, 580 * 8, 700 * 8, "near_mp3_tag: [580,700)")
        expect("near_mp3_tag: bulk [700,end)", P.code_bytes(g["stream"][700:]), g["p"][700 * 8:], 700 * 8)
    finally:
        P.close()


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("name", WAVS)
def test_pcm_wav_resident_never_codes_differently(cm, name):
    """Calls over the text and header, over the first sample, and over the samples: each call returns the reference's
    probabilities, or fails with CMIXB200_ERR_UNSUPPORTED; the call over the text and header never fails."""
    wav_until_unsupported(cm, name)


@pytest.mark.gpu
@pytest.mark.timeout(900)
def test_text_and_near_misses_in_one_batch(cm):
    """full_text, a WebP container and a badly sized WAV side by side in one code_batch_device call."""
    batch(cm, ["full_text", "near_webp", "near_odd_length"])
