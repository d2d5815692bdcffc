"""8-bit PCM WAV audio through the resident predictor: PAQ8's audio8bModel and recordModel(AUDIO) (paq8.cpp:5552-5657,
:5810-5869) on the bytes of a data chunk, the order-N map, run maps and match model in front of them, no other model.

Fixtures tests/golden/audio8_*.npz (tools/make_audio8_goldens.py over tools/gen_audio8.py) and the two 8-bit streams of
tools/gen_wav.py come from dumps of the unmodified reference, every bit of every stream.
CPU (-m "not gpu"): the host PAQ8 build (tools/paq8_check.cpp) against the reference's PAQ8 code CRCs; the generator.
GPU (-m gpu, tolerance 0): bulk calls with every PAQ8 code, lock-step across the first sample and the end of the data, a
batch, an encoder -> decoder round trip, and the jitter build."""
import re

import numpy as np
import pytest

from gen_audio8 import STREAMS, coded_stream, first_sample
from harness import awkward_lock_step, batch, build_host_tool, cm, code_in_pieces, even, golden, round_trip, \
    run_host_tools, run_jitter, jitter_lib, ppmd_arena  # noqa: F401  (cm, jitter_lib, ppmd_arena: fixtures)

HEADER = 5                                                    # cmix -n's header in front of the generated file
TO_END = [n for n in STREAMS if n != "audio8_then16"] + ["wav_pcm8_mono", "wav_pcm8_stereo"]


# ------------------------------------------------------------------------------------------------ CPU
@pytest.fixture(scope="module")
def host_runs(tmp_path_factory):
    tmp = str(tmp_path_factory.mktemp("audio8"))
    exe = build_host_tool("paq8_check", tmp)
    return run_host_tools({name: (exe, tmp, name, golden(name)["stream"]) for name in TO_END + ["audio8_then16"]})


@pytest.mark.parametrize("name", TO_END)
def test_host_build_codes_8bit_audio_to_the_end(host_runs, name):
    rc, out, crc = host_runs[name][:3]
    want = golden(name)["crc_p8"]
    assert rc == 0, "%s:\n%s" % (name, out[-2000:])
    bad = np.nonzero(crc != want[:crc.size])[0]
    assert crc.size == want.size and bad.size == 0, "%s: first differing 4096-bit block %s" % (name, bad[:1])


def test_host_build_stops_at_the_first_16bit_sample(host_runs):
    """An 8-bit file codes to its end; the 16-bit file after it raises the error on the bit before its first sample."""
    rc, out, crc = host_runs["audio8_then16"][:3]
    want = golden("audio8_then16")["crc_p8"]
    assert rc == 3, out[-2000:]
    stop = int(re.search(r"UNSUPPORTED after (\d+) bits", out).group(1))
    assert stop == (HEADER + first_sample("audio8_then16")[1]) * 8 - 1, out[-2000:]
    assert crc.size == stop // 4096 and np.array_equal(crc, want[:crc.size])


@pytest.mark.parametrize("name", [n for n in STREAMS if STREAMS[n][2] == "n"])
def test_generator_reproduces_the_fixture(name):
    assert np.array_equal(coded_stream(name), golden(name)["stream"])


# ------------------------------------------------------------------------------------------------ GPU
def _coded(name):
    """Coded-stream bytes of each first sample and of each byte after a data chunk's end."""
    g = golden(name)
    starts = [HEADER + k for k in first_sample(name)] if name in STREAMS else []
    ends = [HEADER + k + int.from_bytes(g["stream"][HEADER + k - 4:HEADER + k].tobytes(), "little") for k in first_sample(name)] \
        if name in STREAMS else []
    return starts, [e for e in ends if e < g["stream"].size]


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("name", [n for n in STREAMS if n != "audio8_then16"])
def test_bulk_pieces_equal_the_reference(cm, name):
    """Bulk calls of 1024 bytes: Predict() and every PAQ8 code of every bit, the slots an audio bit leaves alone included."""
    g = golden(name)
    P = cm.Predictor(g["vocab"])
    try:
        got = code_in_pieces(P, g, even(0, g["stream"].size, 1024))
    finally:
        P.close()
    assert got["crc_p8"].size == g["crc_p8"].size


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("name", ["audio8_mono_text", "audio8_mono_stereo"])
def test_lock_step_across_the_first_sample_and_the_end(cm, name):
    starts, ends = _coded(name)
    awkward_lock_step(cm, name, (starts[0] - 3, starts[0] + 40))
    awkward_lock_step(cm, name, (ends[0] - 30, ends[0] + 10))


@pytest.mark.gpu
@pytest.mark.timeout(900)
def test_audio_and_text_in_one_batch(cm):
    batch(cm, ["audio8_mono_text", "audio8_stereo_odd", "full_text"])


@pytest.mark.gpu
@pytest.mark.timeout(900)
def test_device_round_trip(cm):
    round_trip(cm, None, "audio8_stereo_odd")


@pytest.mark.gpu
@pytest.mark.timeout(1500)
def test_jitter_build_codes_audio_bit_exactly(jitter_lib):
    """The jitter build over the audio fixtures: random sleeps at every site, then each PAQ8 warp group starved / hurried."""
    from test_schedule_jitter import DENSITY, STARVE_GROUPS
    names = ["audio8_mono_stereo", "audio8_stereo_odd"]
    jobs = [[["random", seed, DENSITY, 0, 0], "bulk", [n]] for seed in (11, 12) for n in names]
    jobs += [[[mode, 0, g, 0, 0], "bulk", ["audio8_stereo_odd", 3072]] for g in STARVE_GROUPS if g.startswith("JG_P8_")
             for mode in ("starve", "hurry")]
    run_jitter(jitter_lib, "audio8 random, starve / hurry", jobs, timeout=1400)
