"""The complete resident predictor on small, sparse and unpadded vocabularies (tools/gen_vocab.py).

The vocabulary is the one input of cmixb200_create that changes array shapes on the device. Its V symbols set the LSTM's
one-hot columns (padded to a multiple of 4), its softmax rows (ceil(V/8) per CTA of the 8-CTA cluster: CTAs past the
last row own none), the [V][25] slice of W_o its BPTT stages and byte_map; bytes outside it have probability 0 in the
LSTM's ByteModel, so a bit whose range holds vocabulary bytes on one side only reads out exactly 0 or 1 and Predict()
returns that value without mixing; PPMD's output and the bracket model's ByteModel mask by it; and the runner writes it
as a 32-byte bitmap after the length. The fixtures tests/golden/vocab_*.npz (tools/make_vocab_goldens.py) come from
coded streams of at least 10000 bytes whose byte set is the alphabet, so the reference chose each vocabulary itself.

CPU (-m "not gpu"): the generator reproduces every fixture; each shape's reason to exist, recomputed from V; the host
builds of PAQ8, FXCM and PPMD against the fixtures' CRCs; the CPU port against reference dumps at level 2 over the first
PORT_BYTES bytes of every shape, at every bit; the runner's header and the host encoder against the reference CLI's
archive; and a table of what each shape reaches next to full_text, full_wrt and full_bin.
GPU (-m gpu, tolerance 0): every shape with everything resident in bulk calls of awkward sizes; lock-step across the
first BPTT between awkward bulk calls; three vocabularies in one batch; device encoder -> device decoder round trips;
and V = 1 and four shapes with the big groups replayed against the port, the LSTM's distribution checked after each
call."""
import os
import subprocess
import time
import zlib

import numpy as np
import pytest

from conftest import ROOT, synthetic_streams
from gen_vocab import ALPHABETS, DUMPED, FULL, STREAMS, coded_stream, generate
from harness import SMALL_COLS, awkward_lock_step, batch, build_host_tool, check_host, cm, code_in_pieces, expect, golden, \
    host_archive, port_bit_for_bit, ppmd_arena, ppmd_host, reference_dumps, round_trip, run_host_tools, \
    stress_pieces  # noqa: F401  (cm, ppmd_arena, ppmd_host: fixtures)

NAMES = list(STREAMS)
PORT_BYTES = 320                          # three BPTT rounds of the LSTM (bytes 100, 200, 300)
REPLAY_ALL = ("fxcm", "paq8")
DBG_LSTM_PROBS = 4                        # CMIXB200_DBG_LSTM_PROBS: the LSTM's 256-float distribution after the last byte
CLI = os.path.join(ROOT, "build", "cmix_b200_cli")

# what each shape is for, as V and its consequences on the device: (V, V mod 4, softmax rows per CTA, CTAs with no row)
CLAIMS = {"two": (2, 2, 1, 6), "digits3": (3, 3, 1, 5), "four": (4, 0, 1, 4), "nine": (9, 1, 2, 3), "lower": (27, 3, 4, 1),
          "v33": (33, 1, 5, 1), "v57": (57, 1, 8, 0), "v58": (58, 2, 8, 0), "high": (129, 1, 17, 0),
          "v254": (254, 2, 32, 0), "v255": (255, 3, 32, 0)}
BASELINE = ["full_text", "full_wrt", "full_bin"]


def _fixture(name):
    return golden("vocab_" + name)


def shape(v):
    """(V mod 4, softmax rows per CTA, CTAs that own no row) of lstm.cuh's 8-CTA split: rows [rank*rpc, min(V, ...))."""
    rpc = -(-v // 8)
    return v % 4, rpc, sum(1 for rank in range(8) if rank * rpc >= v)


def runner_header(n, vocab):
    """What the reference's runner writes before the coder's bytes (runner.cpp:34-52): the coded length in 5 bytes,
    big-endian, then from 10000 bytes on the vocabulary as 32 bytes, symbol 8i + j in bit j of byte i."""
    head = np.array([(n >> (8 * i)) & 0xFF for i in (4, 3, 2, 1, 0)], dtype=np.uint8)
    head[0] &= 0x7F
    return np.concatenate([head, np.packbits(vocab.astype(np.uint8), bitorder="little")]) if n >= 10000 else head


def _inputs(names, n=PORT_BYTES):
    """harness.reference_dumps inputs: each shape's whole file (so the reference takes its vocabulary from it), n bytes coded."""
    return {name: (generate(name, *STREAMS[name]), "n", n) for name in names}


# ------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("name", NAMES)
def test_generator_reproduces_the_fixture(name):
    g = _fixture(name)
    s = coded_stream(name)
    assert g["stream"].size == DUMPED[name] and np.array_equal(s[:g["stream"].size], g["stream"])
    assert int(g["file_bytes"][0]) == s.size >= 10000, "the reference gives a stream under 10000 bytes every symbol"
    assert np.array_equal(np.nonzero(g["vocab"])[0], np.unique(s)), "the vocabulary is not the stream's byte set"
    assert np.array_equal(np.unique(s), ALPHABETS[name])
    assert int(g["vocab"].sum()) == CLAIMS[name][0]


@pytest.mark.parametrize("name", NAMES)
def test_each_shape_reaches_what_it_claims(name):
    """Recomputed from the fixture's V, so that a regenerated fixture cannot lose its reason to exist."""
    v = int(_fixture(name)["vocab"].sum())
    assert (v,) + shape(v) == CLAIMS[name]


@pytest.fixture(scope="module")
def host_runs(tmp_path_factory):
    """The host PAQ8 and FXCM builds over every shape's fixture (whole 4096-bit CRC blocks), in parallel."""
    tmp = str(tmp_path_factory.mktemp("vocab"))
    p8 = build_host_tool("paq8_check", tmp)
    fx = build_host_tool("fxcm_check", tmp)
    jobs = {}
    for name in NAMES:
        g = _fixture(name)
        s = g["stream"][:g["stream"].size // 512 * 512]
        jobs[("p8", name)] = (p8, tmp, "p8_" + name, s, None)
        jobs[("fx", name)] = (fx, tmp, "fx_" + name, s, g["lstmfx"][:s.size * 8])
    return run_host_tools(jobs)


@pytest.mark.parametrize("name", NAMES)
def test_paq8_host_build_matches_reference_codes(host_runs, name):
    g = _fixture(name)
    check_host(host_runs[("p8", name)], g["crc_p8"][:g["stream"].size // 512], "vocab_%s, PAQ8" % name)


@pytest.mark.parametrize("name", NAMES)
def test_fxcm_host_build_matches_reference_codes(host_runs, name):
    g = _fixture(name)
    check_host(host_runs[("fx", name)], g["crc_fx"][:g["stream"].size // 512], "vocab_%s, FXCM" % name)


@pytest.mark.parametrize("name", NAMES)
def test_ppmd_host_build_matches_reference_distributions(ppmd_host, name):
    g = _fixture(name)
    rc, out = ppmd_host(g["stream"], g["vocab"])
    assert rc == 0
    got = np.array([zlib.crc32(out[t].tobytes()) for t in range(out.shape[0])], dtype=np.uint32)
    bad = np.nonzero(got != g["ppmd_crc"])[0]
    assert bad.size == 0, "vocab_%s: first differing PPMD distribution after byte %d" % (name, bad[0])


@pytest.fixture(scope="module")
def level2_dumps(tmp_path_factory):
    """oracle_dump at level 2 over the first PORT_BYTES coded bytes of every shape."""
    t0 = time.perf_counter()
    out = reference_dumps(str(tmp_path_factory.mktemp("dumps2")), level=2, inputs=_inputs(NAMES))
    print("\nreference dumps at level 2, %d shapes x %d bytes: %.1f s" % (len(NAMES), PORT_BYTES, time.perf_counter() - t0))
    return out


@pytest.mark.timeout(900)
@pytest.mark.parametrize("name", NAMES)
def test_port_matches_reference_bit_for_bit(port, level2_dumps, name):
    """The CPU port, which the GPU tests with replayed groups compare against, pinned at this vocabulary: fed the
    reference's codes and PPMD rows, it gives the reference's Predict(), inputs, mixer outputs and selectors at every
    bit and its LSTM distribution after every byte."""
    d, g = level2_dumps[name], _fixture(name)
    assert np.array_equal(d.vocab, g["vocab"]) and np.array_equal(d.stream, g["stream"][:PORT_BYTES])
    expect("vocab_%s: the level-2 dump's Predict()" % name, d.p, g["p"][:PORT_BYTES * 8])
    port_bit_for_bit(port, "vocab_" + name, d.vocab, d.stream, d.ext, d.ppmd, d.p, d.inputs[:, SMALL_COLS], d.inputs[:64],
                     d.mix, d.ctx, d.lstm)


def test_archive_matches_reference_cli(port):
    """The runner's header (length, then the 32-byte vocabulary bitmap) and the host encoder over the reference's
    probabilities give the archive the unmodified reference CLI wrote (`cmix -n`, tests/golden/vocab_<FULL>.cmix)."""
    g = _fixture(FULL)
    s = g["stream"]
    assert s.size == int(g["file_bytes"][0]), "the fixture holds the whole stream"
    ref = np.fromfile(os.path.join(ROOT, "tests", "golden", "vocab_%s.cmix" % FULL), dtype=np.uint8)
    head = runner_header(s.size, g["vocab"])
    assert head.size == 37
    mine = np.concatenate([head, np.frombuffer(host_archive(port, g["p"], np.unpackbits(s)), dtype=np.uint8)])
    assert mine.size == ref.size and np.array_equal(mine, ref), "archive differs from the reference CLI's"


def test_table_of_what_each_shape_reaches():
    """V, rows per CTA, CTAs with no softmax row, bits whose Predict() is exactly 0 or 1 (the LSTM's read-out decides
    them) and BPTT rounds in the prefix, per shape and for the older whole-predictor fixtures."""
    lines = ["%-10s %4s %5s %9s %10s %15s %6s" % ("fixture", "V", "V%4", "rows/CTA", "no-row CTAs", "p in {0,1}", "BPTT")]
    decided = {}
    for name in ["vocab_" + n for n in NAMES] + BASELINE:
        g = golden(name)
        v = int(g["vocab"].sum())
        mod4, rpc, empty = shape(v)
        k = int(np.count_nonzero((g["p"] == 0) | (g["p"] == 1)))
        decided[name] = k / g["p"].size
        lines.append("%-10s %4d %5d %9d %10d %8d/%-6d %6d" % (name[6:] if name.startswith("vocab_") else name, v, mod4, rpc,
                                                               empty, k, g["p"].size, g["stream"].size // 100))
    print("\n" + "\n".join(lines))
    for name in ("two", "digits3"):
        assert decided["vocab_" + name] >= 0.75, "vocab_%s: only %.3f of its bits are decided" % (name, decided["vocab_" + name])


# ------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("name", NAMES)
def test_everything_resident_in_awkward_pieces(cm, name):
    """Every Predict(), FXCM and PAQ8 code CRC and PPMD distribution, in bulk calls of 1, 129, 1000, ... bytes."""
    g = _fixture(name)
    P = cm.Predictor(g["vocab"])
    try:
        code_in_pieces(P, g, stress_pieces(g["stream"].size))
    finally:
        P.close()


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("name", NAMES)
def test_lock_step_across_the_first_bptt(cm, name):
    """Lock-step over bytes [96, 104) between awkward bulk calls: the lock-step read-out (and its 0/1 override) and
    lstm_byte_kernel's BPTT at byte 100."""
    awkward_lock_step(cm, "vocab_" + name, span=(96, 104))


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("names", [("two", "v33", "v255"), ("digits3", "v58", "high")])
def test_three_vocabularies_in_one_batch(cm, names):
    batch(cm, ["vocab_" + n for n in names])


@pytest.mark.gpu
@pytest.mark.timeout(1200)
@pytest.mark.parametrize("name", ["two", FULL])
def test_device_round_trip(cm, port, name):
    """The device encoder writes the host encoder's archive and the device decoder gets the stream back; for the
    whole stream, the runner's header and that archive are the reference CLI's file."""
    archive = round_trip(cm, port, "vocab_" + name)
    if name == FULL:
        g = _fixture(name)
        ref = open(os.path.join(ROOT, "tests", "golden", "vocab_%s.cmix" % name), "rb").read()
        mine = runner_header(g["stream"].size, g["vocab"]).tobytes() + archive
        assert mine == ref, "header + device archive differ from the reference CLI's archive"


@pytest.mark.gpu
@pytest.mark.timeout(1200)
@pytest.mark.skipif(not os.path.exists(CLI), reason="reference CLI + shim not built (make -C cmix_b200/shim)")
def test_reference_cli_round_trip(tmp_path):
    """The reference's own runner, coder and preprocessor compiled against the shim: `-c` then `-d` over the whole
    file of the shape with a vocabulary bitmap in its archive gives the file back."""
    src, arc, back = tmp_path / "in.bin", tmp_path / "out.cmix", tmp_path / "back.bin"
    generate(FULL, *STREAMS[FULL]).tofile(src)
    for args in (["-c", str(src), str(arc)], ["-d", str(arc), str(back)]):
        subprocess.run([CLI, *args], check=True, stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL, timeout=900)
    assert back.read_bytes() == src.read_bytes()


REPLAYED = ["v1", "two", "nine", "v33"]
REPLAY_ENDS = [99, 100, 101, 199, 300, PORT_BYTES]


@pytest.fixture(scope="module")
def ppmd_rows(tmp_path_factory):
    """The reference's PPMD distribution after each of the first PORT_BYTES bytes of the replayed shapes (level 1)."""
    t0 = time.perf_counter()
    names = [n for n in REPLAYED if n != "v1"]
    d = reference_dumps(str(tmp_path_factory.mktemp("dumps1")), level=1, inputs=_inputs(names))
    print("\nreference dumps at level 1, %d shapes x %d bytes: %.1f s" % (len(names), PORT_BYTES, time.perf_counter() - t0))
    return {n: (d[n].stream, d[n].vocab, d[n].ppmd) for n in names}


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("name", REPLAYED)
def test_replayed_groups_against_the_port(cm, port, ppmd_rows, name):
    """FXCM and PAQ8 replayed with seeded codes, PPMD with the reference's rows (V = 1: the flat distribution), against
    the port pinned above; bulk calls end on bytes 99, 100, 101, 199 and 300, and the LSTM's distribution is compared
    after each, so that a difference names the LSTM before it reaches a later Predict()."""
    if name == "v1":
        stream = np.zeros(PORT_BYTES, dtype=np.uint8)
        vocab = np.zeros(256, dtype=np.uint8)
        vocab[0] = 1
        ppmd = np.tile(vocab.astype(np.float32), (PORT_BYTES, 1))
    else:
        stream, vocab, ppmd = ppmd_rows[name]
    codes = synthetic_streams(PORT_BYTES, seed=0x70CAB100 + REPLAYED.index(name))[2]   # seeded codes, [bits][2022]
    v = np.ascontiguousarray(vocab, dtype=np.uint8)
    Q = port.op_create(v.ctypes.data)
    P = cm.Predictor(vocab, replay=REPLAY_ALL)
    want_lstm = np.zeros(256, dtype=np.float32)
    try:
        a = 0
        for b in REPLAY_ENDS:
            s, c, pp = (np.ascontiguousarray(x) for x in (stream[a:b], codes[a * 8:b * 8], ppmd[a:b]))
            want = np.empty((b - a) * 8, dtype=np.float32)
            port.op_run(Q, s.ctypes.data, s.size, c.ctypes.data, pp.ctypes.data, want.ctypes.data)
            port.op_get_lstm_probs(Q, want_lstm.ctypes.data)
            got = P.code_bytes(s, c, pp)
            lstm = P.debug_fetch(DBG_LSTM_PROBS, (256,), np.float32)
            d = np.nonzero(lstm.view(np.uint32) != want_lstm.view(np.uint32))[0]
            assert d.size == 0, "%s: the LSTM's distribution after byte %d differs from the port's at symbol %d (%.9g vs %.9g)" % (
                name, b - 1, d[0], lstm[d[0]], want_lstm[d[0]])
            expect("%s: bulk [%d,%d), replayed" % (name, a, b), got, want, a * 8)
            a = b
    finally:
        P.close()
        port.op_destroy(Q)
