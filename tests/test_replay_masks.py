"""One model group replayed, the other resident: CMIXB200_REPLAY_PAQ8 is how image, PCM WAV audio and JPEG data code on
the device (the resident PAQ8 stops there with CMIXB200_ERR_UNSUPPORTED), and CMIXB200_REPLAY_FXCM is its twin.

The replayed group's codes are the reference's own, dumped at test time by oracle/_ref/oracle_dump from each fixture's
recipe (harness.reference_dumps): the fixtures keep only CRCs of them. The masks ("paq8",), ("fxcm",) and, as the control,
("fxcm", "paq8") run over the six PCM WAV fixtures past their first sample (so FXCM, PPMD, the LSTM, the small models and
the mixers meet the reference on audio data), full_text's text with a JFIF header in it, full_text and reach_fxwiki.
CPU (-m "not gpu"): each dump equals its committed fixture: stream, vocabulary, Predict() and code CRCs.
GPU (-m gpu, tolerance 0): bulk calls in several piece plans, bulk -> lock-step -> bulk, batches, the device encoder and a
lock-step decode, calls without codes (the replayed slots then carry p = 0.5), and the calls a replayed group refuses."""
import numpy as np
import pytest

from conftest import port_replay
from gen_wav import ENTRY, STREAMS
from harness import MAX_PIECE, awkward, cm, code_crcs, code_in_pieces, even, expect, first_bad_byte, golden, host_archive, \
    host_decode, lock_step, ppmd_arena, reference_dumps, target  # noqa: F401  (cm, ppmd_arena: fixtures)

WAVS = [n for n in STREAMS if n.startswith("wav_")]
FIXTURES = WAVS + ["full_text", "reach_fxwiki"]
MASKS = {"paq8": ("paq8",), "fxcm": ("fxcm",), "both": ("fxcm", "paq8")}
SLOTS = {"paq8": (431, 2022), "fxcm": (0, 431), "both": (0, 2022)}           # the replayed slots of each mask
PAQ8_STREAMS = WAVS + ["jfif_text", "full_text"]
FXCM_STREAMS = ["full_text", "reach_fxwiki"]
STREAMS_OF = {"paq8": PAQ8_STREAMS, "fxcm": FXCM_STREAMS, "both": PAQ8_STREAMS + ["reach_fxwiki"]}
CASES = [(m, n) for m in MASKS for n in STREAMS_OF[m]]
LOCK_SPAN = {**{n: (ENTRY - 8, ENTRY + 8) for n in WAVS}, "full_text": (2040, 2056), "jfif_text": (100, 124)}


@pytest.fixture(scope="module")
def dumps(tmp_path_factory):
    return reference_dumps(str(tmp_path_factory.mktemp("dumps")))


def replay_golden(dumps, name):
    """The dump as a fixture dict (stream, vocab, p, first_codes, crc_fx, crc_p8; ppmd_crc where the fixture has it) and
    its codes [bits][2022]."""
    d = dumps[name]
    g = golden(name) if name in FIXTURES else {"name": name}
    crc_fx, crc_p8 = code_crcs(d.ext)
    g.update(stream=d.stream, vocab=d.vocab, p=d.p, first_codes=d.ext[:64], crc_fx=crc_fx, crc_p8=crc_p8)
    return g, d.ext


def feeder(ext):
    """feed_external_bit of bit t's codes: what a caller of the lock-step surface passes before each Predict()."""
    return lambda P, t: P.feed_external_bit(ext[t])


# ------------------------------------------------------------------------------------------------ CPU
@pytest.mark.timeout(900)
@pytest.mark.parametrize("name", FIXTURES)
def test_dump_equals_the_fixture(dumps, name):
    """The codes these tests replay are the reference's that the committed fixture pins."""
    d, g = dumps[name], golden(name)
    n = g["stream"].size
    assert d.n_bytes == n and np.array_equal(d.stream, g["stream"]), "%s: coded stream: %s" % (name, first_bad_byte(d.stream, g["stream"]))
    assert np.array_equal(d.vocab, g["vocab"]), "%s: vocabulary" % name
    expect("%s: Predict() of the dump" % name, d.p, g["p"])
    for what, got, want in zip(("FXCM", "PAQ8"), code_crcs(d.ext), (g["crc_fx"], g["crc_p8"])):
        bad = np.nonzero(got != want)[0]
        assert got.size == want.size and bad.size == 0, "%s: %s codes: first differing 4096-bit block %s" % (name, what, bad[:1])


def test_jfif_text_holds_the_header():
    """jfif_text is `cmix -n`'s coded stream of full_text's first 400 bytes with a JFIF header at byte 103 of the file."""
    from harness import JFIF, reference_inputs
    data, mode, n = reference_inputs()["jfif_text"]
    assert mode == "n" and n == data.size + 5 and data.tobytes().find(JFIF) == 103


# ------------------------------------------------------------------------------------------------ GPU
def _plan(name, n, plan):
    if plan == "one":
        return [(0, n)]
    if plan == "awkward":                   # 1, 129, 7, 1000, 333 bytes, then pieces of at most 2048
        pieces = awkward(0, n)
        return pieces[:-1] + even(*pieces[-1])
    return [(0, 1000), (1000, n)]           # "cross": a call over 2048-byte pieces and the 4096-byte host staging


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("mask,name,plan", [(m, n, plan) for m, n in CASES
                                            for plan in ("one", "awkward") + (("cross",) if n == "full_text" else ())])
def test_bulk_equals_the_reference(cm, dumps, mask, name, plan):
    """Bulk calls from byte 0: Predict() of every bit and, for calls the debug fetch covers, every code the mixer staged."""
    g, ext = replay_golden(dumps, name)
    s = g["stream"]
    pieces = _plan(name, s.size, plan)
    P = cm.Predictor(g["vocab"], replay=MASKS[mask])
    try:
        if all(b - a <= MAX_PIECE for a, b in pieces):
            code_in_pieces(P, g, pieces, ext=ext)
        else:
            for a, b in pieces:
                expect("%s, %s: bulk [%d,%d)" % (name, MASKS[mask], a, b), P.code_bytes(s[a:b], ext[a * 8:b * 8]),
                       g["p"][a * 8:b * 8], a * 8)
    finally:
        P.close()


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("mask,name", CASES)
def test_bulk_lock_step_bulk(cm, dumps, mask, name):
    """Bulk calls to the span, Predict()/Perceive() with feed_external_bit before every Predict() across it (on the WAV
    streams: across the first sample), bulk calls to the end."""
    g, ext = replay_golden(dumps, name)
    s, p = g["stream"], g["p"]
    lo, hi = LOCK_SPAN[name] if name in LOCK_SPAN else target(name, s)
    what = "%s, %s" % (name, MASKS[mask])
    P = cm.Predictor(g["vocab"], replay=MASKS[mask])
    try:
        for a, b in awkward(0, lo):
            expect("%s: bulk [%d,%d)" % (what, a, b), P.code_bytes(s[a:b], ext[a * 8:b * 8]), p[a * 8:b * 8], a * 8)
        lock_step(P, g, lo * 8, hi * 8, "%s: [%d,%d)" % (what, lo, hi), feed=feeder(ext))
        for a, b in awkward(hi, s.size):
            expect("%s: bulk [%d,%d) after lock-step" % (what, a, b), P.code_bytes(s[a:b], ext[a * 8:b * 8]), p[a * 8:b * 8], a * 8)
    finally:
        P.close()


BATCHES = {"paq8": ["wav_pcm8_mono", "wav_pcm16_stereo", "wav_fmt18_list"], "fxcm": ["full_text", "reach_fxwiki", "full_text"]}
BATCHES["both"] = BATCHES["paq8"]


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("mask", MASKS)
def test_batches(cm, dumps, mask):
    """Three streams in one code_batch_device call, then on new predictors in one code_batch call from host buffers (its
    1024-byte staging)."""
    import torch
    from cmix_b200.capi import code_batch, code_batch_device
    runs = [replay_golden(dumps, x) for x in BATCHES[mask]]
    n = min(g["stream"].size for g, _ in runs)
    for entry in ("code_batch_device", "code_batch"):
        preds = []
        try:
            for g, _ in runs:
                preds.append(cm.Predictor(g["vocab"], replay=MASKS[mask]))
            if entry == "code_batch_device":
                dev = torch.device("cuda", 0)
                d_bytes = [torch.from_numpy(g["stream"][:n].copy()).to(dev) for g, _ in runs]
                d_ext = [torch.from_numpy(np.ascontiguousarray(e[:n * 8])).to(dev) for _, e in runs]
                d_out = [torch.empty(n * 8, dtype=torch.float32, device=dev) for _ in runs]
                code_batch_device(preds, d_bytes, n, d_ext, None, d_out)
                torch.cuda.synchronize()
                outs = [o.cpu().numpy() for o in d_out]
                del d_ext
            else:
                outs = [np.empty(n * 8, dtype=np.float32) for _ in runs]
                code_batch(preds, [np.ascontiguousarray(g["stream"][:n]) for g, _ in runs], n,
                           [np.ascontiguousarray(e[:n * 8]) for _, e in runs], None, outs)
            for (g, _), out in zip(runs, outs):
                expect("%s of %s, %s, %d bytes each: %s" % (entry, BATCHES[mask], MASKS[mask], n, g["name"]), out, g["p"][:n * 8])
        finally:
            for P in preds:
                P.close()


CODER = {"paq8": {"wav_pcm16_mono": ENTRY + 64, "jfif_text": None}, "fxcm": {"full_text": 256}}
CODER["both"] = CODER["paq8"]


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("mask,name", [(m, n) for m in MASKS for n in CODER[m]])
def test_device_coder_and_lock_step_decode(cm, port, dumps, mask, name):
    """The device encoder's archive equals the host encoder's over the reference's probabilities; the host decoder over
    lock-step Predict()/Perceive(), fed each bit's codes, gives the stream back (on the WAV: 64 bytes past its first sample)."""
    g, ext = replay_golden(dumps, name)
    s, p = g["stream"], g["p"]
    what = "%s, %s" % (name, MASKS[mask])
    enc = cm.Predictor(g["vocab"], replay=MASKS[mask])
    try:
        enc.coder_begin(2 * s.size + 64)
        expect("%s: encoder" % what, enc.code_bytes(s, ext), p)
        archive = enc.coder_finish()
    finally:
        enc.close()
    want = host_archive(port, p, np.unpackbits(s))
    assert archive == want, "%s: device archive differs from the host encoder's: %s" % (what, first_bad_byte(archive, want))
    n = CODER[mask][name] or s.size
    dec = cm.Predictor(g["vocab"], replay=MASKS[mask])
    try:
        out = host_decode(dec, archive, n, before_predict=feeder(ext))
    finally:
        dec.close()
    assert out == s[:n].tobytes(), "%s, decoder: %s" % (what, first_bad_byte(out, s[:n]))


HALF = {"paq8": ("jfif_text", (0, 100), (100, 140), (140, 200)), "fxcm": ("full_text", (0, 100), (100, 140), (140, 200))}
HALF["both"] = HALF["fxcm"]


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("mask", MASKS)
def test_a_call_without_codes_replays_half(cm, port, dumps, mask):
    """A call with codes, one without, one with: in the middle one the replayed slots carry p = 0.5 (0xFFFF), not what an
    earlier call staged. The resident groups' codes do not depend on the mixer, so the CPU port over the reference's codes,
    with the replayed slots at 0xFFFF over the middle call, is what the device must return."""
    name, first, middle, last = HALF[mask]
    g, ext = replay_golden(dumps, name)
    s, n = g["stream"], last[1]
    lo, hi = SLOTS[mask]
    want_ext = np.array(ext[:n * 8])
    want_ext[middle[0] * 8:middle[1] * 8, lo:hi] = 0xFFFF
    want = port_replay(port, g["vocab"], s[:n], want_ext, dumps[name].ppmd[:n])
    expect("%s: the port over the reference's codes, with them throughout" % name,
           port_replay(port, g["vocab"], s[:first[1]], ext[:first[1] * 8], dumps[name].ppmd[:first[1]]), g["p"][:first[1] * 8])
    P = cm.Predictor(g["vocab"], replay=MASKS[mask])
    try:
        for (a, b), codes in ((first, ext), (middle, None), (last, ext)):
            got = P.code_bytes(s[a:b], None if codes is None else codes[a * 8:b * 8])
            expect("%s, %s: bulk [%d,%d) %s codes" % (name, MASKS[mask], a, b, "without" if codes is None else "with"),
                   got, want[a * 8:b * 8], a * 8)
    finally:
        P.close()


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("mask", MASKS)
def test_refusals_leave_the_stream_as_it_was(cm, dumps, mask):
    """decode_bytes with a group replayed, and a batch whose predictors replay different groups, fail with
    CMIXB200_ERR_ARG; a bulk call after each continues from the same position with the reference's probabilities."""
    import torch
    from cmix_b200.capi import code_batch_device
    g, ext = replay_golden(dumps, "full_text")
    s, p = g["stream"], g["p"]
    what = "full_text, %s" % (MASKS[mask],)
    P = cm.Predictor(g["vocab"], replay=MASKS[mask])
    Q = None
    try:
        expect("%s: bulk [0,100)" % what, P.code_bytes(s[:100], ext[:800]), p[:800])
        with pytest.raises(RuntimeError, match=r"decode_bytes failed \(2\)"):
            P.decode_bytes(b"\0" * 64, 8)
        expect("%s: bulk [100,200) after decode_bytes failed" % what, P.code_bytes(s[100:200], ext[800:1600]), p[800:1600], 800)
        Q = cm.Predictor(g["vocab"])
        dev = torch.device("cuda", 0)
        d_bytes = [torch.from_numpy(s[200:300].copy()).to(dev) for _ in range(2)]
        d_out = [torch.empty(800, dtype=torch.float32, device=dev) for _ in range(2)]
        with pytest.raises(RuntimeError, match=r"code_batch_device failed \(2\)"):
            code_batch_device([P, Q], d_bytes, 100, None, None, d_out)
        expect("%s: bulk [200,300) after a mixed batch failed" % what, P.code_bytes(s[200:300], ext[1600:2400]), p[1600:2400], 1600)
    finally:
        P.close()
        if Q is not None:
            Q.close()
