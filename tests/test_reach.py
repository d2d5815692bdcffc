"""The complete resident predictor on streams built to run the lines of PAQ8, FXCM and PPMD no other fixture runs
(tools/gen_reach.py), and a line-coverage gate over those three model groups.

paq8_*.h, fxcm_model.h / fxcm_text.h and ppmd_model.h are single sources: the CUDA kernels compile the same headers the
host tools (tools/paq8_check.cpp, tools/fxcm_check.cpp, tools/ppmd_host.cpp) compile for the CPU. A line no fixture runs
on the host is therefore never checked on the device either. Fixtures tests/golden/reach_*.npz
(tools/make_reach_goldens.py) hold, in the layout of stress_*.npz, the reference's Predict() of every bit, CRCs of its FXCM
and PAQ8 codes per 4096 bits and of its PPMD distribution per byte, and the LSTM feedback FXCM saw.

CPU (-m "not gpu"): the host builds of PAQ8, FXCM and PPMD against those CRCs; the generator reproduces every stream; and
the gate: the merged line coverage of every fixture (tools/coverage_report.py) leaves no line of the three groups
unexecuted but those in ALLOWED. By default each fixture runs its first GATE_CAP bytes; CMIXB200_SLOW=1 runs 64 KiB of
each (the long_text* fixtures are longer).
GPU (-m gpu, tolerance 0): every fixture with everything resident in bulk calls; bulk calls of awkward sizes around a
lock-step stretch across the bytes each stream targets; three streams in one batch; a device encoder -> device decoder
round trip."""
import os
import zlib
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from conftest import ROOT
from gen_reach import STREAMS, coded_stream
from test_ppmd_model import ppmd_host  # noqa: F401  (fixture)
from test_stress_data import _check_host, _compile, _host_run

NAMES = list(STREAMS)
GATE_CAP = 65536 if os.environ.get("CMIXB200_SLOW") == "1" else 8192

# Lines of the three groups that no valid stream of a few KB runs. Each entry: (header, text of its first line, text of
# its last line or None for one line, reason). Texts are whole stripped lines, so an entry follows its code when lines move;
# a one-line entry covers every line with its text, a range starts at the only line with its first text and ends at the
# next line with its last text.
ALLOWED = [
    ("paq8_top.h", "case 0xAB: M.masks[2] += 5; break;", None,
     "bytes above 0x7F take the word branch of TextModel::Update first, in the reference too: the case is dead"),
    ("paq8_top.h", "case 0xBB: M.masks[2] += 10; break;", None, "as 0xAB"),
    ("paq8_top.h", "case XS_ParseFlags:", "break;",
     "no transition of the x86 parser enters ParseFlags, here or in the reference's exeModel"),
    ("paq8_top.h", "((buf(S, 1) & 0xFE) == 0xC0 || buf(S, 1) == 0xC4 || (buf(S, 1) >= 0xDB && buf(S, 1) <= 0xFE))) "
     "S.error |= ERR_UNSUPPORTED_BLOCK;", None,
     "a JPEG SOI with a plausible marker is an unsupported block: the model stops there, so no parity fixture holds one"),
    ("paq8_model.h", "} else d.extra += nn >> 10;", None,
     "a DMC node array full (2.6 million nodes or more at level 11) takes megabytes of data"),
    ("fxcm_model.h", "X.is_text = 0;", "X.nl1 = X.nl; X.nl = X.pos - 2;",
     "is_text is set only by the WRT dictionary's code word 'text' after '<' (a WRT-coded XML dump)"),
    ("ppmd_model.h", "if (!m.ctx[pc].suffix) return PPMD_CTX_BASE + pc;", "return m.pool[p].succ;",
     "ReduceOrder past the root: a state outside the root has no successor only after the reference's cutOff "
     "(RestoreModelRare, memory exhausted); the model reports an exhausted arena instead"),
]


def _fixture(name):
    z = np.load(os.path.join(ROOT, "tests", "golden", "reach_" + name + ".npz"))
    return {k: z[k] for k in z.files}


# ------------------------------------------------------------------------------------------------ CPU
@pytest.fixture(scope="module")
def host_runs(tmp_path_factory):
    """The host PAQ8 and FXCM builds over every reach fixture, in parallel."""
    tmp = str(tmp_path_factory.mktemp("reach"))
    p8 = _compile(tmp, "paq8_check", ["-ffp-contract=off"])
    fx = _compile(tmp, "fxcm_check")
    jobs = {}
    for name in NAMES:
        g = _fixture(name)
        jobs[("p8", name)] = (p8, "p8_" + name, g["stream"], None)
        jobs[("fx", name)] = (fx, "fx_" + name, g["stream"], g["lstmfx"])
    with ThreadPoolExecutor(os.cpu_count() or 4) as ex:
        futs = {k: ex.submit(_host_run, exe, tmp, label, s, l) for k, (exe, label, s, l) in jobs.items()}
        return {k: f.result() for k, f in futs.items()}


@pytest.mark.parametrize("name", NAMES)
def test_paq8_host_build_matches_reference_codes(host_runs, name):
    _check_host(host_runs[("p8", name)], _fixture(name)["crc_p8"], "reach_%s, PAQ8" % name)


@pytest.mark.parametrize("name", NAMES)
def test_fxcm_host_build_matches_reference_codes(host_runs, name):
    _check_host(host_runs[("fx", name)], _fixture(name)["crc_fx"], "reach_%s, FXCM" % name)


@pytest.mark.parametrize("name", NAMES)
def test_ppmd_host_build_matches_reference_distributions(ppmd_host, name):  # noqa: F811
    g = _fixture(name)
    rc, out = ppmd_host(g["stream"], g["vocab"])
    assert rc == 0
    got = np.array([zlib.crc32(out[t].tobytes()) for t in range(out.shape[0])], dtype=np.uint32)
    bad = np.nonzero(got != g["ppmd_crc"])[0]
    assert bad.size == 0, "reach_%s: first differing PPMD distribution after byte %d" % (name, bad[0])


@pytest.mark.parametrize("name", NAMES)
def test_generator_reproduces_the_fixture(name):
    g = _fixture(name)
    assert np.array_equal(coded_stream(name), g["stream"])
    assert g["vocab"].sum() == 256          # streams under 10000 bytes: the reference's vocabulary is every symbol


def _allowed_lines():
    """{(header, line number)} covered by ALLOWED; every entry must still name lines of its header."""
    from coverage_report import CSRC
    out, stale = set(), []
    for header, first, last, _ in ALLOWED:
        text = [t.strip() for t in open(os.path.join(CSRC, header)).read().split("\n")]
        starts = [i for i, t in enumerate(text) if t == first]
        if not starts or (last is not None and len(starts) > 1):
            stale.append("%s: %s (%d lines have this text)" % (header, first, len(starts)))
            continue
        for i in starts:
            j = i
            if last is not None:
                j = next((k for k in range(i, len(text)) if text[k] == last), None)
                if j is None:
                    stale.append("%s: %s ... %s" % (header, first, last))
                    continue
            out.update((header, k + 1) for k in range(i, j + 1))
    assert not stale, "allowlist entries that name no line, or no single first line: %s" % stale
    return out


@pytest.mark.timeout(1800)
def test_every_line_of_the_shared_models_runs_on_some_fixture():
    """The host builds with --coverage over every committed fixture (first GATE_CAP bytes each): each executable line of
    PAQ8, FXCM and PPMD must run on at least one, or be in ALLOWED with its reason."""
    from coverage_report import measure, unexecuted
    allowed = _allowed_lines()
    coverage, failures = measure(cap=GATE_CAP)
    assert not failures, "coverage runs failed:\n%s" % "\n".join(failures.values())
    assert all(coverage.get(t) for t in ("paq8", "fxcm", "ppmd")), "a model group produced no coverage data"
    missed = [(h, n, text) for _, h, n, text in unexecuted(coverage) if (h, n) not in allowed]
    for tool, files in coverage.items():
        print("%s: %d executable lines, %d unexecuted" % (tool, sum(len(v) for v in files.values()),
                                                         sum(1 for v in files.values() for c in v.values() if c == 0)))
    assert not missed, "%d lines of the shared models run on no fixture (first %d bytes of each):\n%s" % (
        len(missed), GATE_CAP, "\n".join("cmix_b200/csrc/%s:%d: %s" % m for m in missed))


# ------------------------------------------------------------------------------------------------ GPU
# the bytes each stream is built to reach: lock-step runs over [marker + lo, marker + hi)
TARGETS = {"english": (b"+\r\n", -8, 24), "europe": (b"travaux", -4, 20), "xml": (b"<![CDATA[", -4, 52),
           "x86": (b"\x0f\x3a", -4, 28), "dbase": (b"visual foxpro table\n", 18, 70),
           "bmp": (b"\x28\x00\x00\x00\x10\x00\x00\x00", 24, 48), "fxwiki": (b"PPQ", -4, 36)}


def _target(name, s):
    marker, lo, hi = TARGETS[name]
    at = s.tobytes().find(marker)
    assert at >= 0, "reach_%s: marker %r not in the stream" % (name, marker)
    return at + lo, min(at + hi, s.size)


@pytest.fixture(autouse=True)
def _ppmd_arena(monkeypatch):
    if "CMIXB200_PPMD_MB" not in os.environ:
        monkeypatch.setenv("CMIXB200_PPMD_MB", "512")      # three full predictors must fit in 80 GB


@pytest.fixture(scope="module")
def cm():
    import cmix_b200
    cmix_b200.load_library()
    return cmix_b200


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("name", NAMES)
def test_everything_resident_in_bulk(cm, name):
    """Bulk calls of 2048 bytes (a bulk call's debug codes cover its last 2048-byte piece): every Predict(), every FXCM
    and PAQ8 code and every PPMD distribution equal the reference's."""
    from test_stress_data import _mismatch_report
    g = _fixture(name)
    s = g["stream"]
    P = cm.Predictor(g["vocab"])
    ps, exts, ppmd_crc = [], [], []
    try:
        for off in range(0, s.size, 2048):
            part = s[off:off + 2048]
            ps.append(P.code_bytes(part))
            exts.append(P.debug_fetch(10, (part.size * 8, 2022), np.uint16))
            rows = P.debug_fetch(8, (part.size, 256), np.float32)
            ppmd_crc += [zlib.crc32(rows[t].tobytes()) for t in range(part.size)]
    finally:
        P.close()
    ext = np.concatenate(exts)
    crc_fx = np.array([zlib.crc32(np.ascontiguousarray(ext[b:b + 4096, :431]).tobytes()) for b in range(0, ext.shape[0], 4096)], dtype=np.uint32)
    crc_p8 = np.array([zlib.crc32(np.ascontiguousarray(ext[b:b + 4096, 431:]).tobytes()) for b in range(0, ext.shape[0], 4096)], dtype=np.uint32)
    report = _mismatch_report(name, g, np.concatenate(ps), crc_fx, crc_p8, ext[:64], np.array(ppmd_crc, dtype=np.uint32))
    if report:
        pytest.fail(report.replace("stress_", "reach_", 1), pytrace=False)


def _awkward(lo, hi):
    """Pieces of [lo, hi): 1, 129, 7, 1000, 333 bytes, then the rest."""
    out = []
    for n in (1, 129, 7, 1000, 333):
        if lo < hi:
            out.append((lo, min(lo + n, hi)))
            lo = out[-1][1]
    if lo < hi:
        out.append((lo, hi))
    return out


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("name", NAMES)
def test_lock_step_across_the_target_in_awkward_pieces(cm, name):
    """Bulk calls of awkward sizes up to the bytes the stream targets, lock-step Predict()/Perceive() across them, then
    bulk calls of awkward sizes to the end."""
    from test_call_schedules import _expect, _lock_step
    g = _fixture(name)
    s, p = g["stream"], g["p"]
    lo, hi = _target(name, s)
    P = cm.Predictor(g["vocab"])
    try:
        for a, b in _awkward(0, lo):
            _expect("reach_%s: bulk [%d,%d)" % (name, a, b), P.code_bytes(s[a:b]), p[a * 8:b * 8], a * 8)
        _lock_step(P, g, lo * 8, hi * 8, "reach_%s: lock-step [%d,%d)" % (name, lo, hi))
        for a, b in _awkward(hi, s.size):
            _expect("reach_%s: bulk [%d,%d) after lock-step" % (name, a, b), P.code_bytes(s[a:b]), p[a * 8:b * 8], a * 8)
    finally:
        P.close()


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("names", [("english", "europe", "xml"), ("x86", "dbase", "bmp"), ("fxwiki", "english", "x86")])
def test_three_streams_in_one_batch(cm, names):
    """Three streams of the same length side by side in one code_batch_device call (three predictors fit in 80 GB)."""
    import torch
    from cmix_b200.capi import code_batch_device
    from test_call_schedules import _expect
    gs = [_fixture(n) for n in names]
    n = min(g["stream"].size for g in gs)
    preds = []
    try:
        for g in gs:
            preds.append(cm.Predictor(g["vocab"]))
        dev = torch.device("cuda", 0)
        d_bytes = [torch.from_numpy(g["stream"][:n].copy()).to(dev) for g in gs]
        d_out = [torch.empty(n * 8, dtype=torch.float32, device=dev) for _ in gs]
        code_batch_device(preds, d_bytes, n, None, None, d_out)
        torch.cuda.synchronize()
        for g, out, name in zip(gs, d_out, names):
            _expect("batch of %s, %d bytes each: reach_%s" % (list(names), n, name), out.cpu().numpy(), g["p"][:n * 8])
    finally:
        for P in preds:
            P.close()


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("name", ["dbase", "fxwiki"])
def test_device_round_trip(cm, port, name):
    """The device coder writes the archive the host coder writes over the reference's probabilities; the device decoder
    gets the stream back."""
    from test_call_schedules import _expect, _first_bad_byte, _host_archive
    g = _fixture(name)
    s, p = g["stream"], g["p"]
    enc = cm.Predictor(g["vocab"])
    try:
        enc.coder_begin(2 * s.size + 64)
        _expect("reach_%s: encoder" % name, enc.code_bytes(s), p)
        archive = enc.coder_finish()
    finally:
        enc.close()
    want = _host_archive(port, p, np.unpackbits(s))
    assert archive == want, "reach_%s: device archive differs from the host encoder's: %s" % (name, _first_bad_byte(archive, want))
    dec = cm.Predictor(g["vocab"])
    try:
        out = dec.decode_bytes(archive, s.size)
    finally:
        dec.close()
    assert out.tobytes() == s.tobytes(), "reach_%s, decoder: %s" % (name, _first_bad_byte(out, s))
