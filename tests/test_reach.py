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

import numpy as np
import pytest

from gen_reach import STREAMS, coded_stream
from harness import awkward_lock_step, batch, build_host_tool, check_host, cm, code_in_pieces, even, golden, ppmd_arena, \
    ppmd_host, round_trip, run_host_tools  # noqa: F401  (cm, ppmd_arena, ppmd_host: fixtures)

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
    return golden("reach_" + name)


# ------------------------------------------------------------------------------------------------ CPU
@pytest.fixture(scope="module")
def host_runs(tmp_path_factory):
    """The host PAQ8 and FXCM builds over every reach fixture, in parallel."""
    tmp = str(tmp_path_factory.mktemp("reach"))
    p8 = build_host_tool("paq8_check", tmp, ["-DCENSUS"])
    fx = build_host_tool("fxcm_check", tmp, ["-DCENSUS"])
    jobs = {}
    for name in NAMES:
        g = _fixture(name)
        jobs[("p8", name)] = (p8, tmp, "p8_" + name, g["stream"], None)
        jobs[("fx", name)] = (fx, tmp, "fx_" + name, g["stream"], g["lstmfx"])
    return run_host_tools(jobs)


@pytest.mark.parametrize("name", NAMES)
def test_paq8_host_build_matches_reference_codes(host_runs, name):
    check_host(host_runs[("p8", name)], _fixture(name)["crc_p8"], "reach_%s, PAQ8" % name)


@pytest.mark.parametrize("name", NAMES)
def test_fxcm_host_build_matches_reference_codes(host_runs, name):
    check_host(host_runs[("fx", name)], _fixture(name)["crc_fx"], "reach_%s, FXCM" % name)


@pytest.mark.parametrize("name", NAMES)
def test_ppmd_host_build_matches_reference_distributions(ppmd_host, name):
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
@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("name", NAMES)
def test_everything_resident_in_bulk(cm, name):
    """Bulk calls of 2048 bytes (a bulk call's debug codes cover its last 2048-byte piece): every Predict(), every FXCM
    and PAQ8 code and every PPMD distribution equal the reference's."""
    g = _fixture(name)
    P = cm.Predictor(g["vocab"])
    try:
        code_in_pieces(P, g, even(0, g["stream"].size))
    finally:
        P.close()


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("name", NAMES)
def test_lock_step_across_the_target_in_awkward_pieces(cm, name):
    """Bulk calls of awkward sizes up to the bytes the stream targets, lock-step Predict()/Perceive() across them, then
    bulk calls of awkward sizes to the end."""
    awkward_lock_step(cm, "reach_" + name)


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("names", [("english", "europe", "xml"), ("x86", "dbase", "bmp"), ("fxwiki", "english", "x86")])
def test_three_streams_in_one_batch(cm, names):
    """Three streams of the same length side by side in one code_batch_device call (three predictors fit in 80 GB)."""
    batch(cm, ["reach_" + n for n in names])


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("name", ["dbase", "fxwiki"])
def test_device_round_trip(cm, port, name):
    """The device coder writes the archive the host coder writes over the reference's probabilities; the device decoder
    gets the stream back."""
    round_trip(cm, port, "reach_" + name)
