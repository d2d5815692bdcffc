"""The complete resident predictor on degenerate, numeric, record and incompressible data (tools/gen_stress.py).

Text and x86 code seldom reach some device-only paths: the bucket-clash fallback of the context maps (paq8.cuh p8_number /
cm2_mix_body, fxcm.cuh `clash`), more than 24 draws of PAQ8's shared random sequence in one bit (p8_draw_at's replay and
p8_advance_rnd's chunks), the OLS predictors' floor() on smooth numeric data, long stretches of probabilities at the clamps, and
PPMD with all 256 symbols. Fixtures tests/golden/stress_*.npz (tools/make_stress_goldens.py) hold the reference's Predict() of
every bit, CRCs of its FXCM and PAQ8 codes per 4096 bits and of its PPMD distribution per byte, and the LSTM feedback FXCM saw.

CPU (-m "not gpu"): the host builds of PAQ8, FXCM and PPMD against those CRCs; the generator reproduces every stream; and a
census (tools/census.h) of how often the fixtures reach each device-only path, next to the same census of full_text/full_bin.
GPU (-m gpu, tolerance 0): every fixture with everything resident, in bulk calls of awkward sizes; lock-step then bulk; three
classes in one batch; and a device encoder -> device decoder round trip."""
import zlib

import numpy as np
import pytest

from gen_stress import STREAMS, coded_stream
from harness import batch, build_host_tool, check_host, cm, code_in_pieces, expect, golden, lock_step, ppmd_arena, ppmd_host, \
    round_trip, run_host_tools, stress_pieces  # noqa: F401  (cm, ppmd_arena, ppmd_host: fixtures)

NAMES = list(STREAMS)
# the existing whole-predictor fixtures, for comparison in the census (FXCM's LSTM feedback comes from fxcm_*.npz: same streams)
BASELINE = {"full_text": "fxcm_text", "full_bin": "fxcm_bin"}


def _fixture(name):
    return golden("stress_" + name)


# ------------------------------------------------------------------------------------------------ CPU
@pytest.fixture(scope="module")
def host_runs(tmp_path_factory):
    """The host PAQ8 and FXCM builds over every stress fixture and over full_text / full_bin, in parallel."""
    tmp = str(tmp_path_factory.mktemp("stress"))
    p8 = build_host_tool("paq8_check", tmp, ["-DCENSUS"])
    fx = build_host_tool("fxcm_check", tmp, ["-DCENSUS"])
    jobs = {}
    for name in NAMES:
        g = _fixture(name)
        jobs[("p8", name)] = (p8, tmp, "p8_" + name, g["stream"], None)
        jobs[("fx", name)] = (fx, tmp, "fx_" + name, g["stream"], g["lstmfx"])
    for name, fx_name in BASELINE.items():
        s, f = golden(name)["stream"], golden(fx_name)
        assert np.array_equal(f["stream"][:s.size], s)
        jobs[("p8", name)] = (p8, tmp, "p8_" + name, s, None)
        jobs[("fx", name)] = (fx, tmp, "fx_" + name, s, f["lstmfx"][:s.size * 8])
    return run_host_tools(jobs)


@pytest.mark.parametrize("name", NAMES)
def test_paq8_host_build_matches_reference_codes(host_runs, name):
    check_host(host_runs[("p8", name)], _fixture(name)["crc_p8"], "stress_%s, PAQ8" % name)


@pytest.mark.parametrize("name", NAMES)
def test_fxcm_host_build_matches_reference_codes(host_runs, name):
    check_host(host_runs[("fx", name)], _fixture(name)["crc_fx"], "stress_%s, FXCM" % name)


@pytest.mark.parametrize("name", NAMES)
def test_ppmd_host_build_matches_reference_distributions(ppmd_host, name):
    g = _fixture(name)
    rc, out = ppmd_host(g["stream"], g["vocab"])
    assert rc == 0
    got = np.array([zlib.crc32(out[t].tobytes()) for t in range(out.shape[0])], dtype=np.uint32)
    bad = np.nonzero(got != g["ppmd_crc"])[0]
    assert bad.size == 0, "stress_%s: first differing PPMD distribution after byte %d" % (name, bad[0])


@pytest.mark.parametrize("name", NAMES)
def test_generator_reproduces_the_fixture(name):
    g = _fixture(name)
    assert np.array_equal(coded_stream(name), g["stream"])
    assert g["vocab"].sum() == 256          # streams under 10000 bytes: the reference's vocabulary is every symbol


CENSUS_KEYS = [("p8", "clash7", "PAQ8 7-slot map clash (p8_number)"), ("p8", "clash_hist", "PAQ8 history map clash (cm2_mix_body)"),
               ("fx", "fx_clash", "FXCM map clash"), ("p8", "draw_bits", "bits with draws"), ("p8", "max_draws", "most draws in one bit"),
               ("p8", "gt24", "bits with > 24 draws"), ("p8", "gt24_fast", "... without a 7-slot clash (replay)")]


def test_census_reaches_every_device_only_path(host_runs):
    """Counts, per fixture, the coded bits that take each device-only path (the device's own rule applied by the host build,
    tools/census.h). The stress fixtures together must reach every path, and every map family's clash fallback."""
    rows = list(BASELINE) + NAMES
    census = {(m, n): host_runs[(m, n)].census for m in ("p8", "fx") for n in rows}
    assert all(c is not None for c in census.values()), "a host run printed no census"
    lines = ["%-38s" % "coded bits" + "".join("%11s" % n for n in rows) + "%11s" % "stress"]
    lines.append("%-38s" % "bits" + "".join("%11d" % census[("p8", n)]["bits"] for n in rows)
                 + "%11d" % sum(census[("p8", n)]["bits"] for n in NAMES))
    totals = {}
    for m, key, label in CENSUS_KEYS:
        vals = [census[(m, n)][key] for n in rows]
        totals[key] = (max if key == "max_draws" else sum)(census[(m, n)][key] for n in NAMES)
        lines.append("%-38s" % label + "".join("%11d" % v for v in vals) + "%11d" % totals[key])
    families = list(census[("p8", NAMES[0])]["maps"])            # PAQ8 maps in the device's order, then FXCM maps by id
    families += ["fxcm %d" % i for i in sorted(set(int(k.split()[1]) for n in rows for k in census[("fx", n)]["maps"]))]
    fam_totals = {}
    for fam in families:
        m = "fx" if fam.startswith("fxcm") else "p8"
        vals = [census[(m, n)]["maps"].get(fam, 0) for n in rows]
        fam_totals[fam] = sum(census[(m, n)]["maps"].get(fam, 0) for n in NAMES)
        lines.append("%-38s" % ("  clash bits, " + fam) + "".join("%11d" % v for v in vals) + "%11d" % fam_totals[fam])
    print("\n" + "\n".join(lines))
    missing = [label for m, key, label in CENSUS_KEYS if totals[key] == 0]
    assert not missing, "the stress fixtures never reach: %s" % missing
    assert totals["max_draws"] > 24
    p8_families = [f for f in fam_totals if f.startswith("p8")]
    assert len(p8_families) == 19
    never = [f for f in p8_families if fam_totals[f] == 0]
    assert not never, "no stress fixture reaches the clash fallback of %s" % never


# ------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("name", NAMES)
def test_everything_resident_in_awkward_pieces(cm, name):
    """Bulk calls of 1, 129, 1000, ... bytes put sub-chunk boundaries inside runs, records and samples."""
    g = _fixture(name)
    P = cm.Predictor(g["vocab"])
    try:
        code_in_pieces(P, g, stress_pieces(g["stream"].size))
    finally:
        P.close()


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("name", ["zeros", "random", "pcm16"])
def test_lock_step_then_bulk(cm, name):
    g = _fixture(name)
    P = cm.Predictor(g["vocab"])
    try:
        lock_step(P, g, 0, 64 * 8, "stress_%s: lock-step [0,64)" % name)
        expect("stress_%s: lock-step [0,64), bulk [64,%d)" % (name, g["stream"].size), P.code_bytes(g["stream"][64:]), g["p"][64 * 8:], 64 * 8)
    finally:
        P.close()


@pytest.mark.gpu
@pytest.mark.timeout(900)
def test_three_classes_in_one_batch(cm):
    """records, zeros (every context draws) and the mixed stream side by side in one code_batch_device call."""
    batch(cm, ["stress_records", "stress_zeros", "stress_mixed"])


@pytest.mark.gpu
@pytest.mark.timeout(900)
def test_device_round_trip_of_the_mixed_stream(cm, port):
    """The device coder writes the archive the host coder writes over the reference's probabilities; the device decoder
    gets the stream back."""
    round_trip(cm, port, "stress_mixed")
