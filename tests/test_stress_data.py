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
import json
import os
import subprocess
import zlib
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from conftest import ROOT
from gen_stress import STREAMS, coded_stream
from test_ppmd_model import ppmd_host  # noqa: F401  (fixture)

NAMES = list(STREAMS)
# the existing whole-predictor fixtures, for comparison in the census (FXCM's LSTM feedback comes from fxcm_*.npz: same streams)
BASELINE = {"full_text": "fxcm_text", "full_bin": "fxcm_bin"}


def _load(name):
    z = np.load(os.path.join(ROOT, "tests", "golden", name + ".npz"))
    return {k: z[k] for k in z.files}


def _fixture(name):
    return _load("stress_" + name)


# ------------------------------------------------------------------------------------------------ CPU
def _compile(tmp, tool, extra=()):
    exe = os.path.join(tmp, tool)
    subprocess.run(["g++", "-O2", "-std=c++17", "-DCENSUS", *extra, "-I", os.path.join(ROOT, "cmix_b200", "csrc"), "-I",
                    os.path.join(ROOT, "tools"), os.path.join(ROOT, "tools", tool + ".cpp"), "-o", exe], check=True)
    return exe


def _host_run(exe, tmp, label, stream, lstmfx=None):
    """One run of paq8_check / fxcm_check (built with -DCENSUS): (return code, output, CRCs per 4096 bits, census)."""
    prefix = os.path.join(tmp, label)
    stream.tofile(prefix + ".stream")
    if lstmfx is not None:
        lstmfx.tofile(prefix + ".lstmfx.u32")
    r = subprocess.run([exe, prefix, "-", str(stream.size), prefix + ".crc"], capture_output=True, text=True)
    census = [json.loads(line[len("census "):]) for line in r.stdout.splitlines() if line.startswith("census ")]
    crc = np.fromfile(prefix + ".crc", dtype=np.uint32) if os.path.exists(prefix + ".crc") else None
    return r.returncode, r.stdout + r.stderr, crc, census[0] if census else None


@pytest.fixture(scope="module")
def host_runs(tmp_path_factory):
    """The host PAQ8 and FXCM builds over every stress fixture and over full_text / full_bin, in parallel."""
    tmp = str(tmp_path_factory.mktemp("stress"))
    p8 = _compile(tmp, "paq8_check", ["-ffp-contract=off"])
    fx = _compile(tmp, "fxcm_check")
    jobs = {}
    for name in NAMES:
        g = _fixture(name)
        jobs[("p8", name)] = (p8, "p8_" + name, g["stream"], None)
        jobs[("fx", name)] = (fx, "fx_" + name, g["stream"], g["lstmfx"])
    for name, fx_name in BASELINE.items():
        s, f = _load(name)["stream"], _load(fx_name)
        assert np.array_equal(f["stream"][:s.size], s)
        jobs[("p8", name)] = (p8, "p8_" + name, s, None)
        jobs[("fx", name)] = (fx, "fx_" + name, s, f["lstmfx"][:s.size * 8])
    with ThreadPoolExecutor(os.cpu_count() or 4) as ex:
        futs = {k: ex.submit(_host_run, exe, tmp, label, s, l) for k, (exe, label, s, l) in jobs.items()}
        return {k: f.result() for k, f in futs.items()}


def _check_host(run, want, what):
    rc, out, crc, _ = run
    assert rc != 3, "%s: the stream trips PAQ8's image / audio / JPEG gate:\n%s" % (what, out[-2000:])
    assert rc == 0, "%s:\n%s" % (what, out[-2000:])
    bad = np.nonzero(crc != want[:crc.size])[0]
    assert crc.size == want.size and bad.size == 0, "%s: %d CRC blocks, expected %d; first differing 4096-bit block %s" % (
        what, crc.size, want.size, bad[:1])


@pytest.mark.parametrize("name", NAMES)
def test_paq8_host_build_matches_reference_codes(host_runs, name):
    _check_host(host_runs[("p8", name)], _fixture(name)["crc_p8"], "stress_%s, PAQ8" % name)


@pytest.mark.parametrize("name", NAMES)
def test_fxcm_host_build_matches_reference_codes(host_runs, name):
    _check_host(host_runs[("fx", name)], _fixture(name)["crc_fx"], "stress_%s, FXCM" % name)


@pytest.mark.parametrize("name", NAMES)
def test_ppmd_host_build_matches_reference_distributions(ppmd_host, name):  # noqa: F811
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
    census = {(m, n): host_runs[(m, n)][3] for m in ("p8", "fx") for n in rows}
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
@pytest.fixture(autouse=True)
def _ppmd_arena(monkeypatch):
    if "CMIXB200_PPMD_MB" not in os.environ:
        monkeypatch.setenv("CMIXB200_PPMD_MB", "512")      # three full predictors must fit in 80 GB


@pytest.fixture(scope="module")
def cm():
    import cmix_b200
    cmix_b200.load_library()
    return cmix_b200


def _pieces(n):
    """1, 129 and 1000 bytes, then pieces of at most 2000 (a bulk call's debug codes cover its last 2048-byte piece only)."""
    sizes = [1, 129, 1000]
    while sum(sizes) < n:
        sizes.append(min(2000, n - sum(sizes)))
    return sizes


def _mismatch_report(name, g, p, crc_fx, crc_p8, first, ppmd_crc):
    """Every way the device run differs from the fixture, each with its first bit / byte / 4096-bit block."""
    out = []
    d = np.nonzero(p.view(np.uint32) != g["p"].view(np.uint32))[0]
    if d.size:
        k = int(d[0])
        out.append("Predict(): first differing bit %d (byte %d, block %d; %.9g vs %.9g; %d bits differ)"
                   % (k, k // 8, k // 4096, p[k], g["p"][k], d.size))
    bad = np.argwhere(first != g["first_codes"])
    if bad.size:
        out.append("codes of the first 64 bits: first differing (bit, slot) %s" % (bad[0].tolist(),))
    for what, got, want in (("FXCM", crc_fx, g["crc_fx"]), ("PAQ8", crc_p8, g["crc_p8"])):
        b = np.nonzero(got != want)[0]
        if b.size:
            out.append("%s codes: first differing block %d (bits %d..%d)" % (what, b[0], b[0] * 4096, b[0] * 4096 + 4095))
    b = np.nonzero(ppmd_crc != g["ppmd_crc"])[0]
    if b.size:
        out.append("PPMD distribution: first differing after byte %d" % b[0])
    return ("stress_%s: " % name + "; ".join(out)) if out else None


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("name", NAMES)
def test_everything_resident_in_awkward_pieces(cm, name):
    """Bulk calls of 1, 129, 1000, ... bytes put sub-chunk boundaries inside runs, records and samples."""
    g = _fixture(name)
    s = g["stream"]
    P = cm.Predictor(g["vocab"])
    ps, exts, ppmd_crc = [], [], []
    try:
        off = 0
        for n in _pieces(s.size):
            ps.append(P.code_bytes(s[off:off + n]))
            exts.append(P.debug_fetch(10, (n * 8, 2022), np.uint16))
            rows = P.debug_fetch(8, (n, 256), np.float32)
            ppmd_crc += [zlib.crc32(rows[t].tobytes()) for t in range(n)]
            off += n
    finally:
        P.close()
    ext = np.concatenate(exts)
    crc_fx = np.array([zlib.crc32(np.ascontiguousarray(ext[b:b + 4096, :431]).tobytes()) for b in range(0, ext.shape[0], 4096)], dtype=np.uint32)
    crc_p8 = np.array([zlib.crc32(np.ascontiguousarray(ext[b:b + 4096, 431:]).tobytes()) for b in range(0, ext.shape[0], 4096)], dtype=np.uint32)
    report = _mismatch_report(name, g, np.concatenate(ps), crc_fx, crc_p8, ext[:64], np.array(ppmd_crc, dtype=np.uint32))
    if report:
        pytest.fail(report, pytrace=False)


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("name", ["zeros", "random", "pcm16"])
def test_lock_step_then_bulk(cm, name):
    from test_call_schedules import _expect, _lock_step
    g = _fixture(name)
    P = cm.Predictor(g["vocab"])
    try:
        _lock_step(P, g, 0, 64 * 8, "stress_%s: lock-step [0,64)" % name)
        _expect("stress_%s: lock-step [0,64), bulk [64,%d)" % (name, g["stream"].size), P.code_bytes(g["stream"][64:]), g["p"][64 * 8:], 64 * 8)
    finally:
        P.close()


@pytest.mark.gpu
@pytest.mark.timeout(900)
def test_three_classes_in_one_batch(cm):
    """records, zeros (every context draws) and the mixed stream side by side in one code_batch_device call."""
    import torch
    from cmix_b200.capi import code_batch_device
    from test_call_schedules import _expect
    names = ["records", "zeros", "mixed"]
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
            _expect("batch of %s, %d bytes each: stress_%s" % (names, n, name), out.cpu().numpy(), g["p"][:n * 8])
    finally:
        for P in preds:
            P.close()


@pytest.mark.gpu
@pytest.mark.timeout(900)
def test_device_round_trip_of_the_mixed_stream(cm, port):
    """The device coder writes the archive the host coder writes over the reference's probabilities; the device decoder
    gets the stream back."""
    from test_call_schedules import _expect, _first_bad_byte, _host_archive
    g = _fixture("mixed")
    s, p = g["stream"], g["p"]
    enc = cm.Predictor(g["vocab"])
    try:
        enc.coder_begin(2 * s.size + 64)
        _expect("stress_mixed: encoder", enc.code_bytes(s), p)
        archive = enc.coder_finish()
    finally:
        enc.close()
    want = _host_archive(port, p, np.unpackbits(s))
    assert archive == want, "stress_mixed: device archive differs from the host encoder's: %s" % _first_bad_byte(archive, want)
    dec = cm.Predictor(g["vocab"])
    try:
        out = dec.decode_bytes(archive, s.size)
    finally:
        dec.close()
    assert out.tobytes() == s.tobytes(), "stress_mixed, decoder: %s" % _first_bad_byte(out, s)
