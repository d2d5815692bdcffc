"""The device's per-bit clash verdicts and PAQ8's slot cache, pinned to the host census (tools/census.h).

paq8.cuh and fxcm.cuh run the contexts of a context map on separate lanes and walk a map serially only when the per-bit
check finds a clash; on the staying bits PAQ8's 7-slot lanes read their slot and run record from a copy in shared memory
(P8CmCache). A device that flags more clashes than the rule only loses time, and one that flags fewer, or reads a stale copy,
may still code every fixture correctly: parity alone does not pin either. Built with -DCMIXB200_CENSUS
(cmix_b200/csrc/census.cuh) the kernels log per coded bit and stream the clashing maps, the flagged draws and the copies
checked and filled, and compare every copy a staying bit reads with HBM. The host tools built with -DCENSUS write the same
records (CENSUS_LOG).

CPU (-m "not gpu"): the census build compiles for sm_90a and exports cmixb200_census_*, the product library does not; the
host per-bit logs add up to the census JSON line on full_text, full_bin, every stress_* and every reach_* fixture; those
fixtures hold bits where the slot rule and the bucket rule disagree, staying-bit slot clashes, history-map and FXCM clashes;
and host builds that evaluate every clash-free map in a seeded random order (-DCENSUS_PERMUTE, every bit, all three map
families) reproduce the reference's PAQ8 and FXCM codes on all of them.
GPU (-m gpu): the census library in child interpreters (CMIXB200_LIB). Every probability equals the fixture's (tolerance 0),
the device's records equal the host's bit for bit, no copy differs from HBM, and on a lock-step bit (fresh shared memory)
the probe fills every copy it checks. Schedules: bulk calls of 2048 bytes, awkward bulk pieces, lock-step stretches around
the first staying-bit slot clashes, three streams in one batch, and the device decoder's graph."""
import ctypes
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from conftest import ROOT
from gen_reach import STREAMS as REACH_STREAMS
from gen_stress import STREAMS as STRESS_STREAMS
from test_stress_data import _compile

CSRC = os.path.join(ROOT, "cmix_b200", "csrc")
UNITS = ["engine.cu", "fxcm_dev.cu", "paq8_dev.cu"]
EXPORTS = ["cmixb200_census_attach", "cmixb200_census_read", "cmixb200_census_reset", "cmixb200_census_detach"]
STRESS = ["stress_" + n for n in STRESS_STREAMS]
REACH = ["reach_" + n for n in REACH_STREAMS]
FIXTURES = ["full_text", "full_bin"] + STRESS + REACH
FX_FEEDBACK = {"full_text": "fxcm_text", "full_bin": "fxcm_bin"}   # the LSTM feedback FXCM saw on the full_* streams
SEEDS = [0x5EED0101, 0x5EED0202]
SLOT_CLASH = ["stress_ramp", "stress_nested", "stress_mixed"]      # the fixtures with staying-bit slot clashes
P8_NAMES = ["sparse", "sparse1", "distance", "record.cm", "record.cn", "record.co", "record.cp", "record1.cm", "record1.cn",
            "record1.co", "record1.cq", "record1.cp", "word", "nest", "indirect", "xml", "order-n (history)", "text (history)",
            "exe (history)"]
HEAD = ["cap", "p8_bits", "fx_bits", "bit_checked", "bit_filled", "slot_checks", "sm_checks", "mismatches", "first_set",
        "first_bit", "first_map", "first_ctx", "first_byte", "first_cached", "first_hbm", "overflow"]


def _load(name):
    z = np.load(os.path.join(ROOT, "tests", "golden", name + ".npz"))
    return {k: z[k] for k in z.files}


def _lstmfx(name, g):
    return _load(FX_FEEDBACK[name])["lstmfx"][:g["stream"].size * 8] if name in FX_FEEDBACK else g["lstmfx"]


def _staying(bp):
    return (0xDA >> bp) & 1


# ------------------------------------------------------------------------------------------------ host logs
def _host_log(exe, tmp, label, stream, lstmfx=None):
    """One run of paq8_check / fxcm_check built with -DCENSUS: (return code, output, CRCs per 4096 bits, census, log)."""
    prefix = os.path.join(tmp, label)
    stream.tofile(prefix + ".stream")
    if lstmfx is not None:
        lstmfx.tofile(prefix + ".lstmfx.u32")
    env = dict(os.environ, CENSUS_LOG=prefix + ".log")
    r = subprocess.run([exe, prefix, "-", str(stream.size), prefix + ".crc"], capture_output=True, text=True, env=env)
    census = [json.loads(line[len("census "):]) for line in r.stdout.splitlines() if line.startswith("census ")]
    crc = np.fromfile(prefix + ".crc", dtype=np.uint32) if os.path.exists(prefix + ".crc") else None
    log = np.fromfile(prefix + ".log", dtype=np.uint32) if os.path.exists(prefix + ".log") else None
    if log is not None and lstmfx is None:
        log = log.reshape(-1, 3)
    return r.returncode, r.stdout + r.stderr, crc, census[0] if census else None, log


def _host_runs(tmp, defines=()):
    """The host PAQ8 and FXCM builds over every fixture, in parallel: {("p8" | "fx", name): _host_log(...)}."""
    p8 = _compile(tmp, "paq8_check", ["-ffp-contract=off", *defines])
    fx = _compile(tmp, "fxcm_check", list(defines))
    jobs = {}
    for n in FIXTURES:
        g = _load(n)
        jobs[("p8", n)] = (p8, "p8_" + n, g["stream"], None)
        jobs[("fx", n)] = (fx, "fx_" + n, g["stream"], _lstmfx(n, g))
    with ThreadPoolExecutor(os.cpu_count() or 4) as ex:
        futs = {k: ex.submit(_host_log, exe, tmp, label, s, l) for k, (exe, label, s, l) in jobs.items()}
        return {k: f.result() for k, f in futs.items()}


def _check_codes(runs, names):
    """Every run exits 0 and its CRCs equal the reference's."""
    bad = []
    for (m, n), (rc, out, crc, _, _) in sorted(runs.items()):
        if n not in names:
            continue
        want = _load(n)["crc_p8" if m == "p8" else "crc_fx"]
        if rc != 0:
            bad.append("%s %s: exit %d: %s" % (m, n, rc, out[-800:]))
        elif crc.size != want.size or not np.array_equal(crc, want):
            d = np.nonzero(crc != want[:crc.size])[0]
            bad.append("%s %s: %d CRC blocks, expected %d; first differing 4096-bit block %s" % (m, n, crc.size, want.size, d[:1]))
    assert not bad, "\n".join(bad)


@pytest.fixture(scope="module")
def host_logs(tmp_path_factory):
    runs = _host_runs(str(tmp_path_factory.mktemp("census_logs")))
    _check_codes(runs, FIXTURES)
    return runs


def _p8_fields(log):
    w0, w1 = log[:, 0], log[:, 1]
    return {"mask7": w0 & 0xFFFF, "hist": (w0 >> 16) & 7, "bp": (w0 >> 20) & 7, "draws": w1 & 0xFFFF, "checked": w1 >> 16}


def _totals(p8_log, fx_log):
    """The census JSON line's counts, recomputed from the per-bit logs."""
    f = _p8_fields(p8_log)
    clash, stay, draws, bucket = f["mask7"] != 0, np.array([_staying(b) for b in range(8)])[f["bp"]] == 1, f["draws"], p8_log[:, 2] != 0
    out = {"bits": int(p8_log.shape[0]), "draw_bits": int(np.sum(draws > 0)), "max_draws": int(draws.max(initial=0)),
           "gt24": int(np.sum(draws > 24)), "gt24_fast": int(np.sum((draws > 24) & ~clash)), "clash7": int(clash.sum()),
           "clash7_stay": int(np.sum(clash & stay)), "clash_hist": int(np.sum(f["hist"] != 0)),
           "clash7_bpos": [int(np.sum(clash & (f["bp"] == b))) for b in range(8)],
           "bucket7_bpos": [int(np.sum(bucket & (f["bp"] == b))) for b in range(8)]}
    maps = {"p8 " + nm: int(np.sum((p8_log[:, 0] >> k) & 1)) for k, nm in enumerate(P8_NAMES)}
    fx_maps = {"fxcm %d" % k: int(np.sum((fx_log >> k) & 1)) for k in range(31)}
    return out, maps, {k: v for k, v in fx_maps.items() if v}, int(np.sum(fx_log != 0))


def test_census_build_exports_and_the_product_does_not(census_lib):
    import cmix_b200
    lib = ctypes.CDLL(census_lib)
    missing = [e for e in EXPORTS if not hasattr(lib, e)]
    assert not missing, "the census build does not export %s" % missing
    prod = ctypes.CDLL(cmix_b200.build_library())
    leaked = [e for e in EXPORTS if hasattr(prod, e)]
    assert not leaked, "the product library exports %s" % leaked


def test_host_logs_agree_with_the_census_totals(host_logs):
    bad = []
    for n in FIXTURES:
        _, _, _, c8, log8 = host_logs[("p8", n)]
        _, _, _, cfx, logfx = host_logs[("fx", n)]
        assert log8 is not None and logfx is not None, "%s: a host run wrote no per-bit log" % n
        assert log8.shape[0] == logfx.size == _load(n)["stream"].size * 8, n
        totals, maps, fx_maps, fx_clash = _totals(log8, logfx)
        for k, v in totals.items():
            if c8[k] != v:
                bad.append("%s: %s %s in the JSON line, %s from the per-bit log" % (n, k, c8[k], v))
        if {k: v for k, v in c8["maps"].items()} != maps:
            bad.append("%s: PAQ8 per-map clash bits differ: %s vs %s" % (n, c8["maps"], maps))
        if cfx["fx_clash"] != fx_clash or cfx["maps"] != fx_maps:
            bad.append("%s: FXCM clash bits differ: %s %s vs %s %s" % (n, cfx["fx_clash"], cfx["maps"], fx_clash, fx_maps))
        f = _p8_fields(log8)
        stay = np.array([_staying(b) for b in range(8)])[f["bp"]] == 1
        assert np.all(f["checked"][~stay] == 0), "%s: copies checked on a move bit" % n
    assert not bad, "\n".join(bad)


def test_the_fixtures_discriminate(host_logs):
    """A device on the bucket rule, one that never serialises a map family, or one that serialises everything would
    differ from these logs somewhere."""
    rows, sums = [], {"rule": 0, "stay": 0, "hist": 0, "fx": 0, "serial_free": 0}
    for n in FIXTURES:
        log8, logfx = host_logs[("p8", n)][4], host_logs[("fx", n)][4]
        f = _p8_fields(log8)
        stay = np.array([_staying(b) for b in range(8)])[f["bp"]] == 1
        rule = int(np.sum(stay & (f["mask7"] != log8[:, 2])))      # staying bits where the slot and bucket rules disagree
        r = {"rule": rule, "stay": int(np.sum(stay & (f["mask7"] != 0))), "hist": int(np.sum(f["hist"] != 0)),
             "fx": int(np.sum(logfx != 0)), "serial_free": int(np.sum((f["mask7"] == 0) & (f["hist"] == 0)))}
        rows.append("%-16s" % n + "".join("%10d" % r[k] for k in sums))
        for k in sums:
            sums[k] += r[k]
    print("\n%-16s" % "bits" + "".join("%10s" % k for k in sums) + "\n" + "\n".join(rows))
    missing = [k for k, v in sums.items() if v == 0]
    assert not missing, "no fixture has a bit of kind %s" % missing


@pytest.mark.timeout(1800)
@pytest.mark.parametrize("seed", SEEDS)
def test_permuted_builds_match_the_reference(tmp_path_factory, seed):
    """Every clash-free map of every bit evaluated in a seeded random order (7-slot, history and FXCM maps; each flagged
    7-slot context takes the draw of its in-order rank): the codes stay the reference's, so the rule's verdicts make the
    contexts of a map commute on these fixtures."""
    runs = _host_runs(str(tmp_path_factory.mktemp("census_permute")), ["-DCENSUS_PERMUTE=%#x" % seed])
    _check_codes(runs, FIXTURES)
    unpermuted = [k for k, r in runs.items() if not r[3] or r[3]["permuted"] == 0]
    assert not unpermuted, "runs that permuted no map: %s" % unpermuted
    print("seed %#x: %d PAQ8 and %d FXCM map-bits permuted" % (seed, sum(r[3]["permuted"] for k, r in runs.items() if k[0] == "p8"),
                                                               sum(r[3]["permuted"] for k, r in runs.items() if k[0] == "fx")))


# ------------------------------------------------------------------------------------------------ the census build
@pytest.fixture(scope="module")
def census_lib(tmp_path_factory):
    """The library compiled with -DCMIXB200_CENSUS into this module's tmp dir."""
    from cmix_b200.capi import NVCC_COMPILE, NVCC_LINK
    out = tmp_path_factory.mktemp("census_lib")
    objs, jobs = [], []
    for u in UNITS:
        obj = str(out / (u[:-3] + ".o"))
        objs.append(obj)
        jobs.append(subprocess.Popen(["nvcc"] + NVCC_COMPILE + ["-DCMIXB200_CENSUS", "-c", os.path.join(CSRC, u), "-o", obj]))
    assert all(j.wait() == 0 for j in jobs), "nvcc failed on the census build"
    lib = str(out / "libcmixb200_census.so")
    subprocess.run(["nvcc"] + NVCC_LINK + objs + ["-o", lib], check=True)
    return lib


# ------------------------------------------------------------------------------------------------ GPU: child side
class _Log:
    """The census log of one predictor (census build only)."""

    def __init__(self, lib, P, n_bits):
        self.lib, self.P, self.n = lib, P, n_bits
        self._call("attach", lib.cmixb200_census_attach(P._h, ctypes.c_uint(n_bits)))

    def _call(self, what, rc):
        if rc != 0:
            raise RuntimeError("census %s: %s" % (what, self.lib.cmixb200_last_error().decode()))

    def read(self):
        head = np.zeros(16, dtype=np.uint32)
        p8 = np.zeros((self.n, 3), dtype=np.uint32)
        fx = np.zeros(self.n, dtype=np.uint32)
        self._call("read", self.lib.cmixb200_census_read(self.P._h, head.ctypes.data, p8.ctypes.data, fx.ctypes.data, ctypes.c_size_t(self.n)))
        return {"head": head, "p8": p8, "fx": fx}


def _bulk(cm, lib, name, pieces):
    from test_call_schedules import _expect
    g = _load(name)
    s, p = g["stream"], g["p"]
    P = cm.Predictor(g["vocab"])
    try:
        log = _Log(lib, P, s.size * 8)
        for a, b in pieces(s.size):
            _expect("%s: bulk [%d,%d)" % (name, a, b), P.code_bytes(s[a:b]), p[a * 8:b * 8], a * 8)
        return [log.read()]
    finally:
        P.close()


def _lock(cm, lib, name, lo, hi):
    """Bulk calls of 2048 bytes to byte lo, lock-step Predict()/Perceive() over [lo, hi), bulk calls to the end."""
    from test_call_schedules import _expect, _lock_step
    g = _load(name)
    s, p = g["stream"], g["p"]
    P = cm.Predictor(g["vocab"])
    try:
        log = _Log(lib, P, s.size * 8)
        for a in range(0, lo, 2048):
            b = min(a + 2048, lo)
            _expect("%s: bulk [%d,%d)" % (name, a, b), P.code_bytes(s[a:b]), p[a * 8:b * 8], a * 8)
        _lock_step(P, g, lo * 8, hi * 8, "%s: [%d,%d)" % (name, lo, hi))
        for a in range(hi, s.size, 2048):
            b = min(a + 2048, s.size)
            _expect("%s: bulk [%d,%d) after lock-step" % (name, a, b), P.code_bytes(s[a:b]), p[a * 8:b * 8], a * 8)
        return [log.read()]
    finally:
        P.close()


def _batch(cm, lib, names):
    import torch
    from cmix_b200.capi import code_batch_device
    from test_call_schedules import _expect
    gs = [_load(x) for x in names]
    n = min(g["stream"].size for g in gs)
    preds = []
    try:
        for g in gs:
            preds.append(cm.Predictor(g["vocab"]))
        logs = [_Log(lib, P, n * 8) for P in preds]
        dev = torch.device("cuda", 0)
        d_bytes = [torch.from_numpy(g["stream"][:n].copy()).to(dev) for g in gs]
        d_out = [torch.empty(n * 8, dtype=torch.float32, device=dev) for _ in gs]
        code_batch_device(preds, d_bytes, n, None, None, d_out)
        torch.cuda.synchronize()
        for g, out, x in zip(gs, d_out, names):
            _expect("batch of %s, %d bytes each: %s" % (list(names), n, x), out.cpu().numpy(), g["p"][:n * 8])
        return [log.read() for log in logs]
    finally:
        for P in preds:
            P.close()


def _round_trip(cm, lib, name):
    """Device encoder -> device decoder; the logs of both."""
    from test_call_schedules import _expect, _first_bad_byte
    g = _load(name)
    s, p = g["stream"], g["p"]
    enc = cm.Predictor(g["vocab"])
    try:
        log = _Log(lib, enc, s.size * 8)
        enc.coder_begin(2 * s.size + 64)
        _expect("%s: encoder" % name, enc.code_bytes(s), p)
        archive = enc.coder_finish()
        logs = [log.read()]
    finally:
        enc.close()
    dec = cm.Predictor(g["vocab"])
    try:
        log = _Log(lib, dec, s.size * 8)
        out = dec.decode_bytes(archive, s.size)
        assert out.tobytes() == s.tobytes(), "%s, decoder: %s" % (name, _first_bad_byte(out, s))
        return logs + [log.read()]
    finally:
        dec.close()


def _child(jobs_json, out_dir):
    """Run in a child interpreter with CMIXB200_LIB = the census build: each job is [schedule, args]; writes the logs of
    job j to out_dir/j.npz and prints one JSON line per job."""
    import cmix_b200
    from test_reach import _awkward
    lib = cmix_b200.load_library()
    for j, (sched, args) in enumerate(json.loads(jobs_json)):
        t0 = time.perf_counter()
        try:
            if sched == "bulk":
                logs = _bulk(cmix_b200, lib, args[0], lambda n: [(a, min(a + 2048, n)) for a in range(0, n, 2048)])
            elif sched == "awkward":
                logs = _bulk(cmix_b200, lib, args[0], lambda n: _awkward(0, n))
            elif sched == "lock":
                logs = _lock(cmix_b200, lib, *args)
            elif sched == "batch":
                logs = _batch(cmix_b200, lib, args)
            elif sched == "round_trip":
                logs = _round_trip(cmix_b200, lib, args[0])
            else:
                raise ValueError(sched)
            np.savez(os.path.join(out_dir, "%d.npz" % j), **{"%s_%d" % (k, i): v for i, lg in enumerate(logs) for k, v in lg.items()})
            msg = None
        except BaseException as e:      # pytest.fail raises an exception outside pytest's Exception tree
            msg = "%s: %s" % (type(e).__name__, e)
        print(json.dumps({"sched": sched, "args": args, "s": round(time.perf_counter() - t0, 2), "fail": msg}), flush=True)
        if msg and ("CUDA" in msg or "cuda" in msg):
            break                        # the context may be gone: report, do not go on


# ------------------------------------------------------------------------------------------------ GPU: parent side
def _compare(label, dev, host8, hostfx, lock=None):
    """The device's log against the host's; lock = (lo, hi) bits coded in lock-step. Returns failures and a summary row."""
    head = dict(zip(HEAD, (int(v) for v in dev["head"])))
    n = host8.shape[0]
    fails = []
    if head["overflow"] or head["p8_bits"] != n or head["fx_bits"] != n:
        fails.append("%s: %d PAQ8 / %d FXCM bits logged (%d past the log), expected %d" % (label, head["p8_bits"], head["fx_bits"], head["overflow"], n))
        return fails, None
    d8, dfx = dev["p8"], dev["fx"]
    diff = np.nonzero((d8[:, 0] != host8[:, 0]) | (d8[:, 1] != host8[:, 1]))[0]
    if diff.size:
        t = int(diff[0])
        fd, fh = _p8_fields(d8[t:t + 1]), _p8_fields(host8[t:t + 1])
        fails.append("%s: PAQ8 verdicts differ on %d bits; first bit %d (byte %d, bpos %d): 7-slot maps %#06x device / %#06x host, "
                     "history maps %#x / %#x, draws %d / %d, copies checked %d / %d" % (
                         label, diff.size, t, t // 8, t % 8, fd["mask7"][0], fh["mask7"][0], fd["hist"][0], fh["hist"][0],
                         fd["draws"][0], fh["draws"][0], fd["checked"][0], fh["checked"][0]))
    diff = np.nonzero(dfx != hostfx)[0]
    if diff.size:
        t = int(diff[0])
        fails.append("%s: FXCM verdicts differ on %d bits; first bit %d (byte %d, bpos %d): maps %#010x device / %#010x host" % (
            label, diff.size, t, t // 8, t % 8, dfx[t], hostfx[t]))
    if head["mismatches"]:
        fails.append("%s: %d slot-cache reads differ from HBM; first at bit %d, map %s, context %d, byte %d (0-6 slot, 7-8 run "
                     "record, 9-10 StateMap words): cached %d, HBM %d" % (
                         label, head["mismatches"], head["first_bit"], P8_NAMES[head["first_map"]], head["first_ctx"],
                         head["first_byte"], head["first_cached"], head["first_hbm"]))
    f = _p8_fields(d8)
    if lock is not None:
        lo, hi = lock
        short = [t for t in range(lo, hi) if d8[t, 2] != f["checked"][t]]
        if short:
            t = short[0]
            fails.append("%s: lock-step bit %d (bpos %d): the probe filled %d of %d copies (shared memory is new at every launch)" % (
                label, t, t % 8, d8[t, 2], f["checked"][t]))
    row = (int(np.sum(f["mask7"] != 0)), int(np.sum(f["hist"] != 0)), int(np.sum(dfx != 0)), head["slot_checks"],
           head["sm_checks"], int(d8[:, 2].sum()))
    return fails, row


def _run(census_lib, host_logs, label, jobs, tmp, timeout=1500):
    """The jobs in a child interpreter; each job's logs compared with the host's. Fails with every difference."""
    import gc
    import torch
    gc.collect()
    torch.cuda.empty_cache()
    out_dir = str(tmp)
    e = dict(os.environ, CMIXB200_LIB=census_lib)
    e.setdefault("CMIXB200_PPMD_MB", "512")
    code = "import sys; sys.path[:0] = sys.argv[1:4]; import test_device_census as m; m._child(sys.argv[4], sys.argv[5])"
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [
        "-c", code, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools"), ROOT, json.dumps(jobs), out_dir]
    t0 = time.perf_counter()
    r = subprocess.run(cmd, env=e, cwd=ROOT, capture_output=True, text=True, timeout=timeout)
    results = [json.loads(line) for line in r.stdout.splitlines() if line.startswith("{")]
    fails = []
    print("\n%-12s %-44s %7s %7s %7s %9s %9s %9s" % ("schedule", "stream", "clash7", "hist", "fxcm", "copies", "sm words", "fills"))
    for j, x in enumerate(results):
        if x["fail"]:
            fails.append("%s %s: %s" % (x["sched"], x["args"], x["fail"]))
            continue
        z = np.load(os.path.join(out_dir, "%d.npz" % j))
        names = {"batch": x["args"], "round_trip": [x["args"][0]] * 2}.get(x["sched"], [x["args"][0]])
        for i, name in enumerate(names):
            dev = {k: z["%s_%d" % (k, i)] for k in ("head", "p8", "fx")}
            n = dev["p8"].shape[0]
            host8, hostfx = host_logs[("p8", name)][4][:n], host_logs[("fx", name)][4][:n]
            what = "%s %s%s" % (x["sched"], name, " (decoder)" if x["sched"] == "round_trip" and i else "")
            lock = (x["args"][1] * 8, x["args"][2] * 8) if x["sched"] == "lock" else None
            f, row = _compare(what, dev, host8, hostfx, lock)
            fails += f
            if row:
                print("%-12s %-44s %7d %7d %7d %9d %9d %9d" % ((x["sched"], name + (" (decoder)" if x["sched"] == "round_trip" and i else "")) + row))
    print("%s: %d runs in %.0f s" % (label, len(results), time.perf_counter() - t0))
    assert r.returncode == 0, "%s: child failed:\n%s\n%s" % (label, r.stdout[-3000:], r.stderr[-3000:])
    assert not fails, "%s: %d differences:\n%s" % (label, len(fails), "\n".join(fails))
    assert len(results) == len(jobs), "%s: %d of %d runs reported" % (label, len(results), len(jobs))


def _first_slot_clash(host_logs, name):
    """The byte of the first staying-bit slot clash of a fixture (host log)."""
    f = _p8_fields(host_logs[("p8", name)][4])
    stay = np.array([_staying(b) for b in range(8)])[f["bp"]] == 1
    t = np.nonzero(stay & (f["mask7"] != 0))[0]
    assert t.size, "%s has no staying-bit slot clash" % name
    return int(t[0]) // 8


@pytest.mark.gpu
@pytest.mark.timeout(1800)
def test_device_verdicts_in_bulk(census_lib, host_logs, tmp_path):
    """Bulk calls of 2048 bytes over full_text, full_bin, every stress_* and every reach_* fixture."""
    _run(census_lib, host_logs, "bulk", [["bulk", [n]] for n in FIXTURES], tmp_path)


@pytest.mark.gpu
@pytest.mark.timeout(1800)
def test_device_verdicts_in_awkward_pieces_and_lock_step(census_lib, host_logs, tmp_path):
    """Bulk pieces of 1, 129, 7, 1000, 333 bytes (launches start at many positions relative to the cache's fill points), and
    lock-step over the 16 bytes around the first staying-bit slot clash of each fixture that has one: on a lock-step bit the
    probe fills every copy it checks."""
    jobs = [["awkward", [n]] for n in SLOT_CLASH + ["full_text"]]
    for n in SLOT_CLASH:
        at = _first_slot_clash(host_logs, n)
        jobs.append(["lock", [n, max(0, at - 8), at + 8]])
    _run(census_lib, host_logs, "awkward / lock-step", jobs, tmp_path)


@pytest.mark.gpu
@pytest.mark.timeout(1800)
def test_device_verdicts_in_a_batch_and_the_decoder(census_lib, host_logs, tmp_path):
    """Three streams in one code_batch_device call, each with its own log; a device encoder -> device decoder round trip,
    whose graph runs the lock-step kernels."""
    _run(census_lib, host_logs, "batch / decoder", [["batch", SLOT_CLASH], ["round_trip", ["stress_ramp"]]], tmp_path)
