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
import time

import numpy as np
import pytest

from gen_reach import STREAMS as REACH_STREAMS
from gen_stress import STREAMS as STRESS_STREAMS
from harness import awkward, awkward_lock_step, batch, build_host_tool, child_jobs, even, expect, golden, round_trip, run_child, \
    run_host_tools

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


def _lstmfx(name, g):
    return golden(FX_FEEDBACK[name])["lstmfx"][:g["stream"].size * 8] if name in FX_FEEDBACK else g["lstmfx"]


def _staying(bp):
    return (0xDA >> bp) & 1


# ------------------------------------------------------------------------------------------------ host logs
def _host_runs(tmp, defines=()):
    """The host PAQ8 and FXCM builds over every fixture, in parallel, with their per-bit logs: {("p8" | "fx", name): HostRun}."""
    p8 = build_host_tool("paq8_check", tmp, ["-DCENSUS", *defines])
    fx = build_host_tool("fxcm_check", tmp, ["-DCENSUS", *defines])
    jobs = {}
    for n in FIXTURES:
        g = golden(n)
        jobs[("p8", n)] = (p8, tmp, "p8_" + n, g["stream"], None)
        jobs[("fx", n)] = (fx, tmp, "fx_" + n, g["stream"], _lstmfx(n, g))
    return run_host_tools(jobs, log=True)


def _check_codes(runs, names):
    """Every run exits 0 and its CRCs equal the reference's."""
    bad = []
    for (m, n), (rc, out, crc, _, _) in sorted(runs.items()):
        if n not in names:
            continue
        want = golden(n)["crc_p8" if m == "p8" else "crc_fx"]
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
        c8, log8 = host_logs[("p8", n)].census, host_logs[("p8", n)].log
        cfx, logfx = host_logs[("fx", n)].census, host_logs[("fx", n)].log
        assert log8 is not None and logfx is not None, "%s: a host run wrote no per-bit log" % n
        assert log8.shape[0] == logfx.size == golden(n)["stream"].size * 8, n
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
        log8, logfx = host_logs[("p8", n)].log, host_logs[("fx", n)].log
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
    unpermuted = [k for k, r in runs.items() if not r.census or r.census["permuted"] == 0]
    assert not unpermuted, "runs that permuted no map: %s" % unpermuted
    print("seed %#x: %d PAQ8 and %d FXCM map-bits permuted" % (seed, sum(r.census["permuted"] for k, r in runs.items() if k[0] == "p8"),
                                                               sum(r.census["permuted"] for k, r in runs.items() if k[0] == "fx")))


# ------------------------------------------------------------------------------------------------ the census build
@pytest.fixture(scope="module")
def census_lib(tmp_path_factory):
    """The library compiled with -DCMIXB200_CENSUS into this module's tmp dir."""
    from cmix_b200.capi import build_library
    return build_library(defines=["-DCMIXB200_CENSUS"], out_dir=str(tmp_path_factory.mktemp("census_lib")))


# ------------------------------------------------------------------------------------------------ GPU: child side
class _Census:
    """Stands in for the cmix_b200 module in the harness's schedules: each Predictor attaches a census log of n_bits on
    creation and reads it back into `logs` when it closes (census build only). A failed read is kept in `errors`, not
    raised from close(), so that it cannot replace the failure that brought a schedule into its `finally`."""

    def __init__(self, lib, n_bits):
        import cmix_b200
        census, self.logs, self.errors = self, [], []

        def call(what, rc):
            if rc != 0:
                raise RuntimeError("census %s: %s" % (what, lib.cmixb200_last_error().decode()))

        class Predictor(cmix_b200.Predictor):
            def __init__(self, *args, **kw):
                super().__init__(*args, **kw)
                try:
                    call("attach", lib.cmixb200_census_attach(self._h, ctypes.c_uint(n_bits)))
                except BaseException:
                    cmix_b200.Predictor.close(self)
                    raise

            def close(self):
                try:
                    if getattr(self, "_h", None):
                        head = np.zeros(16, dtype=np.uint32)
                        p8 = np.zeros((n_bits, 3), dtype=np.uint32)
                        fx = np.zeros(n_bits, dtype=np.uint32)
                        call("read", lib.cmixb200_census_read(self._h, head.ctypes.data, p8.ctypes.data, fx.ctypes.data,
                                                              ctypes.c_size_t(n_bits)))
                        census.logs.append({"head": head, "p8": p8, "fx": fx})
                except RuntimeError as e:
                    census.errors.append(e)
                finally:
                    super().close()
        self.Predictor = Predictor


def _child(jobs_json, out_dir):
    """Run in a child interpreter with CMIXB200_LIB = the census build: each job is [schedule, args]; writes the logs of
    job j to out_dir/j.npz and prints one JSON line per job."""
    import cmix_b200
    lib = cmix_b200.load_library()

    def run(j, job):
        sched, args = job
        names = args if sched == "batch" else args[:1]
        cm = _Census(lib, 8 * min(golden(n)["stream"].size for n in names))
        if sched in ("bulk", "awkward"):
            g = golden(args[0])
            s, p = g["stream"], g["p"]
            P = cm.Predictor(g["vocab"])
            try:
                for a, b in (even if sched == "bulk" else awkward)(0, s.size):
                    expect("%s: bulk [%d,%d)" % (args[0], a, b), P.code_bytes(s[a:b]), p[a * 8:b * 8], a * 8)
            finally:
                P.close()
        elif sched == "lock":
            awkward_lock_step(cm, args[0], (args[1], args[2]), even)
        elif sched == "batch":
            batch(cm, args)
        elif sched == "round_trip":
            round_trip(cm, None, args[0])
        else:
            raise ValueError(sched)
        if cm.errors:
            raise cm.errors[0]
        np.savez(os.path.join(out_dir, "%d.npz" % j), **{"%s_%d" % (k, i): v for i, lg in enumerate(cm.logs) for k, v in lg.items()})

    child_jobs(json.loads(jobs_json), run)


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
    out_dir = str(tmp)
    t0 = time.perf_counter()
    results = run_child(census_lib, "test_device_census", "_child", [json.dumps(jobs), out_dir], timeout=timeout)
    fails = []
    print("\n%-12s %-44s %7s %7s %7s %9s %9s %9s" % ("schedule", "stream", "clash7", "hist", "fxcm", "copies", "sm words", "fills"))
    for j, x in enumerate(results):
        sched, args = x["job"]
        if x["fail"]:
            fails.append("%s %s: %s" % (sched, args, x["fail"]))
            continue
        z = np.load(os.path.join(out_dir, "%d.npz" % j))
        names = {"batch": args, "round_trip": [args[0]] * 2}.get(sched, [args[0]])
        for i, name in enumerate(names):
            dev = {k: z["%s_%d" % (k, i)] for k in ("head", "p8", "fx")}
            n = dev["p8"].shape[0]
            host8, hostfx = host_logs[("p8", name)].log[:n], host_logs[("fx", name)].log[:n]
            what = "%s %s%s" % (sched, name, " (decoder)" if sched == "round_trip" and i else "")
            lock = (args[1] * 8, args[2] * 8) if sched == "lock" else None
            f, row = _compare(what, dev, host8, hostfx, lock)
            fails += f
            if row:
                print("%-12s %-44s %7d %7d %7d %9d %9d %9d" % ((sched, name + (" (decoder)" if sched == "round_trip" and i else "")) + row))
    print("%s: %d runs in %.0f s" % (label, len(results), time.perf_counter() - t0))
    assert not fails, "%s: %d differences:\n%s" % (label, len(fails), "\n".join(fails))
    assert len(results) == len(jobs), "%s: %d of %d runs reported" % (label, len(results), len(jobs))


def _first_slot_clash(host_logs, name):
    """The byte of the first staying-bit slot clash of a fixture (host log)."""
    f = _p8_fields(host_logs[("p8", name)].log)
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
