"""PAQ8's clash groups (paq8.cuh p8_number): on a bit where two contexts of a 7-slot map share a key (a 64-byte bucket on
bpos 0, 2 and 5, a slot on the staying bits), only the contexts that share a key with another context of their map (the
GROUPED ones) are walked by one lane, in program order over all clashing maps; the others (FREE) run on their own lanes
with their draw from the shared sequence and keep their slot-cache copies, as on a bit without a clash.

CPU (-m "not gpu"): host builds with -DCENSUS_GROUPS_PERMUTE=<seed> (tools/census.h p8_cm_groups_order: the free contexts of
every clashing map in a seeded random order interleaved with the grouped ones, each flagged context taking the draw of its
in-order rank) reproduce the reference's PAQ8 codes on full_text, full_bin, every stress_* and reach_* fixture and the 8-bit
audio and WAV fixtures. Those fixtures hold clashing bits at bpos 0, 2 and 5, a group of three or more contexts, two groups
in one map, groups in two maps on one bit and a staying-bit slot clash (stress_ramp).
GPU (-m gpu): the census build (-DCMIXB200_CENSUS) on the audio and WAV fixtures, which tests/test_device_census.py does not
run, in bulk calls, lock-step around the first bit with groups in two maps and the device decoder: every probability equals
the fixture's (tolerance 0), the device's PAQ8 records equal the host census's bit for bit, and no slot-cache copy differs
from HBM."""
import json
import os

import numpy as np
import pytest

from gen_audio8 import STREAMS as AUDIO8_STREAMS
from gen_reach import STREAMS as REACH_STREAMS
from gen_stress import STREAMS as STRESS_STREAMS
from harness import awkward_lock_step, build_host_tool, child_jobs, even, expect, golden, round_trip, run_child, run_host_tools

AUDIO = [n for n in AUDIO8_STREAMS if n != "audio8_then16"] + ["wav_pcm8_mono", "wav_pcm8_stereo"]
FIXTURES = ["full_text", "full_bin"] + ["stress_" + n for n in STRESS_STREAMS] + ["reach_" + n for n in REACH_STREAMS] + AUDIO
SEEDS = [0x6A0C1, 0x6A0C2, 0x6A0C3]
HEAD = ["cap", "p8_bits", "fx_bits", "bit_checked", "bit_filled", "slot_checks", "sm_checks", "mismatches", "first_set",
        "first_bit", "first_map", "first_ctx", "first_byte", "first_cached", "first_hbm", "overflow"]


def _host(tmp, names, defines=()):
    exe = build_host_tool("paq8_check", tmp, ["-DCENSUS", *defines])
    return run_host_tools({n: (exe, tmp, n, golden(n)["stream"]) for n in names}, log=True)


def _check_codes(runs):
    bad = []
    for n, r in sorted(runs.items()):
        want = golden(n)["crc_p8"]
        if r.rc != 0:
            bad.append("%s: exit %d: %s" % (n, r.rc, r.out[-800:]))
        elif r.crc.size != want.size or not np.array_equal(r.crc, want):
            d = np.nonzero(r.crc != want[:r.crc.size])[0]
            bad.append("%s: %d CRC blocks, expected %d; first differing 4096-bit block %s" % (n, r.crc.size, want.size, d[:1]))
    assert not bad, "\n".join(bad)


@pytest.fixture(scope="module")
def host_logs(tmp_path_factory):
    runs = _host(str(tmp_path_factory.mktemp("groups_logs")), FIXTURES)
    _check_codes(runs)
    return runs


@pytest.mark.timeout(1800)
@pytest.mark.parametrize("seed", SEEDS)
def test_grouped_in_order_and_free_in_any_order_match_the_reference(tmp_path_factory, seed):
    runs = _host(str(tmp_path_factory.mktemp("groups_permute")), FIXTURES, ["-DCENSUS_GROUPS_PERMUTE=%#x" % seed])
    _check_codes(runs)
    unpermuted = [n for n, r in runs.items() if r.census["clash7"] and not r.census["permuted"]]
    assert not unpermuted, "runs with clashing maps that permuted none: %s" % unpermuted
    print("seed %#x: %d clashing map-bits permuted" % (seed, sum(r.census["permuted"] for r in runs.values())))


def test_the_fixtures_reach_every_shape_of_group(host_logs):
    c = {n: r.census for n, r in host_logs.items()}
    for n, x in c.items():
        assert x["grouped"] >= 2 * x["clash7"], "%s: a clashing bit with fewer than two grouped contexts" % n
    bpos = np.sum([x["clash7_bpos"] for x in c.values()], axis=0)
    assert all(bpos[b] for b in (0, 2, 5)), "clashing bits per bpos: %s" % bpos.tolist()
    assert max(x["group_max"] for x in c.values()) >= 3, "no group of three or more contexts"
    assert sum(x["group_maps2"] for x in c.values()), "no map with two groups on one bit"
    two_maps = sum(int(np.sum([bin(int(w)).count("1") >= 2 for w in r.log[:, 0] & 0xFFFF])) for r in host_logs.values())
    assert two_maps, "no bit with groups in two maps"
    assert c["stress_ramp"]["clash7_stay"], "stress_ramp has no staying-bit slot clash"
    print("\n".join("%-20s clash bits %5d, grouped %6d, groups %5d, largest %2d, maps with two groups %4d" % (
        n, x["clash7"], x["grouped"], x["groups"], x["group_max"], x["group_maps2"]) for n, x in sorted(c.items())))


# ------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def census_lib(tmp_path_factory):
    from cmix_b200.capi import build_library
    return build_library(defines=["-DCMIXB200_CENSUS"], out_dir=str(tmp_path_factory.mktemp("census_lib")))


def _child(jobs_json, out_dir):
    """Child interpreter with CMIXB200_LIB = the census build: each job [schedule, [name, ...]] writes its logs to out_dir/j.npz."""
    import cmix_b200
    from test_device_census import _Census
    lib = cmix_b200.load_library()

    def run(j, job):
        sched, args = job
        g = golden(args[0])
        cm = _Census(lib, 8 * g["stream"].size)
        if sched == "bulk":
            P = cm.Predictor(g["vocab"])
            try:
                for a, b in even(0, g["stream"].size):
                    expect("%s: bulk [%d,%d)" % (args[0], a, b), P.code_bytes(g["stream"][a:b]), g["p"][a * 8:b * 8], a * 8)
            finally:
                P.close()
        elif sched == "lock":
            awkward_lock_step(cm, args[0], (args[1], args[2]), even)
        elif sched == "round_trip":
            round_trip(cm, None, args[0])
        else:
            raise ValueError(sched)
        if cm.errors:
            raise cm.errors[0]
        np.savez(os.path.join(out_dir, "%d.npz" % j), **{"%s_%d" % (k, i): v for i, lg in enumerate(cm.logs) for k, v in lg.items()})

    child_jobs(json.loads(jobs_json), run)


def _two_map_byte(log):
    t = np.nonzero([bin(int(w)).count("1") >= 2 for w in log[:, 0] & 0xFFFF])[0]
    assert t.size
    return int(t[0]) // 8


@pytest.mark.gpu
@pytest.mark.timeout(1800)
def test_device_groups_on_audio_and_wav(census_lib, host_logs, tmp_path):
    jobs = [["bulk", [n]] for n in AUDIO]
    for n in ("wav_pcm8_mono", "audio8_mono_text"):
        at = _two_map_byte(host_logs[n].log)
        jobs.append(["lock", [n, max(0, at - 8), at + 8]])
    jobs.append(["round_trip", ["wav_pcm8_stereo"]])
    results = run_child(census_lib, "test_paq8_clash_groups", "_child", [json.dumps(jobs), str(tmp_path)])
    fails = [("%s %s: %s" % (x["job"][0], x["job"][1], x["fail"])) for x in results if x["fail"]]
    for j, x in enumerate(results):
        if x["fail"]:
            continue
        z = np.load(os.path.join(str(tmp_path), "%d.npz" % j))
        name = x["job"][1][0]
        for i in range(2 if x["job"][0] == "round_trip" else 1):
            head = dict(zip(HEAD, (int(v) for v in z["head_%d" % i])))
            d8 = z["p8_%d" % i]
            h8 = host_logs[name].log[:d8.shape[0]]
            what = "%s %s%s" % (x["job"][0], name, " (decoder)" if i else "")
            if head["overflow"] or head["p8_bits"] != h8.shape[0]:
                fails.append("%s: %d PAQ8 bits logged (%d past the log), expected %d" % (what, head["p8_bits"], head["overflow"], h8.shape[0]))
                continue
            diff = np.nonzero((d8[:, 0] != h8[:, 0]) | (d8[:, 1] != h8[:, 1]))[0]
            if diff.size:
                t = int(diff[0])
                fails.append("%s: PAQ8 records differ on %d bits; first bit %d (byte %d): %#x %#x device, %#x %#x host" % (
                    what, diff.size, t, t // 8, d8[t, 0], d8[t, 1], h8[t, 0], h8[t, 1]))
            if head["mismatches"]:
                fails.append("%s: %d slot-cache reads differ from HBM; first at bit %d, map %d, context %d, byte %d" % (
                    what, head["mismatches"], head["first_bit"], head["first_map"], head["first_ctx"], head["first_byte"]))
    assert not fails, "\n".join(fails)
    assert len(results) == len(jobs), "%d of %d runs reported" % (len(results), len(jobs))
