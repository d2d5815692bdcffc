"""PAQ8's slot-granular clash rule for the 7-slot context maps on staying bits (paq8_model.h cm_slot_keys).

On bpos 1, 3, 4, 6 and 7 no context of a 7-slot map moves to a new bucket or updates its run record, so the device checks
two contexts of one map for a clash by the slots they read and write instead of by whole 64-byte buckets; a map that still
clashes walks serially (p8_number / cm_mix). CPU only:
  * the census (tools/census.h, the device's rule on the host) finds no staying-bit clash in full_text / full_bin, while the
    stress fixtures still reach the serial walk on such a bit;
  * a host build that evaluates the contexts of every clash-free map of a staying bit in REVERSE order (each flagged
    context taking the draw of its in-order rank, as the device's lanes do) reproduces the reference's PAQ8 codes.
tests/test_device_census.py generalises the second test to a seeded random order on every bit, in the history maps and
FXCM's maps too (-DCENSUS_PERMUTE), and pins the device's per-bit verdicts to this census."""
import numpy as np
import pytest

from gen_stress import STREAMS
from harness import build_host_tool, golden, run_host_tools

STRESS = ["stress_" + n for n in STREAMS]
BASELINE = ["full_text", "full_bin"]


def _runs(tmp, exe, names):
    return run_host_tools({n: (exe, tmp, n, golden(n)["stream"]) for n in names})


@pytest.fixture(scope="module")
def census_runs(tmp_path_factory):
    tmp = str(tmp_path_factory.mktemp("slot_census"))
    return _runs(tmp, build_host_tool("paq8_check", tmp, ["-DCENSUS"]), BASELINE + STRESS)


def test_staying_bits_clash_only_in_the_stress_fixtures(census_runs):
    rows = BASELINE + STRESS
    census = {n: census_runs[n].census for n in rows}
    assert all(c is not None for c in census.values()), "a host run printed no census"
    lines = ["%-16s %-7s" % ("7-slot clash bits", "rule") + "".join("%8s" % ("bpos %d" % b) for b in range(8))]
    for n in rows:
        for key, rule in (("bucket7_bpos", "bucket"), ("clash7_bpos", "device")):
            lines.append("%-16s %-7s" % (n, rule) + "".join("%8d" % v for v in census[n][key]))
    print("\n" + "\n".join(lines))
    for n in rows:
        c = census[n]
        assert c["clash7_stay"] == sum(c["clash7_bpos"][b] for b in (1, 3, 4, 6, 7))
        assert c["clash7"] == sum(c["clash7_bpos"])
        assert all(c["clash7_bpos"][b] <= c["bucket7_bpos"][b] for b in range(8)), n
        assert all(c["clash7_bpos"][b] == c["bucket7_bpos"][b] for b in (0, 2, 5)), "%s: the bucket rule stays on the move bits" % n
    for n in BASELINE:
        assert census[n]["clash7_stay"] == 0, "%s: %d staying bits clash under the slot rule" % (n, census[n]["clash7_stay"])
    assert sum(census[n]["clash7_stay"] for n in STRESS) > 0, "no fixture reaches the serial walk on a staying bit"


def test_reverse_order_on_clash_free_staying_bits_matches_the_reference(tmp_path_factory):
    tmp = str(tmp_path_factory.mktemp("slot_reverse"))
    exe = build_host_tool("paq8_check", tmp, ["-DCENSUS", "-DCENSUS_REVERSE"])
    runs = _runs(tmp, exe, BASELINE + STRESS)
    for n in BASELINE + STRESS:
        rc, out, crc = runs[n][:3]
        assert rc == 0, "%s:\n%s" % (n, out[-2000:])
        want = golden(n)["crc_p8"]
        bad = np.nonzero(crc != want[:crc.size])[0]
        assert crc.size == want.size and bad.size == 0, "%s: %d CRC blocks, expected %d; first differing 4096-bit block %s" % (
            n, crc.size, want.size, bad[:1])
