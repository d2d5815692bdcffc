"""nvcc contracts no multiply-add in the device code (DESIGN.md §2).

The reference rounds every float product before it adds it, so a contracted a * b + c (one FFMA, one rounding) moves a
probability. Every such operation on the device is written with explicit rounding intrinsics (__fmul_rn, __fadd_rn, ...)
that nvcc may not fuse. This test compiles each device unit to sm_90a machine code with the product's flags, with and
without -fmad=false: if nothing is left for nvcc to contract, the two are the same. The FFMAs that remain come from the
expansions of the IEEE intrinsics (__fdiv_rn, ...) and the explicit fused XM_DFMA; -fmad=false keeps them too. Needs
nvcc, no GPU."""
import os
import subprocess
from concurrent.futures import ThreadPoolExecutor

import pytest

from cmix_b200.capi import NVCC_COMPILE, UNITS
from harness import CSRC, sass_by_function


def _first_difference(a, b):
    """(function, first differing SASS line with and without -fmad=false) of two cubins, or None."""
    fa, fb = sass_by_function(a), sass_by_function(b)
    for name in sorted(set(fa) | set(fb)):
        la, lb = fa.get(name, "").splitlines(), fb.get(name, "").splitlines()
        for x, y in zip(la + [""] * len(lb), lb + [""] * len(la)):
            if x != y:
                return name, x, y
    return None


@pytest.mark.timeout(900)
def test_device_units_are_the_same_with_fmad_false(tmp_path):
    flags = [f for f in NVCC_COMPILE if f != "-lineinfo"]     # line tables are not code

    def compile_(unit, extra):
        out = str(tmp_path / ("%s%s.cubin" % (unit[:-3], "".join(extra))))
        r = subprocess.run(["nvcc"] + flags + extra + ["-cubin", os.path.join(CSRC, unit), "-o", out], capture_output=True, text=True)
        assert r.returncode == 0, "nvcc %s %s:\n%s" % (unit, " ".join(extra), r.stderr[-3000:])
        return out

    jobs = [(u, e) for u in UNITS for e in ((), ("-fmad=false",))]
    with ThreadPoolExecutor(len(jobs)) as ex:                  # the six compiles side by side
        cubins = dict(zip(jobs, ex.map(lambda j: compile_(j[0], list(j[1])), jobs)))
    contracted = []
    for u in UNITS:
        plain, strict = cubins[(u, ())], cubins[(u, ("-fmad=false",))]
        with open(plain, "rb") as f, open(strict, "rb") as g:
            if f.read() == g.read():
                continue
        d = _first_difference(plain, strict)
        contracted.append("%s: %s" % (u, "kernel %s: `%s` becomes `%s` with -fmad=false" % d if d else
                                      "the cubins differ outside the SASS"))
    assert not contracted, "nvcc contracts a multiply-add:\n" + "\n".join(contracted)
