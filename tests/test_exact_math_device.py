"""cmix_b200/csrc/exact_math.h (xm_expf, xm_expm1f, xm_tanhf, xm_logistic) on every input.

These four functions carry every logistic and LSTM gate, so each must return the reference's bits on the device as on
the host. The host build (g++ -ffp-contract=off, tests/exact_math_sweep.cpp) is the reference of the device build
(nvcc with the product's flags, tests/exact_math_sweep.cu); the host build in turn is pinned to glibc, which the
reference calls.

CPU: the host build against glibc on the special classes (zeros, denormals, infinities, NaN payloads, the overflow and
underflow thresholds, the branch points of expm1f and tanhf and their neighbours); over all 2^32 inputs with
CMIXB200_SLOW=1 (it wants many cores).
GPU (-m gpu): the device build against the host build on the special classes, and on all 2^32 inputs in chunks of 2^26
with one checksum per 2^16 inputs; a differing checksum is resolved to the first differing input."""
import ctypes
import os
import subprocess
import time

import numpy as np
import pytest

from conftest import ROOT

FUNCS = ["expf", "expm1f", "tanhf", "logistic"]
BLK_LOG2 = 16                      # XS_SUB_LOG2: one checksum per function and 2^16 consecutive inputs
CHUNK_BLKS = 1 << (26 - BLK_LOG2)  # 2^26 inputs per chunk
N_BLKS = 1 << (32 - BLK_LOG2)
SRC = os.path.join(ROOT, "tests")


def _f32_bits(x):
    return int(np.array(x, dtype=np.float32).view(np.uint32))


def special_inputs():
    """Bit patterns of the classes where a libm restatement goes wrong, each with its neighbours and both signs."""
    centres = [
        0x00000000, 0x00000001, 0x00000002, 0x00400000, 0x007fffff, 0x00800000,   # zero, denormals, smallest normal
        0x3f800000, 0x7f7fffff,                                                    # 1, largest finite
        0x7f800000, 0x7f800001, 0x7fa00000, 0x7fc00000, 0x7fc00001, 0x7fffffff,    # inf, signalling and quiet NaN payloads
        _f32_bits(float.fromhex("0x1.62e42ep6")),     # expf overflows above this
        _f32_bits(float.fromhex("0x1.9fe368p6")),     # expf underflows below minus this
        0x42b00000,                                   # |x| >= 88: xm_expf's special-case branch
        0x33000000, 0x3eb17218, 0x3f851592, 0x4195b844, 0x42b17218,   # expm1f: 2^-25, 0.5 ln2, 1.5 ln2, 27 ln2, 88.72
        _f32_bits(8.8721679688e+01),                  # expm1f's overflow threshold
        _f32_bits(23 * np.log(2)), _f32_bits(56.5 * np.log(2)),       # expm1f: k = 23 and k > 56 reconstructions
        0x24000000, 0x41b00000,                       # tanhf: 2^-55, 22
        _f32_bits(0.5), _f32_bits(0.25),              # expm1f's x < -0.25 split of k = 1
    ]
    out = set()
    for c in centres:
        for d in range(-3, 4):
            u = (c + d) & 0x7fffffff
            if c + d >= 0:
                out.add(u)
                out.add(u | 0x80000000)
    return np.array(sorted(out), dtype=np.uint32)


@pytest.fixture(scope="module")
def host_lib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("xm_host") / "libxs_host.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fopenmp", "-fPIC", "-shared",
                    os.path.join(SRC, "exact_math_sweep.cpp"), "-o", so, "-lm"], check=True)
    lib = ctypes.CDLL(so)
    c = ctypes
    lib.xs_host_sums.argtypes = [c.c_uint32, c.c_uint32, c.c_void_p]
    lib.xs_host_eval.argtypes = [c.c_void_p, c.c_size_t, c.c_void_p]
    lib.xs_libm_eval.argtypes = [c.c_void_p, c.c_size_t, c.c_void_p]
    lib.xs_libm_sweep.argtypes = [c.c_uint32, c.c_uint32, c.c_void_p, c.c_void_p]
    for f in (lib.xs_host_sums, lib.xs_host_eval, lib.xs_libm_eval, lib.xs_libm_sweep):
        f.restype = None
    return lib


@pytest.fixture(scope="module")
def device_lib(tmp_path_factory):
    from cmix_b200.capi import NVCC_COMPILE
    so = str(tmp_path_factory.mktemp("xm_dev") / "libxs_dev.so")
    subprocess.run(["nvcc"] + NVCC_COMPILE + ["-shared", os.path.join(SRC, "exact_math_sweep.cu"), "-o", so], check=True)
    lib = ctypes.CDLL(so)
    c = ctypes
    lib.xs_device_sums.argtypes = [c.c_uint32, c.c_uint32, c.c_void_p]
    lib.xs_device_eval.argtypes = [c.c_void_p, c.c_size_t, c.c_void_p]
    return lib


def _eval(fn, inputs):
    """[4][n] result bits of fn (xs_host_eval / xs_libm_eval / xs_device_eval) over the input bit patterns."""
    inputs = np.ascontiguousarray(inputs, dtype=np.uint32)
    out = np.empty((len(FUNCS), inputs.size), dtype=np.uint32)
    rc = fn(inputs.ctypes.data, inputs.size, out.ctypes.data)
    assert not rc, "CUDA error %d" % rc            # host functions return None
    return out


def _first_difference(got, want, inputs, what):
    """None, or a message naming the first input at which got and want ([4][n] result bits) differ."""
    bad = np.argwhere(got != want)
    if bad.size == 0:
        return None
    f, i = (int(v) for v in bad[np.argsort(bad[:, 1], kind="stable")][0])
    x = inputs[i]
    return "%s: %s(%a) [bits %08x] = %08x, expected %08x (%d differences)" % (
        what, FUNCS[f], float(np.array(x, dtype=np.uint32).view(np.float32)), x, got[f, i], want[f, i], bad.shape[0])


# ------------------------------------------------------------------------------------------------ CPU
def test_host_build_matches_libm_on_special_classes(host_lib):
    xs = special_inputs()
    msg = _first_difference(_eval(host_lib.xs_host_eval, xs), _eval(host_lib.xs_libm_eval, xs), xs, "host build vs glibc")
    assert msg is None, msg


def test_special_inputs_reach_every_branch():
    """The special classes straddle each branch point named in exact_math.h."""
    xs = special_inputs()
    for u in (0x3eb17218, 0x3f851592, 0x41b00000, 0x24000000, 0x42b00000, 0x33000000, 0x4195b844, 0x42b17218):
        assert {u - 1, u, u + 1, (u - 1) | 0x80000000, u | 0x80000000, (u + 1) | 0x80000000} <= set(xs.tolist()), hex(u)
    f = xs.view(np.float32)
    assert np.isnan(f).sum() >= 12 and np.isinf(f).sum() == 2
    assert ((xs & 0x7f800000) == 0).sum() >= 10     # zeros and denormals of both signs


@pytest.mark.skipif(os.environ.get("CMIXB200_SLOW") != "1", reason="2^32 inputs x 4 functions on the CPU: set CMIXB200_SLOW=1")
def test_host_build_matches_libm_on_every_input(host_lib):
    bad = np.zeros(len(FUNCS), dtype=np.uint64)
    first = np.zeros(len(FUNCS), dtype=np.uint32)
    host_lib.xs_libm_sweep(0, N_BLKS, bad.ctypes.data, first.ctypes.data)
    msg = ["%s: %d inputs differ, the first is %08x" % (FUNCS[f], bad[f], first[f]) for f in range(len(FUNCS)) if bad[f]]
    assert not msg, "; ".join(msg)


# ------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
def test_device_build_matches_host_build_on_special_classes(host_lib, device_lib):
    xs = special_inputs()
    msg = _first_difference(_eval(device_lib.xs_device_eval, xs), _eval(host_lib.xs_host_eval, xs), xs, "device vs host build")
    assert msg is None, msg


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_device_build_matches_host_build_on_every_input(host_lib, device_lib):
    t0 = time.time()
    failures = []
    dev = np.empty((CHUNK_BLKS, len(FUNCS)), dtype=np.uint64)
    host = np.empty_like(dev)
    for chunk in range(N_BLKS // CHUNK_BLKS):
        blk0 = chunk * CHUNK_BLKS
        rc = device_lib.xs_device_sums(blk0, CHUNK_BLKS, dev.ctypes.data)
        assert rc == 0, "CUDA error %d" % rc
        host_lib.xs_host_sums(blk0, CHUNK_BLKS, host.ctypes.data)
        bad = np.nonzero((dev != host).any(axis=1))[0]
        if bad.size:
            base = (blk0 + int(bad[0])) << BLK_LOG2
            xs = np.arange(base, base + (1 << BLK_LOG2), dtype=np.uint64).astype(np.uint32)
            msg = _first_difference(_eval(device_lib.xs_device_eval, xs), _eval(host_lib.xs_host_eval, xs), xs,
                                    "chunk %d (inputs %08x..%08x, %d blocks of 2^16 differ)"
                                    % (chunk, blk0 << BLK_LOG2, ((blk0 + CHUNK_BLKS) << BLK_LOG2) - 1, bad.size))
            failures.append(msg or "chunk %d: checksums differ but no input does" % chunk)
    print("\n2^32 inputs x %d functions, device vs host build: %.1f s" % (len(FUNCS), time.time() - t0))
    assert not failures, "\n".join(failures)
