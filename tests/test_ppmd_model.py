"""The PPMD byte model (SURVEY §8 a15) pinned against the unmodified reference.

cmix_b200/csrc/ppmd_model.h is integer-only host/device code; here it is compiled for the host and
compared with fixtures made from per-byte dumps of the reference (tools/make_ppmd_golden.py:
one CRC-32 per byte of the 256-float distribution PPMD::ByteUpdate leaves, ppmd.cpp:1328-1338),
and with the full distributions stored in the golden dumps. The device build of the same header is
checked by tests/test_gpu_parity.py.
"""
import zlib

import numpy as np
import pytest

from harness import golden, ppmd_host  # noqa: F401  (ppmd_host: fixture)


@pytest.mark.parametrize("name", ["ppmd_text40k", "ppmd_bin6k", "ppmd_rand", "ppmd_rep", "ppmd_dic"])
def test_distributions_match_the_reference_dump(ppmd_host, name):
    g = golden(name)
    rc, out = ppmd_host(g["stream"], g["vocab"])
    assert rc == 0
    got = np.array([zlib.crc32(out[t].tobytes()) for t in range(out.shape[0])], dtype=np.uint32)
    bad = np.nonzero(got != g["crc"])[0]
    assert bad.size == 0, "first differing byte %d of %d" % (bad[0], got.size)


def test_full_distributions_of_the_golden_dumps(ppmd_host, golden):
    rc, out = ppmd_host(golden.stream, golden.vocab)
    assert rc == 0
    assert np.array_equal(out, golden.ppmd)
    # a distribution: vocabulary mask respected, sums to one within float rounding
    assert np.all(out[:, golden.vocab == 0] == 0)
    assert np.allclose(out.sum(axis=1), 1.0, atol=1e-5)


def test_arena_exhaustion_is_reported_not_ignored(ppmd_host):
    rng = np.random.default_rng(3)
    stream = rng.integers(0, 256, 40000, dtype=np.uint8)
    rc, _ = ppmd_host(stream, np.ones(256, dtype=np.uint8), arena_mb=1)
    assert rc == 1
