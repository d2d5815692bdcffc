"""tests/golden/overflow_random6k.npz from a dump of the UNMODIFIED reference (build container only).

    python tools/make_overflow_golden.py

The stream is the byte stream of conftest.synthetic_streams(6000, seed=1, vocab_lo=0, vocab_hi=256): uniform bytes with
15 % spaces, which takes eleven mixers past the 10 000-context cap (tests/test_mixer_overflow.py). `cmix -n` codes a
5-byte header (0, then the length as u32 big-endian) before the data; the fixture keeps the first 6000 coded bytes, so
its vocabulary is all 256 symbols. It holds, in the layout of tests/golden/stress_*.npz: the stream, the vocabulary,
Predict() of every bit, one CRC32 per 4096 coded bits over the reference's 431 FXCM codes and over its 1591 PAQ8 codes,
the codes of the first 64 bits, the LSTM feedback FXCM consumed per bit and one CRC32 per byte of the PPMD distribution.
"""
import os
import subprocess
import sys
import tempfile
import zlib

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from oracle_io import Dump  # noqa: E402

ORACLE = os.path.join(ROOT, "oracle", "_ref", "oracle_dump")
N_BYTES, SEED = 6000, 1


def data():
    """The byte stream of conftest.synthetic_streams(N_BYTES, SEED, 0, 256) (drawn first there, from the same generator)."""
    rng = np.random.default_rng(SEED)
    stream = rng.integers(0, 256, size=N_BYTES, dtype=np.uint8)
    stream[rng.random(N_BYTES) < 0.15] = 32
    return stream


def coded_stream():
    n = N_BYTES
    return np.concatenate([np.array([0, n >> 24 & 255, n >> 16 & 255, n >> 8 & 255, n & 255], dtype=np.uint8), data()])[:n]


def main():
    n = N_BYTES
    with tempfile.TemporaryDirectory() as tmp:
        src, prefix = os.path.join(tmp, "in.bin"), os.path.join(tmp, "overflow")
        data().tofile(src)
        subprocess.run([ORACLE, "dump", "n", src, prefix, "1", str(n)], check=True)
        d = Dump(prefix)
        assert d.n_bytes == n and np.array_equal(d.stream, coded_stream())
        nb = n * 8
        ext = d.ext
        crc_fx = np.array([zlib.crc32(np.ascontiguousarray(ext[b:b + 4096, :431]).tobytes()) for b in range(0, nb, 4096)], dtype=np.uint32)
        crc_p8 = np.array([zlib.crc32(np.ascontiguousarray(ext[b:b + 4096, 431:]).tobytes()) for b in range(0, nb, 4096)], dtype=np.uint32)
        ppmd_crc = np.array([zlib.crc32(d.ppmd[t].tobytes()) for t in range(n)], dtype=np.uint32)
        lstmfx = np.fromfile(prefix + ".lstmfx.u32", dtype=np.uint32)
        assert lstmfx.size == nb
        out = os.path.join(ROOT, "tests", "golden", "overflow_random6k.npz")
        np.savez_compressed(out, stream=d.stream, vocab=d.vocab, p=d.p, crc_fx=crc_fx, crc_p8=crc_p8,
                            first_codes=np.ascontiguousarray(ext[:64]), lstmfx=lstmfx, ppmd_crc=ppmd_crc,
                            mode=np.array([d.meta["mode"]]), dictionary=np.array([0]))
    bits = np.unpackbits(d.stream)
    bpb = -np.log2(np.where(bits == 1, d.p, 1 - d.p).astype(np.float64)).sum() / n
    print("overflow_random6k: %d bytes, %.3f bits/byte -> %d KiB" % (n, bpb, os.path.getsize(out) // 1024))


if __name__ == "__main__":
    main()
