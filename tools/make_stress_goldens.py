"""Fixtures of the stress data classes (tools/gen_stress.py) from dumps of the UNMODIFIED reference (build container only).

    python tools/make_stress_goldens.py [name ...]        # default: every entry of gen_stress.STREAMS

Recipe of every committed tests/golden/stress_<name>.npz, with (n_bytes, seed) from gen_stress.STREAMS:
    python tools/gen_stress.py <name> <n_bytes> s.bin <seed>;  oracle_dump dump n s.bin <prefix> 1 <n_bytes>
`cmix -n` codes a 5-byte header (0, then the length as u32 big-endian) before the data; the fixture keeps the first n_bytes
coded bytes (gen_stress.coded_stream). The streams are shorter than 10000 bytes, so the reference's vocabulary is all 256 symbols. Each fixture holds, in the
layout of tests/golden/full_*.npz: the stream, the vocabulary, Predictor::Predict() of every bit, one CRC32 per 4096
coded bits over the reference's 431 FXCM codes and over its 1591 PAQ8 codes, and the codes of the first 64 bits; plus
the LSTM feedback FXCM consumed per bit (`lstmfx`, lstmpr | lstmex << 16, as in fxcm_*.npz) and one CRC32 per byte of the
256-float PPMD distribution left after that byte (`ppmd_crc`, as in ppmd_*.npz).
"""
import os
import subprocess
import sys
import tempfile
import zlib
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import gen_stress  # noqa: E402
from oracle_io import Dump  # noqa: E402

ORACLE = os.path.join(ROOT, "oracle", "_ref", "oracle_dump")


def make(name, tmp, gen=gen_stress, kind="stress", dump=None):
    """tests/golden/<kind>_<name>.npz from stream `name` of generator module `gen` (gen_stress, gen_reach or gen_vocab).
    dump: the coded bytes the fixture keeps, when not the stream's length; the fixture then also holds `file_bytes`, the
    length of the whole coded stream (whose byte set is the reference's vocabulary)."""
    n, seed = gen.STREAMS[name]
    src, prefix = os.path.join(tmp, name + ".bin"), os.path.join(tmp, name)
    gen.generate(name, n, seed).tofile(src)
    extra = {}
    if dump is not None:
        n = dump
    subprocess.run([ORACLE, "dump", "n", src, prefix, "1", str(n)], check=True)
    d = Dump(prefix)
    if dump is not None:
        extra["file_bytes"] = np.array([int(d.meta["stream_bytes"])])
    whole = n == int(d.meta["stream_bytes"])         # a whole stream may end inside a CRC block
    assert d.n_bytes == n and (n % 512 == 0 or whole) and np.array_equal(d.stream, gen.coded_stream(name)[:n])
    nb = n * 8
    ext = d.ext
    crc_fx = np.array([zlib.crc32(np.ascontiguousarray(ext[b:b + 4096, :431]).tobytes()) for b in range(0, nb, 4096)], dtype=np.uint32)
    crc_p8 = np.array([zlib.crc32(np.ascontiguousarray(ext[b:b + 4096, 431:]).tobytes()) for b in range(0, nb, 4096)], dtype=np.uint32)
    ppmd_crc = np.array([zlib.crc32(d.ppmd[t].tobytes()) for t in range(n)], dtype=np.uint32)
    lstmfx = np.fromfile(prefix + ".lstmfx.u32", dtype=np.uint32)
    assert lstmfx.size == nb
    out = os.path.join(ROOT, "tests", "golden", "%s_%s.npz" % (kind, name))
    np.savez_compressed(out, stream=d.stream, vocab=d.vocab, p=d.p, crc_fx=crc_fx, crc_p8=crc_p8, first_codes=np.ascontiguousarray(ext[:64]),
                        lstmfx=lstmfx, ppmd_crc=ppmd_crc, mode=np.array([d.meta["mode"]]), dictionary=np.array([0]), **extra)
    bits = np.unpackbits(d.stream)
    bpb = -np.log2(np.where(bits == 1, d.p, 1 - d.p).astype(np.float64)).sum() / n
    return "%-8s %5d bytes  %.3f bits/byte -> %d KiB" % (name, n, bpb, os.path.getsize(out) // 1024)


def main(gen=gen_stress, kind="stress"):
    names = sys.argv[1:] or list(gen.STREAMS)
    with tempfile.TemporaryDirectory() as tmp, ThreadPoolExecutor(4) as ex:
        for line in ex.map(lambda k: make(k, tmp, gen, kind), names):
            print(line)


if __name__ == "__main__":
    main()
