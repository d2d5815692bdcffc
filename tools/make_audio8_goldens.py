"""Fixtures of the 8-bit audio streams (tools/gen_audio8.py) from dumps of the UNMODIFIED reference (build container only).

    python tools/make_audio8_goldens.py [name ...]     # default: every entry of gen_audio8.STREAMS

Recipe of every committed tests/golden/<name>.npz, with (n_bytes, seed, mode) from gen_audio8.STREAMS:
    python tools/gen_audio8.py <name> w.bin;  oracle_dump dump <mode> w.bin <prefix> 1 <n_bytes>
Each fixture holds, in the layout of tests/golden/full_*.npz: the coded stream, the vocabulary, Predictor::Predict() of
every bit, one CRC32 per 4096 coded bits over the reference's 431 FXCM codes and over its 1591 PAQ8 codes, and the codes
of the first 64 bits.
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
from gen_audio8 import STREAMS, coded_stream, generate  # noqa: E402
from oracle_io import Dump  # noqa: E402

ORACLE = os.path.join(ROOT, "oracle", "_ref", "oracle_dump")


def make(name, tmp):
    n, seed, mode = STREAMS[name]
    src, prefix = os.path.join(tmp, name + ".bin"), os.path.join(tmp, name)
    generate(name, n, seed).tofile(src)
    subprocess.run([ORACLE, "dump", mode, src, prefix, "1", str(n)], check=True, stdout=subprocess.DEVNULL)
    d = Dump(prefix)
    assert d.n_bytes == n and n % 512 == 0 and (mode != "n" or np.array_equal(d.stream, coded_stream(name)))
    nb = n * 8
    ext = d.ext
    crc_fx = np.array([zlib.crc32(np.ascontiguousarray(ext[b:b + 4096, :431]).tobytes()) for b in range(0, nb, 4096)], dtype=np.uint32)
    crc_p8 = np.array([zlib.crc32(np.ascontiguousarray(ext[b:b + 4096, 431:]).tobytes()) for b in range(0, nb, 4096)], dtype=np.uint32)
    out = os.path.join(ROOT, "tests", "golden", name + ".npz")
    np.savez_compressed(out, stream=d.stream[:n], vocab=d.vocab, p=d.p[:nb], crc_fx=crc_fx, crc_p8=crc_p8, first_codes=np.ascontiguousarray(ext[:64]),
                        mode=np.array([d.meta["mode"]]), dictionary=np.array([0]))
    return "%-22s %5d bytes (mode %s) -> %d KiB" % (name, n, mode, os.path.getsize(out) // 1024)


def main():
    names = sys.argv[1:] or list(STREAMS)
    with tempfile.TemporaryDirectory() as tmp, ThreadPoolExecutor(8) as ex:
        for line in ex.map(lambda k: make(k, tmp), names):
            print(line)


if __name__ == "__main__":
    main()
