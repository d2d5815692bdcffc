"""Fixtures of the vocabulary shapes (tools/gen_vocab.py) from dumps of the UNMODIFIED reference (build container only).

    python tools/make_vocab_goldens.py [name ...]        # default: every entry of gen_vocab.STREAMS

Recipe of every committed tests/golden/vocab_<name>.npz, with (n_bytes, seed) from gen_vocab.STREAMS and d =
gen_vocab.DUMPED[name] (4096, or the whole coded stream for gen_vocab.FULL):
    python tools/gen_vocab.py <name> <n_bytes> v.bin <seed>;  oracle_dump dump n v.bin <prefix> 1 <d>
Each coded stream is at least 10000 bytes long, so the reference's vocabulary is its byte set, the shape's alphabet. The
fixture holds, in the layout of stress_*.npz (tools/make_stress_goldens.py), the first d coded bytes, the vocabulary,
Predict() of every bit, CRCs of the FXCM and PAQ8 codes per 4096 bits, the codes of the first 64 bits, the LSTM feedback
FXCM saw and a CRC of the PPMD distribution per byte; plus `file_bytes`, the length of the whole coded stream.
For gen_vocab.FULL it also writes tests/golden/vocab_<FULL>.cmix, the archive of the reference CLI:
    oracle/_ref/cmix_strict -n v.bin vocab_<FULL>.cmix
(its 5-byte length header and 32-byte vocabulary bitmap, then the coder's bytes).
"""
import os
import shutil
import subprocess
import sys
import tempfile
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import gen_vocab  # noqa: E402
from make_stress_goldens import make  # noqa: E402

CLI = os.path.join(ROOT, "oracle", "_ref", "cmix_strict")


def archive(name, tmp):
    """tests/golden/vocab_<name>.cmix: `cmix_strict -n` over the stream's data."""
    n, seed = gen_vocab.STREAMS[name]
    src, out = os.path.join(tmp, name + ".cli.bin"), os.path.join(ROOT, "tests", "golden", "vocab_%s.cmix" % name)
    gen_vocab.generate(name, n, seed).tofile(src)
    subprocess.run([CLI, "-n", src, os.path.join(tmp, name + ".cmix")], check=True, stdout=subprocess.DEVNULL,
                   stderr=subprocess.DEVNULL)
    shutil.copy(os.path.join(tmp, name + ".cmix"), out)
    return "%-8s archive %d bytes" % (name, os.path.getsize(out))


def main():
    names = sys.argv[1:] or list(gen_vocab.STREAMS)
    with tempfile.TemporaryDirectory() as tmp, ThreadPoolExecutor(4) as ex:
        jobs = [ex.submit(make, k, tmp, gen_vocab, "vocab", gen_vocab.DUMPED[k]) for k in names]
        if gen_vocab.FULL in names:
            jobs.append(ex.submit(archive, gen_vocab.FULL, tmp))
        for j in jobs:
            print(j.result())


if __name__ == "__main__":
    main()
