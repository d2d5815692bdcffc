"""Fixtures that let the tests compare with the unmodified reference without it being present.

    python tools/make_ref_goldens.py <reference checkout>

Needs oracle/_ref/ built from that checkout (make -C oracle ref REF=<reference checkout>). Writes under tests/golden/:
    english.dic.gz          the reference's WRT dictionary (input data of `cmix -c english.dic`), gzip-compressed
    text208.cmix            `cmix_strict -n` archive of text208's file (test_oracle_port.py)
    synth2000.npz           stream, vocabulary and Predict() of every bit of oracle_dump over gen_synth text
                            (2000 bytes, seed 0xE9E80002; test_gpu_parity.py)
    reference_tables.json   SHA-256 of the reference's constant tables that the CUDA sources restate
                            (FXCM's WRT byte classes, PAQ8's state / x86 / ASCII tables; test_fxcm_model.py,
                            test_full_predictor.py). Digests only: the tables themselves are not stored.
"""
import gzip
import hashlib
import json
import os
import re
import shutil
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
REF_BIN = os.path.join(ROOT, "oracle", "_ref")
sys.path.insert(0, os.path.join(ROOT, "tools"))

FXCM_TABLES = ("wrt_2b", "wrt_3b", "wrt_4b")
SYNTH_BYTES, SYNTH_SEED = 2000, 0xE9E80002


def digest_ints(values):
    return hashlib.sha256(",".join(str(int(v)) for v in values).encode()).hexdigest()


def digest_hex(s):
    return hashlib.sha256(s.encode()).hexdigest()


def fxcm_reference_tables(ref):
    src = open(os.path.join(ref, "src", "models", "fxcmv1.cpp")).read()
    out = {}
    for name in FXCM_TABLES:
        body = re.sub(r"//.*", "", re.search(name + r"\[\d+\]\s*=\s*\{(.*?)\};", src, re.S).group(1))
        out[name] = [int(x) for x in re.findall(r"\d+", body)]
    return out


def main():
    ref = os.path.abspath(sys.argv[1])
    from gen_synth import synth_text
    from oracle_io import Dump
    import make_paq8_tables

    with open(os.path.join(ref, "dictionary", "english.dic"), "rb") as f:
        dic = gzip.compress(f.read(), compresslevel=9, mtime=0)
    with open(os.path.join(GOLD, "english.dic.gz"), "wb") as f:
        f.write(dic)

    g = np.load(os.path.join(GOLD, "text208.npz"))
    with tempfile.TemporaryDirectory() as tmp:
        src, arc = os.path.join(tmp, "in.bin"), os.path.join(tmp, "out.cmix")
        open(src, "wb").write(g["stream"][5:].tobytes())          # the stream carries the 5-byte DEFAULT block header
        subprocess.run([os.path.join(REF_BIN, "cmix_strict"), "-n", src, arc], check=True, stdout=subprocess.DEVNULL)
        shutil.copyfile(arc, os.path.join(GOLD, "text208.cmix"))

        src = os.path.join(tmp, "synth.txt")
        open(src, "wb").write(synth_text(SYNTH_BYTES, SYNTH_SEED))
        subprocess.run([os.path.join(REF_BIN, "oracle_dump"), "dump", "n", src, os.path.join(tmp, "d"), "1"],
                       check=True, stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
        d = Dump(os.path.join(tmp, "d"))
        np.savez_compressed(os.path.join(GOLD, "synth2000.npz"), stream=d.stream, vocab=d.vocab, p=d.p)

    make_paq8_tables.REF = os.path.join(ref, "src", "models", "paq8.cpp")
    tables = {"fxcm": {k: digest_ints(v) for k, v in fxcm_reference_tables(ref).items()},
              "paq8": {k: digest_hex(v) for k, v in make_paq8_tables.tables().items()}}
    with open(os.path.join(GOLD, "reference_tables.json"), "w") as f:
        json.dump(tables, f, indent=1, sort_keys=True)
        f.write("\n")
    for name in ("english.dic.gz", "text208.cmix", "synth2000.npz", "reference_tables.json"):
        print(name, os.path.getsize(os.path.join(GOLD, name)), "bytes")


if __name__ == "__main__":
    main()
