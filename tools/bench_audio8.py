"""Cost of PAQ8's 8-bit audio mode on the device, beside text: one stream, every model group resident, bulk calls.

    python tools/bench_audio8.py [--kib 256] [--piece 4096]

Codes a seeded 8-bit mono PCM WAV file of `kib` KiB (tools/gen_audio8.py's tone, after a short text) and, for comparison,
the same number of bytes of tools/gen_wav.py's word salad, each through a fresh predictor in bulk calls of `piece` bytes
(cmix -n framing). Prints one JSON line: wall-clock us per coded bit of each (host clock, first piece excluded as
warm-up) and each kernel's CUDA-event time per coded bit (Predictor.kernel_ms; the kernels run on their own streams and
overlap, the stream advances at the slowest one's pace). Writes nothing.
"""
import argparse
import json
import os
import struct
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from gen_audio8 import _tone, wav8  # noqa: E402
from gen_wav import _text  # noqa: E402

KERNELS = ["mix_kernel_v3", "small_kernel", "lstm_kernel", "ppmd_kernel", "fxcm_kernel", "paq8_kernel"]


def framed(data):
    return np.concatenate([np.frombuffer(b"\0" + struct.pack(">I", len(data)), dtype=np.uint8), np.frombuffer(data, dtype=np.uint8)])


def measure(cmix_b200, stream, piece):
    vocab = np.ones(256, dtype=np.uint8)                 # cmix -n: every byte value
    P = cmix_b200.Predictor(vocab, device=0)
    try:
        P.code_bytes(stream[:piece])                     # warm-up: first launches, table fetches
        P.time_mix_kernel(True)
        t0 = time.perf_counter()
        for a in range(piece, stream.size, piece):
            P.code_bytes(stream[a:a + piece])
        dt = time.perf_counter() - t0
        bits = (stream.size - piece) * 8
        kernels = {}
        for w, name in enumerate(KERNELS):
            ms, _ = P.kernel_ms(w)
            kernels[name] = ms * 1e3 / bits
        P.time_mix_kernel(False)
    finally:
        P.close()
    return {"us_per_coded_bit": dt * 1e6 / bits, "kernel_us_per_coded_bit": kernels, "coded_bytes": int(stream.size - piece)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--kib", type=int, default=256)
    ap.add_argument("--piece", type=int, default=4096)
    args = ap.parse_args()
    import cmix_b200
    n = args.kib * 1024
    rng = np.random.default_rng(0xA8D1B)
    lead = _text(rng, 400).tobytes()
    audio = framed(lead + wav8(_tone(rng, n, 1), 1))
    text = framed(_text(np.random.default_rng(0xA8D1C), audio.size - 5).tobytes())
    out = {"gpu": "H100 80GB (sm_90a)", "kib": args.kib, "piece": args.piece,
           "audio8_mono": measure(cmix_b200, audio, args.piece), "text": measure(cmix_b200, text, args.piece)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
