"""Seeded data classes that text and x86 code barely contain: constant, run, numeric, record and incompressible data.

    python tools/gen_stress.py <class> <n_bytes> <out> [seed]

Each class is pure numpy from a seed (no file reads), so a test can regenerate a stream and compare it with its fixture:
    zeros    all 0x00: nearly every context saturates at once (PAQ8's shared random sequence, stretch/mixer clamps)
    runs     random byte values in runs of geometric length (mean 24)
    sine     noisy 8-bit sine (period 37.3 bytes, amplitude 100, noise sigma 2)
    ramp     8-bit ramps whose slope changes every 256 bytes
    pcm16    headerless 16-bit little-endian PCM: two sines plus noise
    records  12-byte binary records (u32 id, u16 type, u16 slowly varying level, u32 timestamp; little-endian)
    csv      a CSV table of integers, decimals and short names
    random   uniform random bytes (PPMD sees all 256 symbols)
    nested   bracket-nested C-like code
    mixed    the classes above in order, 512 bytes each, so that model state carries across changes of data type
None of them carries a header PAQ8's block parser validates (BMP/TGA/PNM/TIFF/WAV/JPEG): every stream codes with the
image, audio and JPEG models off. STREAMS holds the (length, seed) of every fixture tools/make_stress_goldens.py writes.
"""
import sys

import numpy as np

SEGMENT = 512


def _zeros(rng, n):
    return np.zeros(n, dtype=np.uint8)


def _runs(rng, n):
    out = []
    while sum(map(len, out)) < n:
        out.append(np.full(int(rng.geometric(1.0 / 24)), rng.integers(0, 256), dtype=np.uint8))
    return np.concatenate(out)[:n]


def _sine(rng, n):
    t = np.arange(n, dtype=np.float64)
    return np.clip(np.rint(128 + 100 * np.sin(2 * np.pi * t / 37.3) + rng.normal(0, 2, n)), 0, 255).astype(np.uint8)


def _ramp(rng, n):
    slopes = rng.choice([1, 2, 3, 5, 7, 254], size=(n + 255) // 256)
    step = np.repeat(slopes, 256)[:n]
    return (np.cumsum(step) + int(rng.integers(0, 256))).astype(np.int64).astype(np.uint8)


def _pcm16(rng, n):
    t = np.arange((n + 1) // 2, dtype=np.float64)
    v = 7000 * np.sin(2 * np.pi * t / 61.7) + 2500 * np.sin(2 * np.pi * t / 13.1 + 1.0) + rng.normal(0, 40, t.size)
    return np.clip(np.rint(v), -32768, 32767).astype("<i2").view(np.uint8)[:n].copy()


def _records(rng, n):
    k = (n + 11) // 12
    rec = np.zeros(k, dtype=[("id", "<u4"), ("type", "<u2"), ("level", "<u2"), ("time", "<u4")])
    rec["id"] = 100000 + np.arange(k)
    rec["type"] = rng.choice([1, 2, 2, 3, 7], size=k)
    rec["level"] = np.clip(np.cumsum(rng.integers(-40, 41, size=k)) + 20000, 0, 65535)
    rec["time"] = 1600000000 + np.cumsum(rng.integers(900, 1100, size=k))
    return rec.view(np.uint8)[:n].copy()


def _csv(rng, n):
    names = ["alpha", "beta", "gamma", "delta", "omega", "sigma"]
    rows, size, i = ["id,name,count,price,ok\n"], 0, 0
    while size < n:
        row = "%d,%s,%d,%.2f,%s\n" % (i + 1, names[int(rng.integers(0, 6))], int(rng.integers(0, 5000)),
                                     float(rng.integers(0, 100000)) / 100, "yes" if rng.random() < 0.7 else "no")
        rows.append(row)
        size += len(row)
        i += 1
    return np.frombuffer("".join(rows).encode("ascii")[:n], dtype=np.uint8).copy()


def _random(rng, n):
    return rng.integers(0, 256, size=n, dtype=np.uint8)


def _nested(rng, n):
    words = ["x", "y", "idx", "buf", "len", "tmp", "node", "next", "val", "f", "g"]
    out = []

    def expr(depth):
        r = rng.random()
        if depth > 5 or r < 0.3:
            return words[int(rng.integers(0, len(words)))] if rng.random() < 0.7 else str(int(rng.integers(0, 100)))
        if r < 0.55:
            return "%s(%s)" % (words[int(rng.integers(0, len(words)))], ", ".join(expr(depth + 1) for _ in range(int(rng.integers(1, 4)))))
        if r < 0.75:
            return "%s[%s]" % (words[int(rng.integers(0, len(words)))], expr(depth + 1))
        return "(%s %s %s)" % (expr(depth + 1), "+-*/<>"[int(rng.integers(0, 6))], expr(depth + 1))

    def block(depth):
        pad = "  " * depth
        for _ in range(int(rng.integers(1, 4))):
            r = rng.random()
            if depth < 4 and r < 0.35:
                out.append("%s%s (%s) {\n" % (pad, ["if", "while", "for"][int(rng.integers(0, 3))], expr(1)))
                block(depth + 1)
                out.append(pad + "}\n")
            else:
                out.append("%s%s = %s;\n" % (pad, words[int(rng.integers(0, len(words)))], expr(0)))

    while sum(map(len, out)) < n:
        out.append("int %s(int %s) {\n" % (words[int(rng.integers(0, len(words)))], words[int(rng.integers(0, len(words)))]))
        block(1)
        out.append("}\n\n")
    return np.frombuffer("".join(out).encode("ascii")[:n], dtype=np.uint8).copy()


CLASSES = {"zeros": _zeros, "runs": _runs, "sine": _sine, "ramp": _ramp, "pcm16": _pcm16, "records": _records,
           "csv": _csv, "random": _random, "nested": _nested}


def _mixed(rng, n):
    seeds = rng.integers(0, 2 ** 32, size=len(CLASSES))
    segs = [fn(np.random.default_rng(int(s)), SEGMENT) for fn, s in zip(CLASSES.values(), seeds)]
    return np.resize(np.concatenate(segs), n)


def generate(kind, n_bytes, seed):
    """n_bytes of class `kind` from np.random.default_rng(seed)."""
    fn = _mixed if kind == "mixed" else CLASSES[kind]
    out = fn(np.random.default_rng(seed), n_bytes)
    assert out.dtype == np.uint8 and out.size == n_bytes
    return out


# fixture tests/golden/stress_<name>.npz: (n_bytes, seed); lengths are whole 4096-bit CRC blocks
STREAMS = {name: (3072, 0x57E5500 + i) for i, name in enumerate(CLASSES)}
STREAMS["mixed"] = (len(CLASSES) * SEGMENT, 0x57E55FF)


def coded_stream(name):
    """The first n_bytes bytes `cmix -n` codes for fixture `name`: its 5-byte header (0, length u32 big-endian), then the data."""
    n, seed = STREAMS[name]
    return np.concatenate([np.array([0, n >> 24 & 255, n >> 16 & 255, n >> 8 & 255, n & 255], dtype=np.uint8), generate(name, n, seed)])[:n]


if __name__ == "__main__":
    kind, n, path = sys.argv[1], int(sys.argv[2]), sys.argv[3]
    seed = int(sys.argv[4], 0) if len(sys.argv) > 4 else STREAMS[kind][1]
    generate(kind, n, seed).tofile(path)
