"""Seeded streams of 8-bit PCM WAV audio, which PAQ8 codes with audio8bModel (paq8.cpp:5552-5657) and recordModel(AUDIO).

    python tools/gen_audio8.py <name> <out>

Pure numpy from a seed, built from tools/gen_wav.py's text, `wav` and `fmt`. Each stream covers a path of the audio model:
    mono_text       a mono file, then text after its last sample: the ordinary models resume with the state they froze
    stereo_odd      a stereo file with a LIST chunk whose first sample falls on an odd block position
    mono_stereo     a mono file, text, then a stereo file: the model restarts and switches channel layout, and the mixer's
                    layout switches twice each way
    clipped         a clipped square wave and long silence: predictions clip at both ends, the covariance is near singular
    then16          an 8-bit file followed by a 16-bit one, which stops with ERR_UNSUPPORTED on its first sample
    cli             mono_text through the CLI's preprocessor (`cmix -c`)
No stream carries a BMP / TGA / JPEG header (checked by `generate`). STREAMS holds (n_bytes, seed, cmix mode).
"""
import struct
import sys

import numpy as np

from gen_wav import _text, fmt, riff

STREAMS = {
    "audio8_mono_text": (8192, 0xA8D10, "n"),
    "audio8_stereo_odd": (6144, 0xA8D11, "n"),
    "audio8_mono_stereo": (8192, 0xA8D12, "n"),
    "audio8_clipped": (6144, 0xA8D13, "n"),
    "audio8_then16": (4096, 0xA8D14, "n"),
    "audio8_cli": (8192, 0xA8D10, "c"),
}


def _tone(rng, n, channels):
    t = np.arange(n, dtype=np.float64)
    v = np.stack([0.5 * np.sin(2 * np.pi * t / (37.7 + 9 * c)) + 0.25 * np.sin(2 * np.pi * t / (11.1 + 3 * c)) +
                  rng.normal(0, 0.02, n) for c in range(channels)], axis=1)
    return np.clip(np.rint(128 + 120 * v), 0, 255).astype(np.uint8).ravel().tobytes()


def _square(n):
    t = np.arange(n)
    v = np.where((t // 25) % 2 == 0, 255, 0).astype(np.uint8)
    v[n // 2:] = 128                                   # silence: every tap equal
    return v.tobytes()


def wav8(samples, channels, list_chunk=False):
    chunks = [(b"fmt ", fmt(channels, 8))]
    if list_chunk:
        chunks.append((b"LIST", b"INFOISFT\x0e\0\0\0gen_audio8 seed\0"))
    chunks.append((b"data", samples))
    return riff(b"WAVE", chunks)


def _body(name, rng):
    if name in ("audio8_mono_text", "audio8_cli"):
        return _text(rng, 300).tobytes() + wav8(_tone(rng, 6000, 1), 1) + _text(rng, 3000).tobytes()
    if name == "audio8_stereo_odd":
        return _text(rng, 299).tobytes() + wav8(_tone(rng, 2600, 2), 2, list_chunk=True) + _text(rng, 800).tobytes()
    if name == "audio8_mono_stereo":
        return (_text(rng, 200).tobytes() + wav8(_tone(rng, 2500, 1), 1) + _text(rng, 400).tobytes() +
                wav8(_tone(rng, 1900, 2), 2) + _text(rng, 1000).tobytes())
    if name == "audio8_clipped":
        return _text(rng, 256).tobytes() + wav8(_square(5000), 1) + _text(rng, 800).tobytes()
    if name == "audio8_then16":
        s16 = (np.sin(np.arange(800) / 7.0) * 12000).astype("<i2").tobytes()
        return (_text(rng, 200).tobytes() + wav8(_tone(rng, 1500, 1), 1) + _text(rng, 300).tobytes() +
                riff(b"WAVE", [(b"fmt ", fmt(1, 16)), (b"data", s16)]))
    raise KeyError(name)


def _no_image_header(b):
    """None of PAQ8's JPEG / BMP / TGA detectors (paq8_top.h detect_byte) fires on any byte of b (BMP: on its trigger)."""
    a = np.concatenate([np.zeros(64, dtype=np.int64), np.frombuffer(b, dtype=np.uint8).astype(np.int64)])
    def buf(k):                                        # buf(k) at every position pos = 1 .. len(b)
        return a[64 - k + 1:len(a) - k + 1]
    be4 = lambda i: buf(i - 3) | buf(i - 2) << 8 | buf(i - 1) << 16 | buf(i) << 24
    le4 = lambda i: buf(i) | buf(i - 1) << 8 | buf(i - 2) << 16 | buf(i - 3) << 24
    b1 = buf(1)
    jpeg = (buf(4) == 0xFF) & (buf(3) == 0xD8) & (buf(2) == 0xFF) & (((b1 & 0xFE) == 0xC0) | (b1 == 0xC4) | ((b1 >= 0xDB) & (b1 <= 0xFE)))
    bmp = le4(40) == 0x28
    tga = ((((be4(8) & 0xFFFFFF) == 0x010100) & ((be4(4) & 0xFFFFFFC7) == 0x100) & ((b1 == 16) | (b1 == 24) | (b1 == 32))) |
           (((be4(8) & 0xFFFEFF) == 0x000200) & (be4(4) == 0)))
    return not (jpeg | bmp | tga).any()


def generate(name, n_bytes, seed):
    """The file `cmix` codes for fixture `name` (before its 5-byte -n header), n_bytes long."""
    out = _body(name, np.random.default_rng(seed))
    out = out + _text(np.random.default_rng(seed + 1), max(0, n_bytes - len(out))).tobytes()
    out = np.frombuffer(out[:n_bytes], dtype=np.uint8).copy()
    assert out.size == n_bytes and _no_image_header(out.tobytes()), name
    return out


def first_sample(name):
    """Offsets in `generate`'s output of the first sample of each data chunk."""
    n, seed, _ = STREAMS[name]
    b = generate(name, n, seed).tobytes()
    out, k = [], b.find(b"RIFF")
    while k >= 0:
        out.append(b.find(b"data", k) + 8)         # the text holds no "RIFF"; inside a file the next "data" is the chunk
        k = b.find(b"RIFF", k + 4)
    return out


def coded_stream(name):
    """The first n_bytes bytes `cmix -n` codes for fixture `name`: its 5-byte header (0, length u32 big-endian), then the data."""
    n, seed, mode = STREAMS[name]
    assert mode == "n"
    return np.concatenate([np.array([0, n >> 24 & 255, n >> 16 & 255, n >> 8 & 255, n & 255], dtype=np.uint8), generate(name, n, seed)])[:n]


if __name__ == "__main__":
    name, path = sys.argv[1], sys.argv[2]
    n, seed, _ = STREAMS[name]
    generate(name, n, seed).tofile(path)
