"""Seeded RIFF streams around PAQ8's WAV parser (audioModel, paq8.cpp:5806-5852): near misses and real PCM WAV files.

    python tools/gen_wav.py <name> <out>

Pure numpy from a seed. Every stream is text (a seeded word salad), then RIFF data. The reference switches to its audio
models only on the first byte of a `data` chunk whose length is a whole number of sample blocks, after a `WAVE` header with a
PCM `fmt ` chunk of 16 or 18 bytes, 1 or 2 channels and 8 or 16 bits. So:
    NEAR_MISS    never get there and code with the ordinary models
    ENTERS       get there; the RIFF header starts so that the first sample is the first byte of a 4096-bit block of the
                 coded stream (`entry`, counted with `cmix -n`'s 5-byte header), and PAQ8 raises ERR_UNSUPPORTED_BLOCK there
No stream carries a BMP / TGA / JPEG header. STREAMS holds (n_bytes, seed, cmix mode) of every fixture
tools/make_wav_goldens.py writes; mode 'c' runs the CLI's preprocessor over the file first.
"""
import struct
import sys

import numpy as np

WORDS = ("the of and a to in is was file format audio sample chunk header data sound wave stereo mono bits rate "
         "container stream music record time length byte channel signal value level").split()


def _text(rng, n):
    out, size = [], 0
    while size < n:
        w = WORDS[int(rng.integers(len(WORDS)))]
        w += ". " if rng.random() < 0.08 else ", " if rng.random() < 0.05 else " "
        out.append(w)
        size += len(w)
    return np.frombuffer("".join(out).encode()[:n], dtype=np.uint8)


def _samples(rng, n, bits, channels):
    t = np.arange(n, dtype=np.float64)
    v = np.stack([np.sin(2 * np.pi * t / (41.3 + 7 * c)) * 0.6 + rng.normal(0, 0.01, n) for c in range(channels)], axis=1)
    if bits == 8:
        return np.clip(np.rint(128 + 100 * v), 0, 255).astype(np.uint8).ravel()
    return np.clip(np.rint(20000 * v), -32768, 32767).astype("<i2").view(np.uint8).ravel()


def riff(form, chunks):
    body = form + b"".join(cid + struct.pack("<I", len(c)) + c + (b"\0" if len(c) & 1 else b"") for cid, c in chunks)
    return b"RIFF" + struct.pack("<I", len(body)) + body


def fmt(channels, bits, tag=1, extra=None):
    block = channels * bits // 8
    f = struct.pack("<HHIIHH", tag, channels, 8000, 8000 * block, block, bits)
    return f + (struct.pack("<H", extra) if extra is not None else b"")


def wav(rng, n_samples, bits=16, channels=2, tag=1, extra=None, list_chunk=False, data_len=None):
    data = _samples(rng, n_samples, bits, channels).tobytes()
    chunks = [(b"fmt ", fmt(channels, bits, tag, extra))]
    if list_chunk:
        chunks.append((b"LIST", b"INFOISFT\x0e\0\0\0gen_wav seeded\0\0"))
    chunks.append((b"data", data))
    out = riff(b"WAVE", chunks)
    if data_len is not None:                    # rewrite the data chunk's length field (the bytes that follow stay as they are)
        k = out.index(b"data") + 4
        out = out[:k] + struct.pack("<I", data_len) + out[k + 4:]
    return out


def _header_bytes(**kw):
    """Bytes in front of the first sample of wav(**kw)."""
    return wav(np.random.default_rng(0), 1, **kw).index(b"data") + 8


def _near_riff_text(rng):
    mentions = [b" RIFF ", b"RIFF", b"a RIFF WAVE file ", b"RIFF....WAVEfmt "]
    parts = []
    for _ in range(12):
        parts.append(_text(rng, int(rng.integers(80, 200))).tobytes())
        parts.append(mentions[int(rng.integers(len(mentions)))])
    return b"".join(parts)


def _near_avi(rng):
    return riff(b"AVI ", [(b"LIST", b"hdrlavih" + bytes(56)), (b"JUNK", bytes(20)), (b"LIST", b"movi00dc" + rng.bytes(700))])


def _near_webp(rng):
    return riff(b"WEBP", [(b"VP8 ", rng.bytes(900))])


def _near_mp3_tag(rng):
    return wav(rng, 600, bits=16, channels=1, tag=0x0055)


def _near_24bit(rng):
    return riff(b"WAVE", [(b"fmt ", fmt(2, 24)), (b"data", rng.bytes(600 * 6))])


def _near_odd_length(rng):
    return wav(rng, 400, bits=16, channels=2, data_len=1602)         # 16-bit stereo: 4-byte blocks


# name -> (body after the text, text bytes in front of it); NEAR_MISS streams fill up with text to n_bytes
NEAR_MISS = {"riff_text": _near_riff_text, "avi": _near_avi, "webp": _near_webp, "mp3_tag": _near_mp3_tag,
             "bits24": _near_24bit, "odd_length": _near_odd_length}
ENTERS = {
    "pcm8_mono": dict(bits=8, channels=1),
    "pcm8_stereo": dict(bits=8, channels=2),
    "pcm16_mono": dict(bits=16, channels=1),
    "pcm16_stereo": dict(bits=16, channels=2),
    "fmt18_list": dict(bits=16, channels=2, extra=0, list_chunk=True),
    "past_end": dict(bits=16, channels=1, data_len=1 << 20),          # a data chunk longer than the stream
}
ENTRY = 1024                                                          # coded-stream byte of the first sample (bit 8192)

STREAMS = {}
for _i, _name in enumerate(NEAR_MISS):
    STREAMS["near_" + _name] = (3072, 0x3A7E00 + _i, "n")
STREAMS["near_riff_text_cli"] = (3072, 0x3A7E00, "c")
for _i, _name in enumerate(ENTERS):
    STREAMS["wav_" + _name] = (2048, 0x3A7E80 + _i, "n")


def generate(name, n_bytes, seed):
    """The file `cmix` codes for fixture `name` (before its 5-byte -n header), n_bytes long."""
    rng = np.random.default_rng(seed)
    if name.startswith("near_"):
        kind = name[len("near_"):].replace("_cli", "")
        body = NEAR_MISS[kind](rng)
        lead = _text(rng, 600).tobytes()
        out = lead + body + _text(rng, n_bytes).tobytes()
    else:
        kw = ENTERS[name[len("wav_"):]]
        lead = _text(rng, ENTRY - 5 - _header_bytes(**kw)).tobytes()
        out = lead + wav(rng, n_bytes, **kw)
    out = np.frombuffer(out[:n_bytes], dtype=np.uint8).copy()
    assert out.size == n_bytes
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
