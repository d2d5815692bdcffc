"""Seeded streams whose `cmix -n` coded bytes use exactly a chosen alphabet, so the reference gives them that vocabulary.

    python tools/gen_vocab.py <name> <n_bytes> <out> [seed]

The vocabulary is the one input of the predictor that changes array shapes on the device. The reference's runner gives a
coded stream of fewer than 10000 bytes all 256 symbols and a longer one the set of bytes it contains; `-n` codes a 5-byte
header (0x00, then the data length as u32 big-endian) before the data. So every alphabet holds 0x00, and each stream's
length is chosen so that the nonzero bytes of its header lie in the alphabet.

Its V symbols set (cmix_b200/csrc/lstm.cuh): the LSTM's one-hot columns, padded to a multiple of 4; its softmax rows,
ceil(V/8) per CTA of the 8-CTA cluster, so CTAs past the last row own none; and which bits of a byte are decided: where
the vocabulary bytes left in a bit's range all lie on one side, the LSTM's ByteModel reads out exactly 0 or 1 and
Predict() returns that value without mixing. PPMD and the bracket model mask their distributions by the vocabulary too.

Each stream starts with its alphabet in ascending order, then seeded synthetic wiki text (gen_synth.synth_text) mapped
onto the alphabet, with runs of one symbol and a repeated phrase; the alphabet comes again every TOUR bytes. The mapping
keeps the source bytes the alphabet holds, folds capitals to lower case and brackets to the alphabet's own pair where
the alphabet lacks them, and sends every other source byte, most frequent first, to the alphabet's symbols in turn
(those the source does not use first). The text stays learnable, so the LSTM grows confident and the match models fire.

    name     V    alphabet                         what it reaches
    two      2    0x00 0xFF                        V mod 4 = 2; six CTAs own no softmax row; bits 6-0 of every byte
                                                   are decided (Predict() exactly 0 or 1), only bit 7 is coded
    digits3  3    0x00 '0' '1'                     a padding of 1 column; bit 5 and, under '0' and '1', bit 0 are coded
    four     4    0x00 '\\n' '0' '1'                no padding; four CTAs own no row
    nine     9    0x00 ' ' ( ) a e n o t           V mod 4 = 1; ceil(V/8) = 2, so CTA 4 owns one row and three none;
                                                   brackets for the bracket model
    lower    27   0x00 a-z                         V mod 4 = 3; CTA 6 owns 3 rows and CTA 7 none; no brackets. Its
                                                   length bytes must be 0 or a-z, so it is 24832 bytes long (0x6100);
                                                   its fixture holds the whole stream and the reference CLI's archive
    v33      33   0x00 a-z space . , \\n [ ]         CTA 6 owns 3 of its 5 rows and CTA 7 none; bracket pair [ ]
    v57      57   0x00 a-z A-Z space . , \\n         CTA 7 owns exactly 1 row; no brackets
    v58      58   0x00 a-z A-Z space \\n ( ) .       CTA 7 owns exactly 2 rows; V mod 4 = 2 at a larger size
    high     129  0x00 0x80-0xFF                   every ByteModel's first split holds only 0x00 below it; the LSTM's
                                                   index of byte b is b - 127
    v254     254  all but 0x01 and 0xFF            V mod 4 = 2 near full size; the top of the byte range is empty
    v255     255  all but 0xFF                     the last symbol is missing; V mod 4 = 3
V = 1 cannot come from the runner (the header always holds a nonzero length byte). STREAMS holds the (length, seed) of
every fixture tools/make_vocab_goldens.py writes; DUMPED the coded bytes each fixture keeps.
"""
import sys

import numpy as np

from gen_synth import synth_text

TOUR = 2048          # the alphabet in ascending order starts the data and comes again every TOUR bytes
PAIRS = [(ord("("), ord(")")), (ord("["), ord("]")), (ord("{"), ord("}")), (ord("<"), ord(">"))]


def _chars(s):
    return [ord(c) for c in s]


LOWER = _chars("abcdefghijklmnopqrstuvwxyz")
UPPER = _chars("ABCDEFGHIJKLMNOPQRSTUVWXYZ")
ALPHABETS = {
    "two": [0x00, 0xFF],
    "digits3": [0x00] + _chars("01"),
    "four": [0x00] + _chars("\n01"),
    "nine": [0x00] + _chars(" ()aenot"),
    "lower": [0x00] + LOWER,
    "v33": [0x00] + LOWER + _chars(" .,\n[]"),
    "v57": [0x00] + LOWER + UPPER + _chars(" .,\n"),
    "v58": [0x00] + LOWER + UPPER + _chars(" \n()."),
    "high": [0x00] + list(range(0x80, 0x100)),
    "v254": [0x00] + list(range(0x02, 0xFF)),
    "v255": list(range(0x00, 0xFF)),
}
ALPHABETS = {k: sorted(set(v)) for k, v in ALPHABETS.items()}

# fixture tests/golden/vocab_<name>.npz: (data bytes, seed). The coded stream is 5 bytes longer; every length is at least
# 10000 - 5 and its nonzero bytes lie in the alphabet
STREAMS = {"two": (0xFF00, 0x70CAB000), "digits3": (0x3000, 0x70CAB001), "four": (0x300A, 0x70CAB002),
           "nine": (0x2800, 0x70CAB003), "lower": (0x6100, 0x70CAB004), "v33": (0x2E2E, 0x70CAB005),
           "v57": (0x2E00, 0x70CAB006), "v58": (0x2E00, 0x70CAB007), "high": (0x8000, 0x70CAB008),
           "v254": (0x2800, 0x70CAB009), "v255": (0x2800, 0x70CAB00A)}
DUMP = 4096          # coded bytes a fixture keeps (about 40 BPTT rounds of the LSTM) ...
FULL = "lower"       # ... but this one keeps its whole stream
DUMPED = {name: (n + 5 if name == FULL else DUMP) for name, (n, _) in STREAMS.items()}


def _mapping(alphabet, source):
    """A 256-entry table that sends each byte of `source` into `alphabet` (see the module's docstring)."""
    have = set(alphabet)
    fold = np.arange(256)
    for c in UPPER:
        if c not in have and c + 32 in have:
            fold[c] = c + 32
    own = [p for p in PAIRS if p[0] in have and p[1] in have]
    for p in PAIRS:
        if own and not (p[0] in have and p[1] in have):
            fold[p[0]], fold[p[1]] = own[0]
    src = fold[source]
    counts = np.bincount(src, minlength=256)
    ranked = sorted((c for c in range(256) if counts[c]), key=lambda c: (-counts[c], c))
    unused = [a for a in alphabet if not counts[a]]
    order = unused + [a for a in alphabet if a not in unused]
    table = np.zeros(256, dtype=np.uint8)
    k = 0
    for c in ranked:
        if c in have:
            table[c] = c
        else:
            table[c] = order[k % len(order)]
            k += 1
    return table[fold]


def generate(name, n_bytes, seed):
    """n_bytes of stream `name`: its alphabet, then mapped text with runs and a repeated phrase (module docstring)."""
    alphabet = np.array(ALPHABETS[name], dtype=np.uint8)
    rng = np.random.default_rng(seed)
    source = np.frombuffer(synth_text(n_bytes + 4096, seed), dtype=np.uint8)
    text = _mapping(list(alphabet), source)[source].astype(np.uint8)
    phrase = text[:96].copy()
    out, size, pos, tour_at = [], 0, 0, 0
    while size < n_bytes:
        if size >= tour_at:
            out.append(alphabet)
            tour_at += TOUR
        else:
            r = rng.random()
            if r < 0.12:
                out.append(np.full(int(rng.integers(8, 64)), alphabet[int(rng.integers(0, alphabet.size))], dtype=np.uint8))
            elif r < 0.42:
                out.append(phrase)
            else:
                k = int(rng.integers(24, 200))
                out.append(text[pos:pos + k])
                pos = (pos + k) % (text.size - 400)
        size += out[-1].size
    out = np.concatenate(out)[:n_bytes]
    assert out.dtype == np.uint8 and out.size == n_bytes
    return out


def coded_stream(name):
    """The whole stream `cmix -n` codes for fixture `name`: its 5-byte header (0, length u32 big-endian), then the data.
    Its byte set is the alphabet, and it is at least 10000 bytes long, so the reference's vocabulary is the alphabet."""
    n, seed = STREAMS[name]
    s = np.concatenate([np.array([0, n >> 24 & 255, n >> 16 & 255, n >> 8 & 255, n & 255], dtype=np.uint8), generate(name, n, seed)])
    assert s.size >= 10000, "%s: %d coded bytes: the reference would give it every symbol" % (name, s.size)
    assert np.array_equal(np.unique(s), ALPHABETS[name]), "%s: the coded bytes are not the alphabet" % name
    return s


if __name__ == "__main__":
    kind, n, path = sys.argv[1], int(sys.argv[2]), sys.argv[3]
    seed = int(sys.argv[4], 0) if len(sys.argv) > 4 else STREAMS[kind][1]
    generate(kind, n, seed).tofile(path)
