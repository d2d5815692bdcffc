"""Seeded streams that reach the lines of PAQ8, FXCM and PPMD the other fixtures never run.

    python tools/gen_reach.py <name> <n_bytes> <out> [seed]

The models are single sources for host and device, so a line no fixture runs on the host is never checked on the device
either (tools/coverage_report.py lists those lines). Each stream here is built to run some of them, and is pure Python /
numpy from a seed, so a test can regenerate it and compare it with its fixture:
    english  prose with contractions and negations (don't won't can't ain't shan't), -ably/-ibly/-est/-ness/-ful/-ic/
             -ive words, words hyphenated across a line break with '+' (PAQ8's text model joins them), abbreviations
             (Mr. Dr. St.), also with CR LF line ends
    europe   French and German paragraphs in UTF-8, eight at a time, that reach the irregular and suffix tables of both
             stemmers while their language is the detected one
    xml      wiki XML with <![CDATA[ ... ]]>, <!-- ... -->, entities, ISO and German dates, and coordinates (12°34')
    x86      x86-like code: prologues, 0F 38 xx / 0F 3A xx three-byte opcodes behind 66/F2/F3/REX prefixes, ModRM/SIB
    dbase    dBase III and Visual FoxPro (.dbf) files: header, field descriptors, the 263-byte backlink, records
    bmp      a BITMAPINFOHEADER (size 0x28) whose palette is too large for its bit depth, in text: PAQ8's BMP detector
             checks every field and enters no image mode (nor does the reference's)
    fxwiki   wiki markup in FXCM's alphabet (P Q R for { | }, N for >, @ before a capital): {| |- || |} tables with rows of
             unequal cell counts, rows ending in >, brackets left open for hundreds of bytes, lines opening with ', '' and
             [[, list items, and contractions
None of them carries a header PAQ8's image, audio or JPEG gate accepts. STREAMS holds the (length, seed) of every fixture
tools/make_reach_goldens.py writes.
"""
import sys

import numpy as np


def _pick(rng, seq):
    return seq[int(rng.integers(0, len(seq)))]


def _deck(rng, seq):
    """Draws from `seq` in shuffled rounds, so that every entry appears once in each len(seq) draws."""
    pool = []

    def draw():
        if not pool:
            pool.extend(seq[int(i)] for i in rng.permutation(len(seq)))
        return pool.pop()
    return draw


def _text(parts, n):
    data = "".join(parts).encode("utf-8") if isinstance(parts[0], str) else b"".join(parts)
    assert len(data) >= n, "stream generator too short: %d < %d" % (len(data), n)
    return np.frombuffer(data[:n], dtype=np.uint8).copy()


_EN_SUBJ = ["Mr. Smith", "Dr. Jones", "Mrs. Brown", "Ms. Green", "St. Paul", "the old man", "our neighbour", "Jr. Lee",
            "the teacher", "my sister", "the council"]
_EN_NEG = ["don't", "won't", "can't", "ain't", "shan't", "isn't", "doesn't", "wasn't", "couldn't", "wouldn't", "hasn't"]
_EN_VERB = ["agree", "know", "care", "believe", "remember", "listen", "answer", "think", "wait"]
_EN_ADJ = ["coolest", "smallest", "cleanest", "keenest", "densest", "tersest", "finest", "fullest", "dullest", "boldest",
           "noblest", "humblest", "tallest", "thinnest", "hottest", "happiest", "wettest", "strongest", "longest", "cruellest",
           "shrewdest", "newest", "freshest", "highest", "youngest", "palest", "moistest", "surest", "dearest", "clearest",
           "sourest", "barest", "biggest", "oddest", "saddest", "rarest"]
_EN_ING = ["singing", "hanging", "ringing", "bringing", "changing", "arranging", "lunging", "cringing", "bagging", "plunging",
           "longing", "charging", "singingly", "wringing"]
_EN_ADV = ["ably", "nobly", "possibly", "terribly", "crossly", "grossly", "visibly", "reasonably", "gently", "humbly",
           "horribly", "doubly", "feebly", "probably", "sensibly", "suitably", "basically", "idly", "fully", "oddly"]
_EN_NOUN = ["kindness", "goodness", "darkness", "usefulness", "helpfulness", "harmfulness", "sadness", "hopeful", "graceful",
            "peaceful", "artistic", "electric", "heroic", "massive", "active", "expensive", "creative", "formality", "activity",
            "sensitivity", "electricity", "adaptability", "capability", "historic", "generative", "respectful", "childhood",
            "neighbourhood", "argument", "ability", "conditional", "generalization", "organizer", "operator"]
_EN_HYPH = [("exam", "ple"), ("know", "ledge"), ("inter", "national"), ("govern", "ment"), ("cal", "culation"),
            ("hyphen", "ated"), ("par", "agraph"), ("pro", "cessing")]


def _english(rng, n):
    subj, neg, verb, adj, noun, adv, ing, hyph = (_deck(rng, s) for s in (_EN_SUBJ, _EN_NEG, _EN_VERB, _EN_ADJ, _EN_NOUN, _EN_ADV,
                                                                         _EN_ING, _EN_HYPH))
    out = []
    while sum(map(len, out)) < n:
        nl = "\r\n" if rng.random() < 0.3 else "\n"
        s = "%s said: \"I %s %s, it is the %s %s.\" " % (subj(), neg(), verb(), adj(), noun())
        s += "%s %s %s the %s one, %s and %s, " % (subj().capitalize(), adv(), neg(), adj(), ing(), ing())
        a, b = hyph()
        s += "with %s and %s %s+%s%s %s. " % (noun(), noun(), a, nl, b, adv())
        if rng.random() < 0.4:
            s += "It's the %s's %s, isn't it? " % (noun(), noun())
        # the words the stemmers turn contractions and joined hyphenations into, so that a wrong rewrite splits a context
        s += "I am sure we will, you shall, they can and do, for %s. " % "".join(hyph())
        s += nl if rng.random() < 0.5 else nl + nl
        out.append(s)
    return _text(out, n)


_FR = ["monument", "yeux", "travaux", "possibilité", "activités", "électricité", "spécificité",
       "capacité", "stabilité", "réalité", "dangereuse", "heureuses", "première", "dernière",
       "fermières", "cavaliers", "châteaux", "journaux", "évidemment", "puissamment", "lentement", "finissaient",
       "agir", "finirait", "mangerions", "parlaient", "nation", "question", "organisateur", "admiration", "croyance",
       "sportive", "naïf", "sportifs", "ambiguë", "rapidement", "continuellement", "inquiètes", "logique",
       "communisme", "lisible", "aimable", "révolution", "dissolution", "rougissement", "établissements"]
_DE = ["freundlich", "Freundlichkeit", "Schönheit", "Möglichkeit", "Wahrheit", "Einheit", "herrlich",
       "gefährlich", "Ehrlichkeit", "Gerechtigkeit", "Flüssigkeit", "Feuchtigkeit", "königlich",
       "Sicherheit", "Gesundheit", "Kindheit", "Freiheit", "Bitterkeit", "Heiterkeit", "Zeitung", "Wohnung",
       "lesend", "brennend", "katholisch", "praktisch", "lustig", "mächtig", "Ordnung", "ewiglich", "ärgerlich",
       "Lieblichkeit", "Fr. Müller", "Hr. Weber", "Hrn. Schmidt", "heiligen", "Mädchen", "Bundesländer"]


def _europe(rng, n):
    fr, de = _deck(rng, _FR), _deck(rng, _DE)
    out = []
    while sum(len(p.encode("utf-8")) for p in out) < n:
        if len(out) // 8 % 2 == 0:                    # blocks of eight paragraphs: each language becomes the detected one
            words = [fr() for _ in range(9)]
            out.append("La %s et les %s de M. Dupont, avec %s; c'est %s. %s %s %s l'%s, %s %s.\n" % tuple(words + [""])[:10])
        else:
            words = [de() for _ in range(8)]
            out.append("Die %s und die %s der Stadt sind %s; %s hat %s gesagt, dass %s %s ist, %s.\n" % tuple(words))
    return _text(out, n)


def _xml(rng, n):
    titles = ["Paris", "Berlin", "Zürich", "Ångström", "Lyon", "Genève"]
    out = ['<?xml version="1.0" encoding="utf-8"?>\n<mediawiki xmlns="http://www.mediawiki.org/xml/export-0.3/">\n']
    i = 0
    while sum(len(p.encode("utf-8")) for p in out) < n:
        y, m, d = int(rng.integers(1900, 2030)), int(rng.integers(1, 13)), int(rng.integers(1, 29))
        deg, mi = int(rng.integers(10, 90)), int(rng.integers(10, 60))
        out.append("  <page>\n    <title>%s</title>\n    <id>%d</id>\n    <revision>\n      <timestamp>%04d-%02d-%02dT%02d:%02d:00Z</timestamp>\n"
                   % (_pick(rng, titles), 1000 + i, y, m, d, int(rng.integers(0, 24)), int(rng.integers(0, 60))))
        out.append("      <comment><!-- edit %d: fixed the %s --></comment>\n" % (i, _pick(rng, ["links", "dates", "typo"])))
        out.append("      <text xml:space=\"preserve\">Founded on %02d.%02d.%04d (%04d-%02d-%02d) at %d°%d'N, &amp; %d°%d' east &lt;b&gt;</text>\n"
                   % (d, m, y, y, m, d, deg, mi, deg + 1, mi - 5))
        out.append("      <data><![CDATA[if (a < b && c > d) { x = y; } ]]></data>\n    </revision>\n  </page>\n")
        i += 1
    return _text(out, n)


def _x86(rng, n):
    out = bytearray()
    regs = [0xC0, 0xC1, 0xCA, 0xD3, 0x45, 0x4D, 0x04, 0x0C]
    while len(out) < n:
        r = rng.random()
        if r < 0.08:
            out += bytes([0x55, 0x89, 0xE5, 0x83, 0xEC, int(rng.integers(1, 16)) * 4])                 # push ebp; mov ebp,esp; sub esp
        elif r < 0.3:
            pre = _pick(rng, [b"\x66", b"\xf2", b"\xf3", b"", b"\x66\x48", b"\x48"])
            op3 = _pick(rng, [0x00, 0x01, 0x04, 0x0B, 0x10, 0x17, 0x1C, 0x20, 0x29, 0x37, 0x40, 0xDB, 0xDC, 0xF0, 0xF1])
            modrm = _pick(rng, regs)
            out += pre + bytes([0x0F, 0x38, op3, modrm])
            if modrm in (0x45, 0x4D):
                out.append(int(rng.integers(0, 128)))
            elif modrm in (0x04, 0x0C):
                out += bytes([0x24])
        elif r < 0.5:
            pre = _pick(rng, [b"\x66", b"", b"\x66\x48"])
            op3 = _pick(rng, [0x08, 0x0A, 0x0B, 0x0F, 0x14, 0x16, 0x17, 0x20, 0x21, 0x22, 0x40, 0x44, 0x60, 0x63, 0xDF])
            out += pre + bytes([0x0F, 0x3A, op3, _pick(rng, [0xC0, 0xC1, 0xCA, 0xD3]), int(rng.integers(0, 256))])
        elif r < 0.6:
            out += bytes([0xE8]) + int(rng.integers(-4096, 4096)).to_bytes(4, "little", signed=True)      # call rel32
        elif r < 0.7:
            out += bytes([0x8B, _pick(rng, [0x45, 0x4D, 0x55]), int(rng.integers(0, 64)) * 4])             # mov r32,[ebp+d8]
        elif r < 0.8:
            out += bytes([_pick(rng, [0x0F]), _pick(rng, [0x84, 0x85, 0x8C, 0xAF, 0xB6, 0xBE, 0x10, 0x28, 0x58])])
            out += bytes([_pick(rng, regs)])
        elif r < 0.9:
            out += bytes([_pick(rng, [0xF0, 0x2E, 0x3E, 0x64, 0x65, 0x67]), 0x89, 0x08])
        else:
            out += bytes([_pick(rng, [0x74, 0x75, 0xEB]), int(rng.integers(0, 256)), 0xC3 if rng.random() < 0.3 else 0x90])
    return np.frombuffer(bytes(out[:n]), dtype=np.uint8).copy()


def _dbf(rng, version, fields, nrec, backlink):
    """A .dbf file: 32-byte header, 32-byte field descriptors, 0x0D, the 263-byte backlink (Visual FoxPro), records."""
    rlen = 1 + sum(f[2] for f in fields)
    hlen = 32 + 32 * len(fields) + 1 + (263 if backlink else 0)
    h = bytearray(32)
    h[0], h[1], h[2], h[3] = version, 124, 10, 16
    h[4:8] = nrec.to_bytes(4, "little")
    h[8:10] = hlen.to_bytes(2, "little")
    h[10:12] = rlen.to_bytes(2, "little")
    out = bytes(h)
    for name, kind, width in fields:
        d = bytearray(32)
        d[:len(name)] = name.encode("ascii")
        d[11], d[16] = ord(kind), width
        out += bytes(d)
    out += b"\r" + (bytes(263) if backlink else b"")
    names = [b"ALPHA", b"BRAVO", b"CHARLIE", b"DELTA", b"ECHO", b"FOXTROT"]
    for i in range(nrec):
        rec = b" "
        for name, kind, width in fields:
            if kind == "N":
                v = str(int(rng.integers(0, 10 ** min(width, 6)))).encode("ascii")
                rec += v.rjust(width)
            elif kind == "D":
                rec += b"2026%02d%02d" % (int(rng.integers(1, 13)), int(rng.integers(1, 29)))
            else:
                rec += _pick(rng, names).ljust(width)
        out += rec
    return out + b"\x1a"


def _dbase(rng, n):
    fields = [("ID", "N", 6), ("NAME", "C", 10), ("DATE", "D", 8), ("QTY", "N", 5)]
    out = [b"customer table export\n", _dbf(rng, 0x03, fields, 40, False), b"\nvisual foxpro table\n",
           _dbf(rng, 0x30, fields + [("CITY", "C", 9)], 40, True)]
    while sum(map(len, out)) < n:
        out.append(_dbf(rng, _pick(rng, [0x03, 0x83, 0xF5, 0x30]), fields, 20, rng.random() < 0.5))
    return _text(out, n)


def _bmp(rng, n):
    out = [b"A device-independent bitmap header follows; its palette does not fit its bit depth.\n"]
    hdr = bytearray(40)
    hdr[0:4] = (0x28).to_bytes(4, "little")
    hdr[4:8] = (16).to_bytes(4, "little")
    hdr[8:12] = (16).to_bytes(4, "little")
    hdr[12:14] = (1).to_bytes(2, "little")                  # planes
    hdr[14:16] = (1).to_bytes(2, "little")                  # bits per pixel
    hdr[36:40] = (3).to_bytes(4, "little")                  # important colours: 3 > 2 ** 1
    out.append(bytes(hdr))
    out.append(bytes(int(v) for v in rng.integers(0, 4, size=64) * 0x41))
    hdr[12:14] = (2).to_bytes(2, "little")                  # planes 2: fails on the first field check
    hdr[36:40] = bytes(4)
    out += [b"\nAnd one with two planes.\n", bytes(hdr)]
    while sum(map(len, out)) < n:
        out.append(b"%d,%d;" % (int(rng.integers(0, 1000)), int(rng.integers(0, 1000))))
    return _text(out, n)


def _fxwiki(rng, n):
    words = ["the", "city", "river", "north", "station", "line", "year", "county", "people", "house"]
    out = []
    while sum(map(len, out)) < n:
        r = rng.random()
        if r < 0.3:                                   # {| table |- rows || cells |}
            rows = ["PPQ class=Mwikitable\n"]
            for _ in range(int(rng.integers(2, 5))):
                cells = [_pick(rng, words) for _ in range(int(rng.integers(1, 5)))]
                rows.append("Q-\nQ " + " QQ ".join(cells) + "\n")
                if rng.random() < 0.5:
                    rows.append("Q " + _pick(rng, words) + "\n")
            rows.append("QRR\n")
            out.append("".join(rows))
        elif r < 0.45:                                # html rows ending in >
            cells = "".join("Ltd N%s L/td N" % _pick(rng, words) for _ in range(int(rng.integers(1, 4))))
            out.append("Ltr N\nN%s\nN'%s L/tr N\n" % (cells, _pick(rng, words)))
        elif r < 0.55:                                # brackets open for hundreds of bytes
            body = " ".join(_pick(rng, words) for _ in range(int(rng.integers(50, 70))))
            out.append("( [ P %s\n" % body)
        elif r < 0.7:                                 # paragraphs opening with ' '' [[ and list items
            out.append("''@%s'' is a %s. '''@%s''' %s.\n" % (_pick(rng, words), _pick(rng, words), _pick(rng, words), _pick(rng, words)))
            out.append("[[%s]] %s [[%s]]\n" % (_pick(rng, words), _pick(rng, words), _pick(rng, words)))
            out.append("' %s ' %s\n''''@%s\n" % (_pick(rng, words), _pick(rng, words), _pick(rng, words)))
            out.append("Ltext xml:space=\"preserve\"N%s%s is a %s.L/textN\n" % (_pick(rng, ["@", "'''"]), _pick(rng, words), _pick(rng, words)))
        elif r < 0.85:
            out.append("* %s %s\n* @%s %s\n" % (_pick(rng, words), _pick(rng, words), _pick(rng, words), _pick(rng, words)))
        else:
            out.append("@we %s %s, @they %s, it %s and %s.\n" % (_pick(rng, _EN_NEG), _pick(rng, _EN_VERB), _pick(rng, _EN_NEG),
                                                            _pick(rng, _EN_NEG), _pick(rng, _EN_NEG)))
    return _text(out, n)


CLASSES = {"english": _english, "europe": _europe, "xml": _xml, "x86": _x86, "dbase": _dbase, "bmp": _bmp, "fxwiki": _fxwiki}


def generate(kind, n_bytes, seed):
    """n_bytes of class `kind` from np.random.default_rng(seed)."""
    out = CLASSES[kind](np.random.default_rng(seed), n_bytes)
    assert out.dtype == np.uint8 and out.size == n_bytes
    return out


# fixture tests/golden/reach_<name>.npz: (n_bytes, seed); lengths are whole 4096-bit CRC blocks
STREAMS = {name: (3072, 0x4EAC400 + i) for i, name in enumerate(CLASSES)}


def coded_stream(name):
    """The first n_bytes bytes `cmix -n` codes for fixture `name`: its 5-byte header (0, length u32 big-endian), then the data."""
    n, seed = STREAMS[name]
    return np.concatenate([np.array([0, n >> 24 & 255, n >> 16 & 255, n >> 8 & 255, n & 255], dtype=np.uint8), generate(name, n, seed)])[:n]


if __name__ == "__main__":
    kind, n, path = sys.argv[1], int(sys.argv[2]), sys.argv[3]
    seed = int(sys.argv[4], 0) if len(sys.argv) > 4 else STREAMS[kind][1]
    generate(kind, n, seed).tofile(path)
