#!/usr/bin/env python
"""Build a profiling variant of the library (-DP8_PROF -DFX_PROF: per-phase cycle counters in the producer kernels) into
cmix_b200/csrc/prof/ and print where a bit's time goes. Never used by the product path, the tests or bench.py.

    python tools/prof_build.py build            # here (nvcc cross-compiles)
    python tools/prof_build.py run [n_bytes]    # on the GPU box: CMIXB200_LIB=<prof lib> is set by this script
"""
import ctypes
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "cmix_b200", "csrc")
PROF_DIR = os.path.join(CSRC, "prof")
PROF_LIB = os.path.join(PROF_DIR, "libcmixb200.so")


# PAQ8's slots. 0-11 add up to the model CTA's bit, 16-19 to the mixer CTA's. From 24 on: inside a byte the time a warp spent
# in the probe (24 + warp) and apply (48 + warp) phases; on the bit that starts a byte the time, counted from the end of the
# bookkeeping, at which a chain reached a point. The byte boundary's critical path is the latest of 24-30, 34-36 and 38,
# which is what slot 2 waits for.
P8_LABELS = {
    0: "bookkeeping", 2: "byte boundary: until every chain is done (the join)", 3: "inside a byte: probe",
    6: "byte boundary: probe of the 7-slot maps and the text history map", 7: "number (bits with a clash)", 8: "apply",
    9: "selector sets, joining warp 12", 10: "waiting for a free ring slot", 11: "handing the bit over",
    16: "mixer CTA: waiting for the model CTA", 17: "mixer CTA: SGD", 18: "mixer CTA: dot products", 19: "mixer CTA: final mixer, SSE",
    24: "OLS 0 done | probe, warp 0", 25: "OLS 1 done | probe, warp 1", 26: "OLS 2 done | probe, warp 2", 27: "XML done | probe, warp 3",
    28: "distance, record1 done | probe, warp 4", 29: "word chain done | probe, warp 5", 30: "nest, indirect done | probe, warp 6",
    31: "D-chain: order-N and x86 contexts set | probe, warp 7", 32: "D-chain: history maps probed, match model | probe, warp 8",
    33: "D-chain: history maps applied | probe, warp 9", 34: "D-chain: sparse done | probe, warp 10", 35: "D-chain: sparse1 done | probe, warp 11",
    36: "D-chain: record done", 38: "text chain done",
}
P8_LABELS.update({48 + w: "apply, warp %d" % w for w in range(16)})
for w in range(13, 16):
    P8_LABELS[24 + w] = (P8_LABELS[24 + w] + " | " if 24 + w in P8_LABELS else "") + "probe, warp %d" % w
# 64 + g: single-lane unit g, the time from its warp's entry into the phase's unit code to the end of the unit (the latest
# lane; where a warp's lanes diverge into several units this includes the units that ran before it). Inside a byte only.
P8_UNITS = {
    0: "probe: pic_core", 1: "probe: match_core", 2: "probe: record_pre", 3: "probe: rcm_mix x3", 4: "probe: dmc_st x10",
    5: "probe: smatch_head",
    10: "apply: sm32_p x5 (match x3, order 0-1 x2)", 11: "apply: scm_mix x18 (match, record, sparse1, linear)",
    12: "apply: stm_mix x13 (match, record, sparse match)", 13: "apply: imap_mix x3 (record)", 14: "apply: DMC combination, add(64)",
    17: "apply: pic_unit x3",
    20: "lane 0: bit_begin, block_parse", 21: "lane 0: word_stats snapshot", 22: "lane 0: its share of clearing `seen`",
    23: "lane 0: epilogue (main_select_fixed, padding)",
}
P8_LABELS.update({64 + g: "unit: " + s for g, s in P8_UNITS.items()})
# 88 + k: leg k of a 7-slot map context's bit, the longest lane of the bit (each leg apart)
P8_LEGS = ["probe: state read", "probe: touched_buckets", "probe: p8_claim", "apply: draw",
           "apply: store and move (bucket_find at bpos 2, 5, 0)", "apply: run record input", "apply: cell state and StateMap load",
           "apply: other exports"]
P8_LABELS.update({88 + k: "7-slot lane leg: " + s for k, s in enumerate(P8_LEGS)})
P8_ROWS, P8_SLOTS = 6, 128
P8_CLASSES = ["byte boundary", "inside a byte", "same bucket", "same bucket, clash", "new bucket", "new bucket, clash"]


P8_PROF_N = P8_SLOTS - 1   # the model CTA's bits in a row

# FXCM's slots. 0-6 add up to the model CTA's bit (12 and 13 split lane 0's share of slot 0; the rest of it is the
# barrier), 16-20 to the mixer CTA's.
FX_LABELS = {
    0: "model CTA: bookkeeping", 1: "model CTA: unit offsets", 2: "model CTA: probe", 3: "model CTA: apply",
    4: "model CTA: map epilogue, selectors", 5: "model CTA: waiting for a free ring slot", 6: "model CTA: handing the bit over",
    12: "  of 0, lane 0: bit_head_model", 13: "  of 0, lane 0: text_byte at the byte boundary",
    16: "mixer CTA: error terms, failure history", 17: "mixer CTA: SGD", 18: "mixer CTA: waiting for the model CTA",
    19: "mixer CTA: row moves, dot products", 20: "mixer CTA: squash, final mixers, APMs",
}


def paq8_classes(a):
    """The model CTA's cycles per bit by phase and unit, one column per class of bit (row 1 = rows 2-5)."""
    n = a[:, P8_PROF_N]
    cols = [r for r in range(P8_ROWS) if n[r]]
    print("paq8 model CTA: cycles per bit by class of bit (bits: %s)" % ", ".join("%s %d" % (P8_CLASSES[r], n[r]) for r in cols))
    print("  %-5s " % "slot" + "".join("%19s" % P8_CLASSES[r] for r in cols))
    for k in list(range(16)) + list(range(24, P8_PROF_N)):
        if any(a[r, k] for r in cols):
            print("  %-5d " % k + "".join("%19.0f" % (a[r, k] / n[r]) for r in cols) + "   " + P8_LABELS.get(k, ""))
    print("  %-5s " % "total" + "".join("%19.0f" % (a[r, :16].sum() / n[r]) for r in cols))


def build():
    sys.path.insert(0, ROOT)
    from cmix_b200.capi import build_library
    os.makedirs(PROF_DIR, exist_ok=True)
    print(build_library(force=True, defines=["-DP8_PROF", "-DFX_PROF"], out_dir=PROF_DIR))


def run(n_bytes):
    os.environ.setdefault("CMIXB200_LIB", PROF_LIB)   # or another profiling build, to compare two
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import numpy as np
    import torch
    import cmix_b200
    from cmix_b200.capi import load_library
    from gen_synth import synth_text
    text = np.frombuffer(synth_text(n_bytes * 2, 0xE9E80001), dtype=np.uint8).copy()
    vocab = np.zeros(256, dtype=np.uint8)
    vocab[np.unique(text)] = 1
    P = cmix_b200.Predictor(vocab)
    P.code_bytes(text[:n_bytes])
    lib = load_library()
    sm_mhz = torch.cuda.get_device_properties(0).clock_rate / 1e3 if hasattr(torch.cuda.get_device_properties(0), "clock_rate") else 1980.0
    for name, fn, size in (("paq8", "cmixb200_p8_prof", P8_ROWS * P8_SLOTS), ("fxcm", "cmixb200_fx_prof", 2 * 24)):
        if not hasattr(lib, fn):
            continue
        buf = (ctypes.c_ulonglong * size)()
        getattr(lib, fn)(buf, 1)
    P.time_mix_kernel(True)
    P.code_bytes(text[n_bytes:2 * n_bytes])
    for w, k in enumerate(["mix", "small", "lstm", "ppmd", "fxcm", "paq8"]):
        ms, n = P.kernel_ms(w)
        print("%-6s %8.2f us/bit (%d launches)" % (k, ms * 1e3 / (n_bytes * 8), n))
    for name, fn, rows in (("paq8", "cmixb200_p8_prof", P8_SLOTS), ("fxcm", "cmixb200_fx_prof", 24)):
        try:
            f = getattr(lib, fn)
        except AttributeError:
            continue
        n_rows = P8_ROWS if name == "paq8" else 2
        buf = (ctypes.c_ulonglong * (n_rows * rows))()
        f(buf, 0)
        a = np.array(list(buf), dtype=np.float64).reshape(n_rows, rows)
        if name == "paq8":
            paq8_classes(a)
            a = a[:2, :P8_PROF_N]
        print("%s: cycles per bit by phase (byte-boundary bits | other bits); clock %.0f MHz" % (name, sm_mhz))
        for k in range(a.shape[1]):
            if a[0, k] or a[1, k]:
                print("  phase %2d  %9.0f | %9.0f   %s" % (k, a[0, k] / n_bytes, a[1, k] / (7 * n_bytes), (P8_LABELS if name == "paq8" else FX_LABELS).get(k, "")))
        # PAQ8 and FXCM run on two CTAs: PAQ8's model CTA counts in slots 0-15 (10: waiting for a free ring slot), FXCM's in
        # 0-11, their mixer CTAs in 16-23; each CTA's total is its time per bit, less the mixer CTA's code-row writes
        parts = (("model CTA", 0, 16), ("mixer CTA", 16, 24)) if name == "paq8" else (("model CTA", 0, 12), ("mixer CTA", 16, 24))
        for label, lo, hi in parts:
            print("  %-9s %9.0f | %9.0f   -> %.1f us/bit average" % (label, a[0, lo:hi].sum() / n_bytes, a[1, lo:hi].sum() / (7 * n_bytes),
                                                                    a[:, lo:hi].sum() / (8 * n_bytes) / sm_mhz))
    P.close()


if __name__ == "__main__":
    if sys.argv[1] == "build":
        build()
    else:
        run(int(sys.argv[2]) if len(sys.argv) > 2 else 1024)
