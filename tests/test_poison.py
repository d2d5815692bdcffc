"""No kernel reads shared memory, or device memory the engine did not zero, before something has written it.

On a quiet GPU a read before the write usually finds what the previous launch or call left there, often the value the
code expects; on a shared GPU another user's kernel may have run on the SM in between, and the archive differs from the
reference's only sometimes. cmix_b200/csrc/poison.cuh, built with -DCMIXB200_POISON, puts a pattern in front of every
such read, and every probability, every FXCM / PAQ8 code and every PPMD distribution must still equal the reference
fixture's (tolerance 0). What is poisoned, and the claim each fill tests:

  shared memory, at every kernel's entry (jit_entry): the whole window of the CTA but the system's reserved region, then
    a CTA barrier. Claim: every kernel writes each shared cell before it reads it, in that launch.
  Alloc(..., zero=false), at create: the PPMD arenas (ctx, pool, text) and model registers, the SSE tables s6 / s7 / x1 /
    x2, the bracket model's bk_first / bk_second, every DirectTable's predictions, the LSTM's output, input and gate
    weights, the FXCM / PAQ8 states (d_fx, d_fx_text, d_p8), their table blocks and the dictionary text. Claim: the fill
    kernels, uploads and ppmd_init_kernel write every cell the models read.
  DeviceBuf::Grow, each new buffer: every per-call buffer and staging buffer. Claim: as below, and the 0xFFFF fills of
    d_ext_gen / d_ext_bit, which stay, are the only contents a call finds there.
  each bulk piece: d_small_x, d_sel, d_lstm_x, d_decay, d_lstm_fx, d_ppmd_gen and the resident groups' slots of
    d_ext_gen. Claim: the producers (and the decay upload) write every bit's inputs, selectors, PPMD rows, LSTM feedback
    and codes of the piece before the mixer, or the next producer, reads them; the mixer never takes a code its producer
    has not yet written in this piece.
  each code_bytes / code_batch sub-step: the staging buffers of the bytes, codes and distributions, and d_p. Claim: the
    kernels read only the bytes of the call, and write each probability before the coder or the copy back reads it.
  each lock-step Predict(): StreamState's lock-step scratch (x .. small_x). Claim: Predict()'s kernels write it before
    the final kernel or Perceive() read it.
  each lock-step Perceive(): the resident groups' slots of d_ext_bit, and d_ppmd_byte at the end of a byte with no
    distribution fed. Claim: the FXCM / PAQ8 bit kernels write every code of the next Predict(), and the PPMD model the
    distribution its consumers read.
  decode_bytes: its output buffer, d_ppmd_byte and the lock-step scratch; coder_begin: the archive buffer d_code.

Patterns (cmixb200_poison_config): PATTERN_A, one word everywhere, a quiet NaN as fp32 and far above any 12-bit code,
count or index as u32 or either u16 half; PATTERN_B, a hash per word with the top bit set, seeded by the pattern.

CPU (-m "not gpu"): the poison build compiles for sm_90a; every kernel of it fills shared memory and no product kernel
does; the PPMD model's host build reproduces the reference with its arenas filled with 0xA5 or 0xFF bytes.
GPU (-m gpu): the poison library in a child interpreter (CMIXB200_LIB), once per pattern, over the call schedules
below. The pretraining of full_wrt (412 001 bytes) runs under PATTERN_A; CMIXB200_SLOW=1 runs it under both."""
import ctypes
import json
import os
import time
import zlib

import numpy as np
import pytest

from harness import KERNELS, awkward, batch, child_jobs, code_in_pieces, even, expect, golden, lock_step, \
    ppmd_host, pretrain_buffer, reference_dumps, round_trip, run_child, sass_by_kernel, target, TARGETS  # noqa: F401  (ppmd_host: fixture)

SLOW = os.environ.get("CMIXB200_SLOW") == "1"
PATTERN_A = 0x7FC0A5A5
PATTERN_B = 0xC0FFEE01
PATTERNS = {"A": PATTERN_A, "B": PATTERN_B}
FILL_SR = "SR_SMEMSZ"          # %total_smem_size: read by the fill at kernel entry, by nothing else
BULK = ["full_text", "full_bin", *TARGETS, "stress_random", "stress_zeros", "stress_mixed", "stress_pcm16",
        "audio8_stereo_odd", "wav_pcm8_mono", "vocab_two", "vocab_v255", "overflow_random6k"]
LOCK_BYTES = 16                # the lock-step stretch of a fixture without a target: 16 bytes from the middle
REPLAY_WAV = "wav_pcm16_mono"


@pytest.fixture(scope="session")
def poison_lib(tmp_path_factory):
    """The library compiled with -DCMIXB200_POISON, once per session."""
    from cmix_b200.capi import build_library
    out = tmp_path_factory.getbasetemp() / "poison"
    out.mkdir(exist_ok=True)
    return build_library(defines=["-DCMIXB200_POISON"], out_dir=str(out))


# ------------------------------------------------------------------------------------------------ CPU
def test_poison_build_fills_shared_memory_in_every_kernel_and_the_product_nowhere(poison_lib):
    import cmix_b200
    poison = sass_by_kernel(poison_lib)
    missing = [k for k in KERNELS if k not in poison]
    assert not missing, "kernels not in the poison build: %s" % missing
    unfilled = [k for k in KERNELS if FILL_SR not in poison[k]]
    assert not unfilled, "kernels of the poison build that do not fill shared memory: %s" % unfilled
    assert hasattr(ctypes.CDLL(poison_lib), "cmixb200_poison_config")
    prod = sass_by_kernel(cmix_b200.build_library())
    assert sorted(prod) == sorted(poison), "the two builds hold different kernels"
    filling = [k for k, s in prod.items() if FILL_SR in s]
    assert not filling, "product kernels that read %s: %s" % (FILL_SR, filling)
    assert not hasattr(ctypes.CDLL(cmix_b200.build_library()), "cmixb200_poison_config")


def _ppmd_fixtures():
    names = sorted(f[:-4] for f in os.listdir(os.path.join(os.path.dirname(__file__), "golden")) if f.endswith(".npz"))
    return [n for n in names if n.startswith("ppmd_") or "ppmd_crc" in np.load(os.path.join(os.path.dirname(__file__), "golden", n + ".npz")).files]


@pytest.mark.parametrize("fill", [0xA5, 0xFF])
@pytest.mark.parametrize("name", _ppmd_fixtures())
def test_ppmd_reads_no_arena_cell_it_has_not_written(ppmd_host, name, fill):
    """ppmd_model.h, the code the device runs, on the host with its three arenas filled with `fill` instead of zeroed:
    the distribution after every byte is still the reference's."""
    g = golden(name)
    want = g["crc"] if name.startswith("ppmd_") else g["ppmd_crc"]
    rc, out = ppmd_host(g["stream"], g["vocab"], fill=fill)
    assert rc == 0
    got = np.array([zlib.crc32(out[t].tobytes()) for t in range(out.shape[0])], dtype=np.uint32)
    bad = np.nonzero(got != want)[0]
    assert got.size == want.size and bad.size == 0, "%s, fill %#x: first differing byte %s of %d" % (name, fill, bad[:1], got.size)


# ------------------------------------------------------------------------------------------------ the child
def _span(name, s):
    """The lock-step stretch: the bytes a reach_* stream targets, else LOCK_BYTES from the middle."""
    if name in TARGETS:
        return target(name, s)
    lo = s.size // 2
    return lo, lo + LOCK_BYTES


def _split(pieces):
    """Pieces longer than the debug fetch covers, cut in MAX_PIECE pieces."""
    return [q for a, b in pieces for q in even(a, b)]


def pieces_lock_step(cm, name):
    """Two predictors. One codes bulk pieces of 1, 129, 7, 1000, 333 bytes, then the rest, every code and PPMD distribution
    checked (code_in_pieces) over the stream's whole 4096-bit blocks. The other codes the same pieces to the lock-step
    stretch, Predict()/Perceive() across it, then the same pieces to the end; Predict() is checked at every bit."""
    g = golden(name)
    s, p = g["stream"], g["p"]
    whole = s.size - s.size % 512
    P = cm.Predictor(g["vocab"])
    try:
        code_in_pieces(P, g, _split(awkward(0, whole)))
    finally:
        P.close()
    lo, hi = _span(name, s)
    P = cm.Predictor(g["vocab"])
    try:
        for a, b in awkward(0, lo):
            expect("%s: bulk [%d,%d)" % (name, a, b), P.code_bytes(s[a:b]), p[a * 8:b * 8], a * 8)
        lock_step(P, g, lo * 8, hi * 8, "%s: lock-step [%d,%d)" % (name, lo, hi))
        for a, b in awkward(hi, s.size):
            expect("%s: bulk [%d,%d) after lock-step" % (name, a, b), P.code_bytes(s[a:b]), p[a * 8:b * 8], a * 8)
    finally:
        P.close()


def host_batch(cm, names, n):
    """code_batch from host buffers over the first n bytes of each stream: its 1024-byte sub-steps and double-buffered
    staging."""
    from cmix_b200.capi import code_batch
    gs = [golden(x) for x in names]
    preds = []
    try:
        for g in gs:
            preds.append(cm.Predictor(g["vocab"]))
        outs = [np.empty(n * 8, dtype=np.float32) for _ in gs]
        code_batch(preds, [np.ascontiguousarray(g["stream"][:n]) for g in gs], n, None, None, outs)
        for g, out in zip(gs, outs):
            expect("code_batch of %s, %d bytes each: %s" % (names, n, g["name"]), out, g["p"][:n * 8])
    finally:
        for P in preds:
            P.close()


def pretrain_wrt(cm, dict_path):
    """full_wrt: the dictionary's pretraining in bulk to 64 bytes from its end, those 64 bytes bit by bit through
    Pretrain(), then bulk calls over the stream."""
    pre = pretrain_buffer(dict_path)
    g = golden("full_wrt")
    P = cm.Predictor(g["vocab"], dictionary_path=dict_path)
    try:
        P.pretrain_bytes(pre[:-64])
        for byte in pre[-64:]:
            for k in range(7, -1, -1):
                P.Pretrain((byte >> k) & 1)
        code_in_pieces(P, g, even(0, g["stream"].size))
    finally:
        P.close()


def replay_paq8(cm, name, prefix):
    """PAQ8 replayed from the reference's codes (oracle_dump's at prefix), FXCM and PPMD resident: bulk pieces from byte 0,
    the replayed slots copied into poisoned scratch."""
    from oracle_io import Dump
    from harness import code_crcs
    d = Dump(prefix)
    g = golden(name)
    crc_fx, crc_p8 = code_crcs(d.ext)
    g.update(p=d.p, first_codes=d.ext[:64], crc_fx=crc_fx, crc_p8=crc_p8)
    P = cm.Predictor(g["vocab"], replay=("paq8",))
    try:
        code_in_pieces(P, g, _split(awkward(0, g["stream"].size)), ext=d.ext)
    finally:
        P.close()


def poison_child(pattern, jobs_json):
    """Run in a child interpreter with CMIXB200_LIB = the poison build: the pattern, then each job [schedule, args]. Prints
    one JSON line per job."""
    import cmix_b200
    lib = cmix_b200.load_library()
    lib.cmixb200_poison_config.argtypes = [ctypes.c_uint]
    if lib.cmixb200_poison_config(int(pattern)) != 0:
        raise RuntimeError("poison config: " + lib.cmixb200_last_error().decode())
    port = []

    def run(j, job):
        sched, args = job
        if sched == "pieces":
            pieces_lock_step(cmix_b200, *args)
        elif sched == "batch":
            batch(cmix_b200, *args)
        elif sched == "host_batch":
            host_batch(cmix_b200, *args)
        elif sched == "round_trip":
            if not port:
                from oracle_io import load_port
                port.append(load_port())
            round_trip(cmix_b200, port[0], *args)
        elif sched == "wrt":
            pretrain_wrt(cmix_b200, *args)
        elif sched == "replay_paq8":
            replay_paq8(cmix_b200, *args)
        elif sched == "one_after_another":      # the second predictor is given the first's freed memory, refilled
            for name in args:
                pieces_lock_step(cmix_b200, name)
        else:
            raise ValueError(sched)

    child_jobs(json.loads(jobs_json), run)


def run_poison(poison_lib, pattern, jobs, timeout=1500):
    """The jobs in a child interpreter on the poison build under `pattern`; prints each job's time and fails with every
    failing job's first difference."""
    t0 = time.perf_counter()
    lines = run_child(poison_lib, "test_poison", "poison_child", [str(PATTERNS[pattern]), json.dumps(jobs)], timeout=timeout)
    results = [x for x in lines if "job" in x]
    fails = []
    for x in results:
        sched, args = x["job"]
        what = args if sched != "replay_paq8" else args[:1]
        print("pattern %s  %-18s %-60s %6.1f s%s" % (pattern, sched, str(what)[:60], x["s"], "  FAIL" if x["fail"] else ""))
        if x["fail"]:
            fails.append("pattern %s (%#x), schedule %s %s: %s" % (pattern, PATTERNS[pattern], sched, what, x["fail"]))
    print("pattern %s: %d runs in %.0f s" % (pattern, len(results), time.perf_counter() - t0))
    assert not fails, "%d of %d runs differ from the reference under poison:\n%s" % (len(fails), len(results), "\n".join(fails))
    assert len(results) == len(jobs), "pattern %s: %d of %d runs reported" % (pattern, len(results), len(jobs))


# ------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
@pytest.mark.timeout(1800)
@pytest.mark.parametrize("pattern", sorted(PATTERNS))
def test_bulk_pieces_around_lock_step(poison_lib, pattern):
    """Every fixture of BULK: awkward bulk pieces, a lock-step stretch, bulk pieces to the end."""
    run_poison(poison_lib, pattern, [["pieces", [n]] for n in BULK])


@pytest.mark.gpu
@pytest.mark.timeout(1800)
@pytest.mark.parametrize("pattern", sorted(PATTERNS))
def test_batches_coder_replay_and_reuse(poison_lib, pattern, port, tmp_path):
    """Three reach_* streams in one code_batch_device; code_batch from host buffers across three 1024-byte sub-steps;
    device encoder -> device decoder on full_text; PAQ8 replayed from the reference's codes on a 16-bit WAV stream; two
    predictors created and closed one after the other."""
    dumps = reference_dumps(str(tmp_path), names=[REPLAY_WAV])
    reach = list(TARGETS)
    jobs = [["batch", [reach[:3]]], ["host_batch", [["reach_x86", "stress_mixed"], 3072]],
            ["round_trip", ["full_text", 1024]], ["replay_paq8", [REPLAY_WAV, dumps[REPLAY_WAV].prefix]],
            ["one_after_another", ["reach_dbase", "vocab_two"]]]
    run_poison(poison_lib, pattern, jobs)


@pytest.mark.gpu
@pytest.mark.timeout(1800)
@pytest.mark.parametrize("pattern", sorted(PATTERNS) if SLOW else ["A"])
def test_pretraining(poison_lib, pattern, dict_path):
    """full_wrt with the dictionary and its 412 KB of pretraining, in bulk and then bit by bit."""
    run_poison(poison_lib, pattern, [["wrt", [dict_path]]])
