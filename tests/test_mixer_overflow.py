"""The mixers' shared overflow row, in every kernel and call schedule, against the CPU restatement (oracle/port).

Mixer::GetContextData (reference mixer.cpp:16-36) gives each new context its own weight row until a mixer holds 10 000 of
them; every later new context shares one overflow row and its step counter. On the device that is assign_row /
resolve_slot (mixer.cuh), and three places must then agree with the reference: the bulk kernel's double-buffered row cache
(mixer_bulk.cuh: K_SAME / K_SWAP / K_LATE_SWITCH, evict and reload, per-buffer steps and dirty flags), the T warp's
resident layer-1 rows, and the lock-step kernels (mixer_lock.cuh). Past the cap many contexts share one row, so rows
switch more often, the shared counter drives max_steps, and the shrink of every 1024th step of a row comes sooner.

The streams code 6000 bytes over all 256 symbols, which takes eleven mixers past the cap (seed 1: the first at byte
2231), three of them in layer 1. A third stream alternates fresh bytes with repeats of its first 1500 bytes, so that
rows assigned before the cap are revisited after it, a few bits away from contexts that fall into the overflow row.
FXCM, PAQ8 and PPMD are replayed from seeded codes, so the port is the reference; every probability must equal the
port's bit for bit. Each test asserts that its stream reaches the cap where it claims to, from the selectors the device
used.

The port runs each stream once (module fixture, streams in parallel threads: about 30 s per stream on one core)."""
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from conftest import synthetic_streams
from harness import AUX, DBG_SEL, LAYER1, N_MIXERS, SEL_PITCH, cm, expect, onsets, ppmd_arena  # noqa: F401  (cm, ppmd_arena: fixtures)

pytestmark = pytest.mark.gpu

N_BYTES = 6000
REPLAY_ALL = ("fxcm", "paq8")
# seed 1: mixer -> the byte at which it meets its 10 001st context (the first one that takes the overflow row)
SEED1_ONSETS = {4: 2231, 23: 2424, 2: 2437, 3: 2437, 16: 3410, 44: 3410, 19: 3923, 43: 3923, 22: 4038, 45: 4038, 5: 5371}
# bulk calls of awkward sizes whose boundaries fall on seed 1's onsets
PIECES = [1, 127, 129, 1000, 974, 193, 13, 973, 513, 115, 1333, 629]


def churn_streams(n_bytes, seed):
    """Fresh random bytes (1500, then runs of 4..48) alternating with runs that repeat a window of the first 1500 bytes;
    model codes and PPMD distributions made as in conftest.synthetic_streams."""
    rng = np.random.default_rng(seed)
    parts, n = [rng.integers(0, 256, size=1500, dtype=np.uint8)], 1500
    fresh = True
    while n < n_bytes:
        k = int(rng.integers(4, 49))
        if fresh:
            seg = rng.integers(0, 256, size=k, dtype=np.uint8)
        else:
            o = int(rng.integers(0, 1500 - k))
            seg = parts[0][o:o + k]
        parts.append(seg)
        n += k
        fresh = not fresh
    stream = np.concatenate(parts)[:n_bytes]
    stream[:1500][rng.random(1500) < 0.15] = 32
    vocab = np.zeros(256, dtype=np.uint8)
    vocab[np.unique(stream)] = 1
    bits = np.unpackbits(stream)
    noise = rng.normal(0.0, 1.2, size=(bits.size, 2022)).astype(np.float32)
    skill = rng.uniform(0.0, 1.5, size=2022).astype(np.float32)
    logit = noise + skill * (2.0 * bits[:, None].astype(np.float32) - 1.0)
    codes = np.clip(np.rint(4095.0 / (1.0 + np.exp(-logit))), 0, 4095).astype(np.uint16)
    codes[:, 429:431] = 0xFFFF
    ppmd = rng.gamma(0.3, 1.0, size=(n_bytes, 256)).astype(np.float32) + 1e-6
    nxt = np.roll(stream, -1)
    ppmd[np.arange(n_bytes), nxt] += rng.uniform(0, 8, size=n_bytes).astype(np.float32)
    ppmd *= vocab[None, :]
    ppmd = (ppmd / ppmd.sum(axis=1, keepdims=True)).astype(np.float32)
    return stream, vocab, codes, ppmd


STREAMS = {
    "seed1": lambda: synthetic_streams(N_BYTES, seed=1, vocab_lo=0, vocab_hi=256),
    "seed2": lambda: synthetic_streams(N_BYTES, seed=2, vocab_lo=0, vocab_hi=256),
    "churn": lambda: churn_streams(N_BYTES, seed=3),
}


def port_trace(port, vocab, stream, codes, ppmd):
    """The port's Predict() of every bit and the 47 mixer contexts it selected for it."""
    v = np.ascontiguousarray(vocab, dtype=np.uint8)
    codes = np.ascontiguousarray(codes)
    ppmd = np.ascontiguousarray(ppmd)
    bits = np.unpackbits(stream)
    p = np.empty(bits.size, dtype=np.float32)
    ctx = np.empty((bits.size, N_MIXERS), dtype=np.uint32)
    P = port.op_create(v.ctypes.data)
    e0, q0, c0, row = codes.ctypes.data, ppmd.ctypes.data, ctx.ctypes.data, codes.shape[1] * 2
    for t in range(bits.size):
        p[t] = port.op_predict(P, e0 + t * row)
        port.op_get_mixer_contexts(P, c0 + t * N_MIXERS * 4)
        port.op_perceive(P, int(bits[t]), q0 + (t // 8) * 1024)
    port.op_destroy(P)
    return p, ctx


@pytest.fixture(scope="module")
def runs(port):
    """name -> (stream, vocab, codes, ppmd, port probabilities, port contexts, port onsets), ports in parallel threads."""
    t0 = time.time()
    data = {k: f() for k, f in STREAMS.items()}
    with ThreadPoolExecutor(len(data)) as ex:
        futs = {k: ex.submit(port_trace, port, d[1], d[0], d[2], d[3]) for k, d in data.items()}
        out = {k: d + futs[k].result() for k, d in data.items()}
    print("\nport over %d streams of %d bytes: %.1f s" % (len(out), N_BYTES, time.time() - t0))
    for k, r in out.items():
        out[k] = r + (onsets(r[5]),)
        print("%s: mixers past the cap at byte %s" % (k, sorted(out[k][6].items(), key=lambda kv: (kv[1], kv[0]))))
    return out


def test_streams_reach_the_cap_where_stated(runs):
    """What the schedules below rely on: seed 1 takes the eleven mixers of SEED1_ONSETS past the cap at those bytes, and
    every stream takes at least one layer-1 mixer (the T warp's rows) past it well before its end."""
    assert runs["seed1"][6] == SEED1_ONSETS
    for name, r in runs.items():
        on = r[6]
        assert any(m in LAYER1 and b < N_BYTES - 1000 for m, b in on.items()), "%s: no layer-1 mixer past the cap: %s" % (name, on)
        assert len([b for b in on.values() if b < N_BYTES - 1000]) >= 4, "%s: %s" % (name, on)


@pytest.mark.timeout(600)
@pytest.mark.parametrize("name", list(STREAMS))
def test_one_bulk_call(cm, runs, name):
    """One code_bytes_device call over the whole stream; the device's selectors of every bit equal the port's contexts,
    so the onsets are the device's own."""
    import torch
    stream, vocab, codes, ppmd, want, ctx, on = runs[name]
    dev = torch.device("cuda", 0)
    P = cm.Predictor(vocab, replay=REPLAY_ALL)
    try:
        out = torch.empty(stream.size * 8, dtype=torch.float32, device=dev)
        P.code_bytes_device(torch.from_numpy(stream).to(dev), stream.size, torch.from_numpy(codes.view(np.int16)).to(dev),
                            torch.from_numpy(ppmd).to(dev), out)
        torch.cuda.synchronize()
        sel = P.debug_fetch(DBG_SEL, (stream.size * 8, SEL_PITCH), np.uint32)[:, :N_MIXERS]
    finally:
        P.close()
    cols = [m for m in range(N_MIXERS) if m != AUX]
    bad = np.argwhere(sel[:, cols] != ctx[:, cols])
    assert bad.size == 0, "%s: device selector of mixer %d at bit %d differs from the port's context" % (name, cols[bad[0][1]], bad[0][0])
    assert onsets(sel) == on
    print("%s: device reaches the cap at %s" % (name, sorted(on.items(), key=lambda kv: (kv[1], kv[0]))))
    expect("%s: one bulk call" % name, out.cpu().numpy(), want)


@pytest.mark.timeout(600)
@pytest.mark.parametrize("name", list(STREAMS))
def test_bulk_calls_of_awkward_sizes(cm, runs, name):
    stream, vocab, codes, ppmd, want, _, _ = runs[name]
    assert sum(PIECES) == stream.size
    P = cm.Predictor(vocab, replay=REPLAY_ALL)
    try:
        off = 0
        for n in PIECES:
            expect("%s: bulk calls of %s, the call [%d,%d)" % (name, PIECES, off, off + n),
                   P.code_bytes(stream[off:off + n], codes[off * 8:(off + n) * 8], ppmd[off:off + n]), want[off * 8:(off + n) * 8], off * 8)
            off += n
    finally:
        P.close()


@pytest.mark.timeout(600)
@pytest.mark.parametrize("name", list(STREAMS))
def test_lock_step_across_the_first_onsets(cm, runs, name):
    """Bulk up to 30 bytes before the first onset, 300 bytes of Predict()/Perceive() (the lock-step kernels meet the
    overflow row of several mixers), then bulk to the end."""
    stream, vocab, codes, ppmd, want, _, on = runs[name]
    lo = min(on.values()) - 30
    hi = lo + 300
    crossed = sorted(m for m, b in on.items() if lo <= b < hi)
    assert crossed, "%s: no onset in lock-step [%d,%d)" % (name, lo, hi)
    sched = "%s: bulk [0,%d), lock-step [%d,%d) (mixers %s reach the cap), bulk [%d,%d)" % (name, lo, lo, hi, crossed, hi, stream.size)
    bits = np.unpackbits(stream)
    P = cm.Predictor(vocab, replay=REPLAY_ALL)
    try:
        expect(sched + ", bulk", P.code_bytes(stream[:lo], codes[:lo * 8], ppmd[:lo]), want[:lo * 8])
        got = np.empty((hi - lo) * 8, dtype=np.float32)
        for t in range(lo * 8, hi * 8):
            P.feed_external_bit(codes[t])
            got[t - lo * 8] = P.Predict()
            if t % 8 == 7:
                P.feed_external_byte(ppmd[t // 8])
            P.Perceive(int(bits[t]))
        expect(sched + ", lock-step", got, want[lo * 8:hi * 8], lo * 8)
        expect(sched + ", bulk", P.code_bytes(stream[hi:], codes[hi * 8:], ppmd[hi:]), want[hi * 8:], hi * 8)
    finally:
        P.close()


@pytest.mark.timeout(600)
def test_streams_in_one_batch(cm, runs):
    """The three streams side by side in code_batch (1024-byte staging): each keeps its own overflow row and counters."""
    from cmix_b200.capi import code_batch
    names = list(STREAMS)
    rs = [runs[k] for k in names]
    preds = []
    try:
        for r in rs:
            preds.append(cm.Predictor(r[1], replay=REPLAY_ALL))
        outs = [np.empty(N_BYTES * 8, dtype=np.float32) for _ in rs]
        code_batch(preds, [r[0] for r in rs], N_BYTES, [r[2] for r in rs], [r[3] for r in rs], outs)
    finally:
        for P in preds:
            P.close()
    for name, r, out in zip(names, rs, outs):
        expect("batch of %s: %s" % (names, name), out, r[4])
