"""Call schedules of the complete resident predictor (every model group on the device) against the reference's Predict().

Each mode switch, batch shape and sub-chunk plan of engine.cu is its own host path: bulk -> lock-step -> bulk, Pretrain
(bulk and per bit) -> Predict(), decode after a bulk prefix or after pretraining, bulk calls of every size class, and
three resident streams at different positions in one launch set (one or two launch groups). The fixtures
(tests/golden/full_*.npz) hold the reference's Predict() for every bit of one stream from a fresh predictor, so whatever
the schedule, each probability must equal the fixture's float bit for bit (tolerance 0).

One full predictor holds about 22 GB of HBM: single-stream tests close each predictor before opening the next."""
import os
import time

import numpy as np
import pytest

from harness import child_jobs, cm, expect, first_bad_byte, golden, host_archive, lock_step, ppmd_arena, pretrain_buffer, \
    run_child  # noqa: F401  (cm, ppmd_arena: fixtures)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def pre(dict_path):
    return pretrain_buffer(dict_path)


def _pretrain(P, data, what):
    t0 = time.perf_counter()
    P.pretrain_bytes(data)
    print("%s: pretrain_bytes(%d bytes) %.1f s" % (what, len(data), time.perf_counter() - t0))


# ------------------------------------------------------------------------------------------------ one stream
@pytest.mark.timeout(900)
@pytest.mark.parametrize("name", ["full_text", "full_bin"])
def test_bulk_then_lock_step_then_bulk(cm, name):
    """The first lock-step Predict() after a bulk call takes the resident models' current codes; a bulk call mid-byte is
    refused without disturbing the stream; bulk resumes where lock-step left off."""
    g = golden(name)
    s, p = g["stream"], g["p"]
    sched = "%s: bulk [0,300), lock-step [300,341), bulk [341,1024)" % name
    P = cm.Predictor(g["vocab"])
    try:
        expect(sched + ", bulk", P.code_bytes(s[:300]), p[:300 * 8])
        lock_step(P, g, 300 * 8, 340 * 8 + 3, sched)
        with pytest.raises(RuntimeError, match="byte boundary"):
            P.code_bytes(s[341:400])
        lock_step(P, g, 340 * 8 + 3, 341 * 8, sched + " (after the refused bulk call)")
        expect(sched + ", bulk", P.code_bytes(s[341:1024]), p[341 * 8:1024 * 8], 341 * 8)
    finally:
        P.close()


@pytest.mark.timeout(900)
def test_pretrain_then_lock_step(cm, dict_path, pre):
    """The shim's order for `cmix -c english.dic`: pretrain_bytes over header + dictionary, then Predict()/Perceive()."""
    g = golden("full_wrt")
    sched = "full_wrt: pretrain_bytes(dictionary), lock-step [0,32), bulk [32,1024)"
    P = cm.Predictor(g["vocab"], dictionary_path=dict_path)
    try:
        _pretrain(P, pre, "full_wrt")
        lock_step(P, g, 0, 32 * 8, sched)
        expect(sched + ", bulk", P.code_bytes(g["stream"][32:1024]), g["p"][32 * 8:1024 * 8], 32 * 8)
    finally:
        P.close()


@pytest.mark.timeout(900)
def test_bit_level_pretrain_with_resident_models(cm, dict_path, pre):
    """Pretrain(bit) through the resident FXCM and PAQ8 bit kernels continues bulk pretraining exactly."""
    g = golden("full_wrt")
    P = cm.Predictor(g["vocab"], dictionary_path=dict_path)
    try:
        _pretrain(P, pre[:-64], "full_wrt")
        for byte in pre[-64:]:
            for j in range(7, -1, -1):
                P.Pretrain((byte >> j) & 1)
        expect("full_wrt: pretrain_bytes(all but 64 bytes), Pretrain(bit) x 512, bulk [0,1024)",
               P.code_bytes(g["stream"][:1024]), g["p"][:1024 * 8])
    finally:
        P.close()


def _decode_schedule(cm, port, g, prepare, n_prefix, n_code, sched, dictionary=None):
    """Encoder and decoder are brought to the same state by `prepare`; the device coder then writes the reference's archive
    for the next n_code bytes, the device decoder gets them back, and a bulk call after the decoder still matches."""
    s, p = g["stream"], g["p"]
    lo, hi = n_prefix, n_prefix + n_code
    enc = cm.Predictor(g["vocab"], dictionary_path=dictionary)
    try:
        prepare(enc)
        enc.coder_begin(2 * n_code + 64)
        expect(sched + ", encoder bulk", enc.code_bytes(s[lo:hi]), p[lo * 8:hi * 8], lo * 8)
        archive = enc.coder_finish()
    finally:
        enc.close()
    want = host_archive(port, p[lo * 8:hi * 8], np.unpackbits(s[lo:hi]))
    assert archive == want, "%s: device archive differs from the host encoder's: %s" % (sched, first_bad_byte(archive, want))
    dec = cm.Predictor(g["vocab"], dictionary_path=dictionary)
    try:
        prepare(dec)
        out = dec.decode_bytes(archive, n_code)
        assert out.tobytes() == s[lo:hi].tobytes(), "%s, decoder: %s" % (sched, first_bad_byte(out, s[lo:hi]))
        expect(sched + ", bulk after the decoder", dec.code_bytes(s[hi:hi + 32]), p[hi * 8:(hi + 32) * 8], hi * 8)
    finally:
        dec.close()


@pytest.mark.timeout(900)
def test_decode_after_a_bulk_prefix(cm, port):
    g = golden("full_text")

    def prefix(P):
        expect("full_text: bulk prefix [0,256)", P.code_bytes(g["stream"][:256]), g["p"][:256 * 8])
    _decode_schedule(cm, port, g, prefix, 256, 768, "full_text: bulk [0,256), coded/decoded [256,1024)")


@pytest.mark.timeout(1200)
def test_decode_after_pretraining(cm, port, dict_path, pre):
    g = golden("full_wrt")
    _decode_schedule(cm, port, g, lambda P: _pretrain(P, pre, "full_wrt"), 0, 512,
                     "full_wrt: pretrain_bytes(dictionary), coded/decoded [0,512)", dictionary=dict_path)


@pytest.mark.timeout(900)
def test_decode_then_lock_step(cm):
    """Lock-step after the decoder: the first Predict() is ordered behind the decoder's last graph and takes the codes its
    FXCM and PAQ8 bit kernels left in d_ext_bit; a bulk call follows."""
    g = golden("full_text")
    s, p = g["stream"], g["p"]
    n, m = 256, 288
    sched = "full_text: coded/decoded [0,%d), lock-step [%d,%d), bulk [%d,1024)" % (n, n, m, m)
    enc = cm.Predictor(g["vocab"])
    try:
        enc.coder_begin(2 * n + 64)
        expect(sched + ", encoder bulk", enc.code_bytes(s[:n]), p[:n * 8])
        archive = enc.coder_finish()
    finally:
        enc.close()
    dec = cm.Predictor(g["vocab"])
    try:
        out = dec.decode_bytes(archive, n)
        assert out.tobytes() == s[:n].tobytes(), "%s, decoder: %s" % (sched, first_bad_byte(out, s[:n]))
        lock_step(dec, g, n * 8, m * 8, sched)
        expect(sched + ", bulk", dec.code_bytes(s[m:1024]), p[m * 8:1024 * 8], m * 8)
    finally:
        dec.close()


@pytest.mark.timeout(900)
def test_bulk_split_schedule(cm):
    """Bulk calls of 1, 16, 17, 129, 257, 4097 and 1627 bytes: n <= 16, the halving tail, the geometric head and full
    sub-chunks of RunPipelined, RunPieces' 2048-byte pieces and code_bytes' 4096-byte host staging; together = one call."""
    g = golden("full_text")
    sizes = [1, 16, 17, 129, 257, 4097, 1627]
    assert sum(sizes) == g["stream"].size
    P = cm.Predictor(g["vocab"])
    try:
        off = 0
        for n in sizes:
            expect("full_text: bulk calls of %s, the call [%d,%d)" % (sizes, off, off + n),
                   P.code_bytes(g["stream"][off:off + n]), g["p"][off * 8:(off + n) * 8], off * 8)
            off += n
    finally:
        P.close()


# ------------------------------------------------------------------------------------------------ batches
N_DEV, N_HOST = 2560, 1100          # one code_batch_device call (two 2048-byte pieces), then one code_batch (crosses 1024)


def _three_stream_batch(cm, dict_path, port, label):
    """Streams A (full_text from byte 0), B (full_bin, first advanced alone by 512 bytes: a different bits_done, so its own
    learning-rate decay) and C (full_wrt with dictionary, pretraining and the device coder) in one launch set."""
    import torch
    from cmix_b200.capi import code_batch, code_batch_device
    gs = [golden("full_text"), golden("full_bin"), golden("full_wrt")]
    names = ["A full_text", "B full_bin", "C full_wrt"]
    start = [0, 512, 0]
    preds, footprint = [], []
    try:
        for g, name in zip(gs, names):
            free0 = torch.cuda.mem_get_info()[0]
            preds.append(cm.Predictor(g["vocab"], dictionary_path=dict_path if name.startswith("C") else None))
            footprint.append((free0 - torch.cuda.mem_get_info()[0]) / 1e9)
            print("%s: %s predictor holds %.2f GB of HBM (PPMD arena %s MB)" % (label, name, footprint[-1], os.environ["CMIXB200_PPMD_MB"]))
        _pretrain(preds[2], pretrain_buffer(dict_path), label + ": C")
        expect(label + ": B alone, bulk [0,512)", preds[1].code_bytes(gs[1]["stream"][:512]), gs[1]["p"][:512 * 8])
        preds[2].coder_begin(N_DEV + N_HOST + 64)
        dev = torch.device("cuda", 0)
        d_bytes = [torch.from_numpy(g["stream"][o:o + N_DEV].copy()).to(dev) for g, o in zip(gs, start)]
        d_out = [torch.empty(N_DEV * 8, dtype=torch.float32, device=dev) for _ in gs]
        code_batch_device(preds, d_bytes, N_DEV, None, None, d_out)
        torch.cuda.synchronize()
        for g, o, out, name in zip(gs, start, d_out, names):
            expect("%s: code_batch_device of %d bytes, stream %s at byte %d" % (label, N_DEV, name, o),
                   out.cpu().numpy(), g["p"][o * 8:(o + N_DEV) * 8], o * 8)
        outs = [np.empty(N_HOST * 8, dtype=np.float32) for _ in gs]
        code_batch(preds, [g["stream"][o + N_DEV:o + N_DEV + N_HOST] for g, o in zip(gs, start)], N_HOST, None, None, outs)
        for g, o, out, name in zip(gs, start, outs, names):
            lo = o + N_DEV
            expect("%s: code_batch of %d bytes, stream %s at byte %d" % (label, N_HOST, name, lo),
                   out, g["p"][lo * 8:(lo + N_HOST) * 8], lo * 8)
        archive = preds[2].coder_finish()
    finally:
        for P in preds:
            P.close()
    n = N_DEV + N_HOST
    want = host_archive(port, gs[2]["p"][:n * 8], np.unpackbits(gs[2]["stream"][:n]))
    assert archive == want, "%s: C's device archive differs from the host encoder's: %s" % (label, first_bad_byte(archive, want))
    return footprint


@pytest.mark.timeout(900)
def test_resident_batch_of_three_streams(cm, dict_path, port):
    _three_stream_batch(cm, dict_path, port, "one launch group")


@pytest.mark.timeout(1200)
def test_resident_batch_in_two_launch_groups(cm, dict_path, port):
    """The same batch with CMIXB200_GROUP=2 (C runs on its own lead's CUDA streams) and CMIXB200_SUBCHUNK=48. Both are read
    once per process, so the batch runs in a child interpreter once this process holds no predictor."""
    env = {"CMIXB200_GROUP": "2", "CMIXB200_SUBCHUNK": "48"}
    results = run_child(None, "test_call_schedules", "_child", [dict_path], env=env, timeout=1100)
    assert len(results) == 1 and not results[0]["fail"], "two launch groups, sub-chunk 48: %s" % results


def _child(dict_path):
    import cmix_b200
    from oracle_io import load_port
    cmix_b200.load_library()
    child_jobs(["batch"], lambda j, job: _three_stream_batch(cmix_b200, dict_path, load_port(), "two launch groups, sub-chunk 48"))
