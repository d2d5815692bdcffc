"""What the test modules share: fixture loading, the GPU call schedules, the host-tool and variant-library builds, and
the child interpreters that run a variant library. Not collected (no test_ prefix); modules import from it by name."""
import ctypes
import json
import os
import re
import subprocess
import sys
import time
import zlib
from collections import namedtuple
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from conftest import ROOT

CSRC = os.path.join(ROOT, "cmix_b200", "csrc")
DBG_PPMD_ROWS, DBG_EXT_GEN = 8, 10       # debug_fetch: the last bulk call's PPMD rows [bytes][256], generated codes [bits][2022]
MAX_PIECE = 2048                         # a bulk call's debug fetches cover its last 2048-byte piece only


def golden(name):
    """tests/golden/<name>.npz as a dict of arrays, plus "name"."""
    z = np.load(os.path.join(ROOT, "tests", "golden", name + ".npz"))
    return dict({k: z[k] for k in z.files}, name=name)


# ------------------------------------------------------------------------------------------------ fixtures
@pytest.fixture(scope="module")
def cm():
    import cmix_b200
    cmix_b200.load_library()
    return cmix_b200


@pytest.fixture(autouse=True)
def ppmd_arena(monkeypatch):
    """A 512 MB PPMD arena, so that three full predictors fit in 80 GB (autouse in the modules that import it)."""
    if "CMIXB200_PPMD_MB" not in os.environ:
        monkeypatch.setenv("CMIXB200_PPMD_MB", "512")


@pytest.fixture(scope="session")
def jitter_lib(tmp_path_factory):
    """The library compiled with -DCMIXB200_JITTER (cmix_b200/csrc/jitter.cuh), once per session.

    Each module that imports this fixture holds its own copy of it, so it builds into one fixed directory of the session:
    the second module's call finds the library up to date there."""
    from cmix_b200.capi import build_library
    out = tmp_path_factory.getbasetemp() / "jitter"
    out.mkdir(exist_ok=True)
    return build_library(defines=["-DCMIXB200_JITTER"], out_dir=str(out))


@pytest.fixture(scope="module")
def ppmd_host(tmp_path_factory):
    """tools/ppmd_host.cpp as a shared library: run(stream, vocab, arena_mb=64) -> (return code, [bytes][256] distributions)."""
    lib = ctypes.CDLL(build_host_tool("ppmd_host", str(tmp_path_factory.mktemp("ppmd")), ["-shared", "-fPIC"]))
    lib.ppmd_host_run.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_uint]
    lib.ppmd_host_run.restype = ctypes.c_int

    def run(stream, vocab, arena_mb=64):
        stream = np.ascontiguousarray(stream, dtype=np.uint8)
        vocab = np.ascontiguousarray(vocab, dtype=np.uint8)
        out = np.zeros((stream.size, 256), dtype=np.float32)
        rc = lib.ppmd_host_run(stream.ctypes.data, stream.size, vocab.ctypes.data, out.ctypes.data, arena_mb)
        return rc, out
    return run


# ------------------------------------------------------------------------------------------------ checks
def expect(schedule, got, want, first_bit=0):
    """got == want on the float bits; on failure name the schedule, the first differing bit and both values."""
    got = np.ascontiguousarray(got, dtype=np.float32)
    want = np.ascontiguousarray(want, dtype=np.float32)
    assert got.shape == want.shape, "%s: %s probabilities, expected %s" % (schedule, got.shape, want.shape)
    d = np.nonzero(got.view(np.uint32) != want.view(np.uint32))[0]
    if d.size:
        k = int(d[0])
        pytest.fail("%s: first differing bit %d (byte %d; got %.9g, reference %.9g; %d of %d bits differ)"
                    % (schedule, first_bit + k, (first_bit + k) // 8, got[k], want[k], d.size, got.size), pytrace=False)


def lock_step(P, g, lo, hi, schedule):
    """Predict()/Perceive(bit) over bits [lo, hi) of the fixture's stream, each Predict() checked as it comes."""
    bits = np.unpackbits(g["stream"])
    for t in range(lo, hi):
        expect(schedule + ", lock-step", np.float32([P.Predict()]), g["p"][t:t + 1], t)
        P.Perceive(int(bits[t]))


def host_archive(port, p, bits):
    """Encoder::Encode/Flush on the host (oracle port) over the reference's probabilities."""
    e = port.op_enc_create()
    for pr, b in zip(p, bits):
        port.op_enc_encode(e, float(pr), int(b))
    buf = np.zeros(bits.size // 4 + 64, dtype=np.uint8)
    n = port.op_enc_finish(e, buf.ctypes.data, buf.size)
    port.op_enc_destroy(e)
    return buf[:n].tobytes()


def first_bad_byte(got, want):
    got, want = np.frombuffer(bytes(got), dtype=np.uint8), np.frombuffer(bytes(want), dtype=np.uint8)
    if got.size != want.size:
        return "length %d, expected %d" % (got.size, want.size)
    d = np.nonzero(got != want)[0]
    return "first differing byte %d (%d vs %d)" % (d[0], got[d[0]], want[d[0]]) if d.size else "equal"


def pretrain_buffer(dict_path):
    """What `cmix -c english.dic` feeds Pretrain(): a 5-byte header, then the dictionary with newlines as spaces."""
    d = open(dict_path, "rb").read()
    return bytes([0, (len(d) >> 24) & 255, (len(d) >> 16) & 255, (len(d) >> 8) & 255, len(d) & 255]) + d.replace(b"\n", b" ")


# ------------------------------------------------------------------------------------------------ piece plans
def even(lo, hi, size=MAX_PIECE):
    """Pieces of [lo, hi) of `size` bytes, the last one shorter."""
    return [(a, min(a + size, hi)) for a in range(lo, hi, size)]


def awkward(lo, hi):
    """Pieces of [lo, hi): 1, 129, 7, 1000, 333 bytes, then the rest."""
    out = []
    for n in (1, 129, 7, 1000, 333):
        if lo < hi:
            out.append((lo, min(lo + n, hi)))
            lo = out[-1][1]
    if lo < hi:
        out.append((lo, hi))
    return out


def stress_pieces(n):
    """Pieces of [0, n): 1, 129 and 1000 bytes, then pieces of at most 2000."""
    sizes = [1, 129, 1000]
    while sum(sizes) < n:
        sizes.append(min(2000, n - sum(sizes)))
    ends = np.cumsum(sizes).tolist()
    return list(zip([0] + ends[:-1], ends))


# the bytes each reach_* stream is built to reach: lock-step runs over [marker + lo, marker + hi)
TARGETS = {"reach_english": (b"+\r\n", -8, 24), "reach_europe": (b"travaux", -4, 20), "reach_xml": (b"<![CDATA[", -4, 52),
           "reach_x86": (b"\x0f\x3a", -4, 28), "reach_dbase": (b"visual foxpro table\n", 18, 70),
           "reach_bmp": (b"\x28\x00\x00\x00\x10\x00\x00\x00", 24, 48), "reach_fxwiki": (b"PPQ", -4, 36)}


def target(name, s):
    marker, lo, hi = TARGETS[name]
    at = s.tobytes().find(marker)
    assert at >= 0, "%s: marker %r not in the stream" % (name, marker)
    return at + lo, min(at + hi, s.size)


# ------------------------------------------------------------------------------------------------ the mixers' overflow row
SLOT_LIMIT = 10000                    # state.h / mixer.cpp:17
N_MIXERS, SEL_PITCH, AUX = 47, 48, 12  # selector 12 (auxiliary_context_) is computed inside the mix kernel
LAYER1 = range(26, 46)
DBG_SEL = 2                            # CMIXB200_DBG_SEL: [bits of the last bulk call][SEL_PITCH] u32


def onsets(ctx):
    """{mixer: byte of the bit that brings its (SLOT_LIMIT + 1)-th distinct context} over ctx [bits][mixers]."""
    out = {}
    for m in range(N_MIXERS):
        if m == AUX:
            continue
        _, first = np.unique(ctx[:, m], return_index=True)
        if first.size > SLOT_LIMIT:
            out[m] = int(np.sort(first)[SLOT_LIMIT]) // 8
    return out


# ------------------------------------------------------------------------------------------------ GPU schedules
def code_in_pieces(P, g, pieces, after=None):
    """Bulk calls over the (a, b) byte pieces, in order from byte 0, then every way the run differs from the fixture's
    prefix it covers, each with its first bit, byte or block: Predict(), the first 64 code rows, the FXCM and PAQ8 code
    CRCs per 4096 bits and, where the fixture has them, the PPMD distribution CRCs per byte. after(P, a, b) runs after each
    call. Returns {"p", "crc_fx", "crc_p8"}."""
    s = g["stream"]
    ps, exts, ppmd_crc = [], [], []
    for a, b in pieces:
        assert b - a <= MAX_PIECE, "%s: piece [%d,%d) is longer than the debug fetch covers" % (g["name"], a, b)
        ps.append(P.code_bytes(s[a:b]))
        exts.append(P.debug_fetch(DBG_EXT_GEN, ((b - a) * 8, 2022), np.uint16))
        if "ppmd_crc" in g:
            rows = P.debug_fetch(DBG_PPMD_ROWS, (b - a, 256), np.float32)
            ppmd_crc += [zlib.crc32(rows[t].tobytes()) for t in range(b - a)]
        if after is not None:
            after(P, a, b)
    p, ext = np.concatenate(ps), np.concatenate(exts)
    nb = p.size

    def crc(lo, hi):
        return np.array([zlib.crc32(np.ascontiguousarray(ext[t:t + 4096, lo:hi]).tobytes()) for t in range(0, nb, 4096)],
                        dtype=np.uint32)
    got = {"p": p, "crc_fx": crc(0, 431), "crc_p8": crc(431, 2022)}
    out = []
    d = np.nonzero(p.view(np.uint32) != g["p"][:nb].view(np.uint32))[0]
    if d.size:
        k = int(d[0])
        out.append("Predict(): first differing bit %d (byte %d, block %d; %.9g vs %.9g; %d bits differ)"
                   % (k, k // 8, k // 4096, p[k], g["p"][k], d.size))
    bad = np.argwhere(ext[:64] != g["first_codes"])
    if bad.size:
        out.append("codes of the first 64 bits: first differing (bit, slot) %s" % (bad[0].tolist(),))
    for what, key in (("FXCM", "crc_fx"), ("PAQ8", "crc_p8")):
        b = np.nonzero(got[key] != g[key][:(nb + 4095) // 4096])[0]
        if b.size:
            out.append("%s codes: first differing block %d (bits %d..%d)" % (what, b[0], b[0] * 4096, b[0] * 4096 + 4095))
    if "ppmd_crc" in g:
        b = np.nonzero(np.array(ppmd_crc, dtype=np.uint32) != g["ppmd_crc"][:nb // 8])[0]
        if b.size:
            out.append("PPMD distribution: first differing after byte %d" % b[0])
    if out:
        pytest.fail("%s: " % g["name"] + "; ".join(out), pytrace=False)
    return got


def awkward_lock_step(cm, name, span=None, plan=awkward):
    """Bulk calls in `plan`'s pieces up to span = (lo, hi) (by default the bytes the stream targets), lock-step
    Predict()/Perceive() across it, then bulk calls in `plan`'s pieces to the end."""
    g = golden(name)
    s, p = g["stream"], g["p"]
    lo, hi = span or target(name, s)
    P = cm.Predictor(g["vocab"])
    try:
        for a, b in plan(0, lo):
            expect("%s: bulk [%d,%d)" % (name, a, b), P.code_bytes(s[a:b]), p[a * 8:b * 8], a * 8)
        lock_step(P, g, lo * 8, hi * 8, "%s: lock-step [%d,%d)" % (name, lo, hi))
        for a, b in plan(hi, s.size):
            expect("%s: bulk [%d,%d) after lock-step" % (name, a, b), P.code_bytes(s[a:b]), p[a * 8:b * 8], a * 8)
    finally:
        P.close()


def batch(cm, names, n=None):
    """The streams side by side in one code_batch_device call, over the first n bytes (at most the shortest stream)."""
    import torch
    from cmix_b200.capi import code_batch_device
    gs = [golden(x) for x in names]
    n = min([g["stream"].size for g in gs] + ([n] if n else []))
    preds = []
    try:
        for g in gs:
            preds.append(cm.Predictor(g["vocab"]))
        dev = torch.device("cuda", 0)
        d_bytes = [torch.from_numpy(g["stream"][:n].copy()).to(dev) for g in gs]
        d_out = [torch.empty(n * 8, dtype=torch.float32, device=dev) for _ in gs]
        code_batch_device(preds, d_bytes, n, None, None, d_out)
        torch.cuda.synchronize()
        for g, out, x in zip(gs, d_out, names):
            expect("batch of %s, %d bytes each: %s" % (list(names), n, x), out.cpu().numpy(), g["p"][:n * 8])
    finally:
        for P in preds:
            P.close()


def round_trip(cm, port, name, n_decode=None):
    """Device encoder -> archive equal to the host encoder's over the reference's probabilities (port=None: not compared)
    -> device decoder over the first n_decode bytes."""
    g = golden(name)
    s, p = g["stream"], g["p"]
    enc = cm.Predictor(g["vocab"])
    try:
        enc.coder_begin(2 * s.size + 64)
        expect("%s: encoder" % name, enc.code_bytes(s), p)
        archive = enc.coder_finish()
    finally:
        enc.close()
    if port is not None:
        want = host_archive(port, p, np.unpackbits(s))
        assert archive == want, "%s: device archive differs from the host encoder's: %s" % (name, first_bad_byte(archive, want))
    n = n_decode or s.size
    dec = cm.Predictor(g["vocab"])
    try:
        out = dec.decode_bytes(archive, n)
    finally:
        dec.close()
    assert out.tobytes() == s[:n].tobytes(), "%s, decoder: %s" % (name, first_bad_byte(out, s[:n]))


def wav_until_unsupported(cm, name):
    """Calls over the text and header, over the first sample, and over the samples: each returns the reference's
    probabilities, or fails with CMIXB200_ERR_UNSUPPORTED; the call over the text and header never fails."""
    from gen_wav import ENTRY
    g = golden(name)
    s = g["stream"]
    P = cm.Predictor(g["vocab"])
    try:
        for lo, hi in ((0, ENTRY - 1), (ENTRY - 1, ENTRY + 1), (ENTRY + 1, s.size)):
            try:
                got = P.code_bytes(s[lo:hi])
            except RuntimeError as e:
                assert lo > 0 and "image / audio / JPEG" in str(e), "%s: bytes [%d,%d): %s" % (name, lo, hi, e)
                break
            expect("%s: bytes [%d,%d)" % (name, lo, hi), got, g["p"][lo * 8:hi * 8], lo * 8)
    finally:
        P.close()


# ------------------------------------------------------------------------------------------------ host tools
HostRun = namedtuple("HostRun", "rc out crc census log")


def build_host_tool(tool, out_dir, flags=()):
    """tools/<tool>.cpp built with g++ -O2, its own flags (coverage_report.HOST_FLAGS) and `flags`; returns its path."""
    from coverage_report import gxx
    exe = os.path.join(out_dir, tool)
    subprocess.run(gxx(tool, exe, ["-O2", *flags]), check=True)
    return exe


def run_host_tool(exe, out_dir, label, stream, lstmfx=None, log=False, dictionary=None):
    """One run of paq8_check or fxcm_check: its return code, output, CRCs per 4096 bits, census JSON line (built with
    -DCENSUS) and, with log=True, its per-bit census log (CENSUS_LOG; PAQ8's as [bits][3] words)."""
    prefix = os.path.join(out_dir, label)
    stream.tofile(prefix + ".stream")
    if lstmfx is not None:
        lstmfx.tofile(prefix + ".lstmfx.u32")
    env = dict(os.environ, CENSUS_LOG=prefix + ".log") if log else None
    r = subprocess.run([exe, prefix, dictionary or "-", str(stream.size), prefix + ".crc"], capture_output=True, text=True,
                       env=env)
    census = [json.loads(line[len("census "):]) for line in r.stdout.splitlines() if line.startswith("census ")]
    crc = np.fromfile(prefix + ".crc", dtype=np.uint32) if os.path.exists(prefix + ".crc") else None
    words = np.fromfile(prefix + ".log", dtype=np.uint32) if log and os.path.exists(prefix + ".log") else None
    if words is not None and os.path.basename(exe) == "paq8_check":
        words = words.reshape(-1, 3)
    return HostRun(r.returncode, r.stdout + r.stderr, crc, census[0] if census else None, words)


def run_host_tools(runs, log=False):
    """{key: run_host_tool(*args, log=log)} over {key: args}, in parallel."""
    with ThreadPoolExecutor(os.cpu_count() or 4) as ex:
        futs = {k: ex.submit(run_host_tool, *args, log=log) for k, args in runs.items()}
        return {k: f.result() for k, f in futs.items()}


def check_host(run, want, what):
    """A host run exits 0 and its CRCs equal the reference's, every block."""
    assert run.rc != 3, "%s: the stream trips PAQ8's image / audio / JPEG gate:\n%s" % (what, run.out[-2000:])
    assert run.rc == 0, "%s:\n%s" % (what, run.out[-2000:])
    bad = np.nonzero(run.crc != want[:run.crc.size])[0]
    assert run.crc.size == want.size and bad.size == 0, "%s: %d CRC blocks, expected %d; first differing 4096-bit block %s" % (
        what, run.crc.size, want.size, bad[:1])


# ------------------------------------------------------------------------------------------------ child interpreters
def run_child(lib, module, entry, args, env=None, timeout=1500):
    """module.entry(*args) in a child interpreter, with CMIXB200_LIB=lib when lib is given (a variant library, or settings
    read once per process); fails if the child does. Returns the JSON lines it printed."""
    import gc
    import torch
    gc.collect()
    torch.cuda.empty_cache()
    e = dict(os.environ, **(env or {}))
    if lib:
        e["CMIXB200_LIB"] = lib
    e.setdefault("CMIXB200_PPMD_MB", "512")
    code = "import sys; sys.path[:0] = sys.argv[1:4]; import %s as m; m.%s(*sys.argv[4:])" % (module, entry)
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [
        "-c", code, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools"), ROOT, *args]
    r = subprocess.run(cmd, env=e, cwd=ROOT, capture_output=True, text=True, timeout=timeout)
    assert r.returncode == 0, "%s.%s: child failed:\n%s\n%s" % (module, entry, r.stdout[-3000:], r.stderr[-3000:])
    lines = r.stdout.splitlines()
    own = [line for line in lines if not line.startswith("{")]      # the child's own diagnostics
    if own:
        print("\n".join(own))
    return [json.loads(line) for line in lines if line.startswith("{")]


def child_jobs(jobs, run):
    """The child side of run_child: run(j, job) for each job in turn, one JSON line per job ({"job", "s", "fail"})."""
    for j, job in enumerate(jobs):
        t0 = time.perf_counter()
        try:
            run(j, job)
            msg = None
        except BaseException as e:      # pytest.fail raises an exception outside pytest's Exception tree
            msg = "%s: %s" % (type(e).__name__, e)
        print(json.dumps({"job": job, "s": round(time.perf_counter() - t0, 2), "fail": msg}), flush=True)
        if msg and ("CUDA" in msg or "cuda" in msg):
            break                        # the context may be gone: report, do not go on


def sass_by_function(path):
    """{function name: its SASS instructions} of a cubin or library (cuobjdump -sass; addresses and encodings dropped)."""
    text = subprocess.run(["cuobjdump", "-sass", path], check=True, capture_output=True, text=True).stdout
    funcs, name = {}, None
    for line in text.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            name = m.group(1)
            funcs.setdefault(name, [])
        elif name is not None:
            ins = re.sub(r"/\*.*?\*/", "", line).strip()
            if ins:
                funcs[name].append(ins)
    return {k: "\n".join(v) for k, v in funcs.items()}


# ------------------------------------------------------------------------------------------------ the jitter build
def _jitter_text():
    return open(os.path.join(CSRC, "jitter.cuh")).read()


def _enum(first):
    """Names of the enum of jitter.cuh that starts with `first`, in order (their values)."""
    body = re.search(r"enum \{\s*(%s\b.*?)\};" % first, _jitter_text(), re.S).group(1)
    body = re.sub(r"//[^\n]*", "", body)
    return [n.strip() for n in body.split(",") if n.strip() and "=" not in n]


def jitter_files():
    """JIT_FILE_LIST of jitter.cuh: a site's file index."""
    return re.findall(r'"([\w.]+)"', re.search(r"#define JIT_FILE_LIST(.*?)\n(?!\s)", _jitter_text(), re.S).group(1))


MODES = {n: i for i, n in enumerate(_enum("JIT_OFF"))}
GROUPS = {n: i for i, n in enumerate(_enum("JG_NONE"))}
JK = {n: i for i, n in enumerate(_enum("JK_FILL"))}
MAX_LINE = 2048


def jitter_child(jobs_json):
    """Run in a child interpreter with CMIXB200_LIB = the jitter build: each job is [config, schedule, args]. Prints one JSON
    line per job and, last, {"fired": the sites that slept}."""
    import cmix_b200
    lib = cmix_b200.load_library()
    lib.cmixb200_jitter_config.argtypes = [ctypes.c_int, ctypes.c_uint, ctypes.c_int, ctypes.c_int, ctypes.c_int]
    lib.cmixb200_jitter_counts.argtypes = [ctypes.c_void_p, ctypes.c_size_t]
    port = []

    def bulk(name, n=None, piece=MAX_PIECE):
        """Bulk calls of `piece` bytes over the first n bytes."""
        g = golden(name)
        P = cmix_b200.Predictor(g["vocab"])
        try:
            code_in_pieces(P, g, even(0, g["stream"][:n].size, piece))
        finally:
            P.close()

    def run(j, job):
        cfg, sched, args = job
        mode, a = cfg[0], cfg[2]
        a = GROUPS[a] if mode in ("starve", "hurry") else JK[a] if mode == "entry" else a
        if lib.cmixb200_jitter_config(MODES["JIT_" + mode.upper()], cfg[1], a, cfg[3], cfg[4]) != 0:
            raise RuntimeError("jitter config: " + lib.cmixb200_last_error().decode())
        if sched == "bulk":
            bulk(*args)
        elif sched == "wrt":            # full_wrt's first 2048 bytes after the dictionary: all but its last 64 bytes in bulk,
            pre = pretrain_buffer(args[0])  # those bit by bit
            g = golden("full_wrt")
            P = cmix_b200.Predictor(g["vocab"], dictionary_path=args[0])
            try:
                P.pretrain_bytes(pre[:-64])
                for byte in pre[-64:]:
                    for k in range(7, -1, -1):
                        P.Pretrain((byte >> k) & 1)
                code_in_pieces(P, g, even(0, 2048))
            finally:
                P.close()
        elif sched == "wav":
            wav_until_unsupported(cmix_b200, *args)
        elif sched == "awkward":
            awkward_lock_step(cmix_b200, *args)
        elif sched == "batch":
            batch(cmix_b200, *args)
        elif sched == "round_trip":
            if not port:
                from oracle_io import load_port
                port.append(load_port())
            round_trip(cmix_b200, port[0], *args)
        else:
            raise ValueError(sched)

    child_jobs(json.loads(jobs_json), run)
    lib.cmixb200_jitter_config(MODES["JIT_OFF"], 0, 0, 0, 0)
    n = len(jitter_files()) * MAX_LINE
    counts = np.zeros(n, dtype=np.uint32)
    if lib.cmixb200_jitter_counts(counts.ctypes.data, n) == 0:
        print(json.dumps({"fired": {int(i): int(counts[i]) for i in np.nonzero(counts)[0]}}), flush=True)


def _describe(cfg):
    mode, seed, a, b, c = cfg
    if mode == "random":
        return "mode random, seed %#x, density %d/65536" % (seed, a)
    if mode == "entry":
        return "mode entry, kernel %s, %d us every %d launches" % (a, b, c)
    return "mode %s, group %s" % (mode, a)


def run_jitter(jitter_lib, label, jobs, env=None, timeout=1500):
    """The jobs in a child interpreter on the jitter build; fails with every failing job's configuration and first
    difference. Returns {site: sleeps} over the jobs."""
    t0 = time.perf_counter()
    lines = run_child(jitter_lib, "harness", "jitter_child", [json.dumps(jobs)], env=env, timeout=timeout)
    results = [x for x in lines if "job" in x]
    fired = {int(k): v for x in lines if "fired" in x for k, v in x["fired"].items()}
    fails = []
    for x in results:
        cfg, sched, args = x["job"]
        what = args if sched != "wrt" else "full_wrt"
        print("%-40s %-10s %-45s %6.1f s%s" % (cfg, sched, what[:3] if sched != "wrt" else what, x["s"], "  FAIL" if x["fail"] else ""))
        if x["fail"]:
            fails.append("%s, schedule %s %s: %s" % (_describe(cfg), sched, what, x["fail"]))
    print("%s: %d runs in %.0f s" % (label, len(results), time.perf_counter() - t0))
    assert not fails, "%s: %d of %d runs differ from the reference:\n%s" % (label, len(fails), len(results), "\n".join(fails))
    assert len(results) == len(jobs), "%s: %d of %d runs reported" % (label, len(results), len(jobs))
    return fired
