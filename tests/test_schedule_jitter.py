"""Every kernel's synchronisation under perturbed warp, CTA and stream schedules.

A missing barrier, mbarrier wait or cross-stream event shows only when some warp, CTA or kernel runs late, and then as a
wrong bit in an archive, not as a crash. cmix_b200/csrc/jitter.cuh puts a hook at every synchronisation site (after each
barrier or wait, before each arrive-only barrier or remote arrive, at every flag spin's exit, at every kernel's entry);
built with -DCMIXB200_JITTER the hook sleeps there on a deterministic schedule: random(seed, density), starve(group) (one
warp group sleeps at each of its sites), hurry(group) (everyone else does), entry(kernel, us, every_n) (a kernel's
launches start late). Whatever the schedule, every probability, every FXCM / PAQ8 code and every PPMD distribution must
equal the reference fixture's (tolerance 0).

CPU (-m "not gpu"): the jitter build compiles for sm_90a; every kernel of the jitter build sleeps and no kernel of the
product library does; every barrier primitive in cmix_b200/csrc is reached through a helper that carries a site.
GPU (-m gpu): the jitter library runs in child interpreters (CMIXB200_LIB), each over a list of (configuration, schedule,
fixture) runs; the last test checks that every site slept at least once over the module, or is in NEVER_FIRES.
The pretraining of full_wrt (412 001 bytes) runs under one random seed; CMIXB200_SLOW=1 runs it under all three."""
import ctypes
import json
import os
import re
import subprocess
import sys
import time
import zlib

import numpy as np
import pytest

from conftest import ROOT

CSRC = os.path.join(ROOT, "cmix_b200", "csrc")
UNITS = ["engine.cu", "fxcm_dev.cu", "paq8_dev.cu"]
SLOW = os.environ.get("CMIXB200_SLOW") == "1"
SEEDS = [0x5EED0001, 0x5EED0002, 0x5EED0003]
DENSITY = 16384                                   # random mode: a quarter of the visits sleep
KERNELS = ["fill_f32", "fill_u32", "fill_sse_rows", "fill_u16", "encode_kernel", "encode_flush_kernel", "decode_begin_kernel",
           "decode_step_kernel", "fxcm_kernel", "fxcm_bit_kernel", "lstm_kernel", "lock_predict_inputs_kernel",
           "lstm_byte_kernel", "mix_kernel_v3", "mix_predict_rows_kernel", "mix_predict_final_kernel", "mix_perceive_kernel",
           "paq8_kernel", "paq8_bit_kernel", "ppmd_init_kernel", "ppmd_kernel", "ppmd_byte_kernel", "small_kernel",
           "small_predict_kernel", "small_perceive_kernel"]
REACH = ["english", "europe", "xml", "x86", "dbase", "bmp", "fxwiki"]
WAV = "wav_pcm16_mono"

# Sites no run of this module sleeps at, each with the reason: (file, stripped text of the line, reason).
NEVER_FIRES = []


def _jitter_text():
    return open(os.path.join(CSRC, "jitter.cuh")).read()


def _enum(first):
    """Names of the enum of jitter.cuh that starts with `first`, in order (their values)."""
    body = re.search(r"enum \{\s*(%s\b.*?)\};" % first, _jitter_text(), re.S).group(1)
    body = re.sub(r"//[^\n]*", "", body)
    return [n.strip() for n in body.split(",") if n.strip() and "=" not in n]


def _files():
    return re.findall(r'"([\w.]+)"', re.search(r"#define JIT_FILE_LIST(.*?)\n(?!\s)", _jitter_text(), re.S).group(1))


MODES = {n: i for i, n in enumerate(_enum("JIT_OFF"))}
GROUPS = {n: i for i, n in enumerate(_enum("JG_NONE"))}
JK = {n: i for i, n in enumerate(_enum("JK_FILL"))}
MAX_LINE = 2048


# ------------------------------------------------------------------------------------------------ the jitter build
@pytest.fixture(scope="module")
def jitter_lib(tmp_path_factory):
    """The library compiled with -DCMIXB200_JITTER into this module's tmp dir (as tools/prof_build.py builds its variant)."""
    from cmix_b200.capi import NVCC_COMPILE, NVCC_LINK
    out = tmp_path_factory.mktemp("jitter")
    objs, jobs = [], []
    for u in UNITS:
        obj = str(out / (u[:-3] + ".o"))
        objs.append(obj)
        jobs.append(subprocess.Popen(["nvcc"] + NVCC_COMPILE + ["-DCMIXB200_JITTER", "-c", os.path.join(CSRC, u), "-o", obj]))
    assert all(j.wait() == 0 for j in jobs), "nvcc failed on the jitter build"
    lib = str(out / "libcmixb200_jitter.so")
    subprocess.run(["nvcc"] + NVCC_LINK + objs + ["-o", lib], check=True)
    return lib


def _sass_by_kernel(lib):
    """{kernel name: its SASS} from cuobjdump -sass."""
    text = subprocess.run(["cuobjdump", "-sass", lib], check=True, capture_output=True, text=True).stdout
    out = {}
    for part in re.split(r"\n\s*Function : ", text)[1:]:
        mangled, _, body = part.partition("\n")
        name = next((k for k in KERNELS if re.search(r"\d%s[A-Z]" % k, mangled)), mangled.strip())
        out[name] = out.get(name, "") + body
    return out


def test_jitter_build_sleeps_in_every_kernel_and_the_product_nowhere(jitter_lib):
    import cmix_b200
    jit = _sass_by_kernel(jitter_lib)
    missing = [k for k in KERNELS if k not in jit]
    assert not missing, "kernels not in the jitter build: %s" % missing
    quiet = [k for k in KERNELS if "NANOSLEEP" not in jit[k]]
    assert not quiet, "kernels of the jitter build without a sleep: %s" % quiet
    lib = ctypes.CDLL(jitter_lib)
    assert hasattr(lib, "cmixb200_jitter_config") and hasattr(lib, "cmixb200_jitter_counts")
    prod = _sass_by_kernel(cmix_b200.build_library())
    assert sorted(prod) == sorted(jit), "the two builds hold different kernels"
    sleeping = [k for k, s in prod.items() if "NANOSLEEP" in s]
    assert not sleeping, "product kernels that sleep: %s" % sleeping
    assert not hasattr(ctypes.CDLL(cmix_b200.build_library()), "cmixb200_jitter_config")


# ------------------------------------------------------------------------------------------------ the lint
PRIMITIVES = [(re.compile(r"__syncthreads\s*\("), "__syncthreads"), (re.compile(r"\.sync\s*\(\s*\)"), "cluster / group sync"),
              (re.compile(r"\bbar(rier)?\.(sync|arrive|red)"), "named barrier"),
              (re.compile(r"mbarrier\.(try_wait|test_wait|arrive(?!\.expect_tx))"), "mbarrier wait / arrive")]
SPIN = re.compile(r"\bwhile\s*\(.*\)\s*\{\s*\}|\bdo\s*\{.*\}\s*while\s*\((?!0\s*\))")   # do {} while (0) is a macro body


def _source_files():
    return sorted(f for f in os.listdir(CSRC) if f.endswith((".cu", ".cuh", ".h")) and f != "jitter.cuh")


def _sites():
    """(file, line) of every site: each use of JIT_HERE, JIT_SYNCTHREADS or jit_entry."""
    out = []
    for f in _source_files():
        for i, line in enumerate(open(os.path.join(CSRC, f)).read().split("\n"), 1):
            if re.search(r"\bJIT_HERE\b|JIT_SYNCTHREADS\(\)|\bjit_entry\(", line):
                out.append((f, i))
    return out


def test_every_barrier_primitive_carries_a_site():
    """A raw barrier, mbarrier wait, remote arrive or flag spin outside a site-carrying helper, a helper call without
    JIT_HERE, or a kernel without jit_entry fails here with its line."""
    bad = []
    files = _files()
    for f in _source_files():
        lines = open(os.path.join(CSRC, f)).read().split("\n")
        helper = None            # (definition line, whether it takes `int site` and calls jit_point(site)) of the function we are in
        helpers = set()
        for i, line in enumerate(lines):
            if line.startswith(("__device__", "template")) and "(" in line:
                body = "\n".join(lines[i:i + 12])
                end = body.find("\n}")
                body = body if end < 0 else body[:end]
                ok = "int site)" in line and "jit_point(site)" in (line if line.rstrip().endswith("}") else body)
                helper = ok
                if ok:
                    helpers.add(re.search(r"(\w+)\(", line.split("void")[-1] if "void" in line else line).group(1))
            elif line and not line[0].isspace() and not line.startswith(("//", "#", "}")):
                helper = None
            code = line.split("//")[0]
            for pat, what in PRIMITIVES:
                if pat.search(code) and not helper and not (what == "cluster / group sync" and "jit_cluster_sync" in code):
                    bad.append("%s:%d: raw %s: %s" % (f, i + 1, what, line.strip()))
            if SPIN.search(code) and not helper and "jit_point(JIT_HERE)" not in (code + lines[i + 1]):
                bad.append("%s:%d: flag spin without jit_point(JIT_HERE) at its exit: %s" % (f, i + 1, line.strip()))
        for i, line in enumerate(lines):
            code = line.split("//")[0]
            for h in helpers:
                for m in re.finditer(r"\b%s\(" % h, code):
                    if not line.startswith(("__device__", "template")) and "JIT_HERE" not in code:
                        bad.append("%s:%d: %s without JIT_HERE: %s" % (f, i + 1, h, line.strip()))
            if line.startswith("__global__"):
                j = i
                while "{" not in lines[j]:
                    j += 1
                if "jit_entry(" not in lines[j]:
                    bad.append("%s:%d: kernel without jit_entry: %s" % (f, i + 1, line.strip()))
        if any("JIT_HERE" in l or "jit_entry(" in l for l in lines):
            assert f in files, "%s has sites but is not in JIT_FILE_LIST" % f
            assert len(lines) < MAX_LINE, "%s: sites past line %d do not fit JIT_MAX_LINE" % (f, MAX_LINE)
    assert not bad, "synchronisation outside the jitter sites:\n" + "\n".join(bad)
    assert len(_sites()) > 150


# ------------------------------------------------------------------------------------------------ GPU runs
def _fixture(name):
    z = np.load(os.path.join(ROOT, "tests", "golden", ("reach_" + name if name in REACH else name) + ".npz"))
    return {k: z[k] for k in z.files}


def _report(label, g, p, ext, ppmd_crc):
    """_mismatch_report over the first p.size bits of the fixture."""
    from test_stress_data import _mismatch_report
    nb = p.size
    want = dict(g, p=g["p"][:nb], crc_fx=g["crc_fx"][:(nb + 4095) // 4096], crc_p8=g["crc_p8"][:(nb + 4095) // 4096],
                ppmd_crc=g["ppmd_crc"][:nb // 8] if "ppmd_crc" in g else np.zeros(0, dtype=np.uint32))
    crc = lambda lo, hi: np.array([zlib.crc32(np.ascontiguousarray(ext[b:b + 4096, lo:hi]).tobytes()) for b in range(0, nb, 4096)], dtype=np.uint32)
    ppmd = np.array(ppmd_crc, dtype=np.uint32) if "ppmd_crc" in g else np.zeros(0, dtype=np.uint32)
    r = _mismatch_report(label, want, p, crc(0, 431), crc(431, 2022), ext[:64], ppmd)
    if r:
        pytest.fail(r.replace("stress_" + label, label), pytrace=False)


def _bulk(cm, name, n=None, piece=2048, dictionary=None, pretrain=None):
    """Bulk calls of `piece` bytes over the first n bytes: probabilities, codes and PPMD distributions. `pretrain`: bytes
    pretrained before the first bit, all but the last 64 in bulk (pretrain_bytes), those bit by bit (Pretrain(bit))."""
    g = _fixture(name)
    s = g["stream"][:n]
    P = cm.Predictor(g["vocab"], dictionary_path=dictionary)
    ps, exts, ppmd_crc = [], [], []
    try:
        if pretrain is not None:
            P.pretrain_bytes(pretrain[:-64])
            for byte in pretrain[-64:]:
                for j in range(7, -1, -1):
                    P.Pretrain((byte >> j) & 1)
        for off in range(0, s.size, piece):
            part = s[off:off + piece]
            ps.append(P.code_bytes(part))
            exts.append(P.debug_fetch(10, (part.size * 8, 2022), np.uint16))
            if "ppmd_crc" in g:
                rows = P.debug_fetch(8, (part.size, 256), np.float32)
                ppmd_crc += [zlib.crc32(rows[t].tobytes()) for t in range(part.size)]
    finally:
        P.close()
    _report(name, g, np.concatenate(ps), np.concatenate(exts), ppmd_crc)


def _wav(cm, name):
    """The WAV stream stops with CMIXB200_ERR_UNSUPPORTED no earlier than its first sample, every probability before equal."""
    from gen_wav import ENTRY
    from test_call_schedules import _expect
    g = _fixture(name)
    s = g["stream"]
    P = cm.Predictor(g["vocab"])
    try:
        for lo, hi in ((0, ENTRY - 1), (ENTRY - 1, ENTRY + 1), (ENTRY + 1, s.size)):
            try:
                got = P.code_bytes(s[lo:hi])
            except RuntimeError as e:
                assert lo > 0 and "image / audio / JPEG" in str(e), "%s: bytes [%d,%d): %s" % (name, lo, hi, e)
                break
            _expect("%s: bytes [%d,%d)" % (name, lo, hi), got, g["p"][lo * 8:hi * 8], lo * 8)
    finally:
        P.close()


def _awkward(cm, name):
    """Bulk calls of awkward sizes up to the bytes the stream targets, lock-step across them, awkward bulk calls to the end."""
    from test_call_schedules import _expect, _lock_step
    from test_reach import _awkward as pieces, _target
    g = _fixture(name)
    s, p = g["stream"], g["p"]
    lo, hi = _target(name, s)
    P = cm.Predictor(g["vocab"])
    try:
        for a, b in pieces(0, lo):
            _expect("reach_%s: bulk [%d,%d)" % (name, a, b), P.code_bytes(s[a:b]), p[a * 8:b * 8], a * 8)
        _lock_step(P, g, lo * 8, hi * 8, "reach_%s: lock-step [%d,%d)" % (name, lo, hi))
        for a, b in pieces(hi, s.size):
            _expect("reach_%s: bulk [%d,%d) after lock-step" % (name, a, b), P.code_bytes(s[a:b]), p[a * 8:b * 8], a * 8)
    finally:
        P.close()


def _batch(cm, names, n=None):
    """Three streams side by side in one code_batch_device call."""
    import torch
    from cmix_b200.capi import code_batch_device
    from test_call_schedules import _expect
    gs = [_fixture(x) for x in names]
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
            _expect("batch of %s, %d bytes each: %s" % (list(names), n, x), out.cpu().numpy(), g["p"][:n * 8])
    finally:
        for P in preds:
            P.close()


def _round_trip(cm, port, name, n_decode=None):
    """Device encoder -> archive equal to the host encoder's over the reference's probabilities -> device decoder."""
    from test_call_schedules import _expect, _first_bad_byte, _host_archive
    g = _fixture(name)
    s, p = g["stream"], g["p"]
    enc = cm.Predictor(g["vocab"])
    try:
        enc.coder_begin(2 * s.size + 64)
        _expect("%s: encoder" % name, enc.code_bytes(s), p)
        archive = enc.coder_finish()
    finally:
        enc.close()
    want = _host_archive(port, p, np.unpackbits(s))
    assert archive == want, "%s: device archive differs from the host encoder's: %s" % (name, _first_bad_byte(archive, want))
    n = n_decode or s.size
    dec = cm.Predictor(g["vocab"])
    try:
        out = dec.decode_bytes(archive, n)
    finally:
        dec.close()
    assert out.tobytes() == s[:n].tobytes(), "%s, decoder: %s" % (name, _first_bad_byte(out, s[:n]))


def _child(jobs_json):
    """Run in a child interpreter with CMIXB200_LIB = the jitter build: each job is [config, schedule, args]. Prints one JSON
    line per job and, last, the sites that slept."""
    import cmix_b200
    from cmix_b200.capi import load_library
    lib = load_library()
    lib.cmixb200_jitter_config.argtypes = [ctypes.c_int, ctypes.c_uint, ctypes.c_int, ctypes.c_int, ctypes.c_int]
    lib.cmixb200_jitter_counts.argtypes = [ctypes.c_void_p, ctypes.c_size_t]
    port = None
    for cfg, sched, args in json.loads(jobs_json):
        mode = cfg[0]
        a = cfg[2]
        if mode in ("starve", "hurry"):
            a = GROUPS[a]
        elif mode == "entry":
            a = JK[a]
        t0 = time.perf_counter()
        try:
            if lib.cmixb200_jitter_config(MODES["JIT_" + mode.upper()], cfg[1], a, cfg[3], cfg[4]) != 0:
                raise RuntimeError("jitter config: " + lib.cmixb200_last_error().decode())
            if sched == "bulk":
                _bulk(cmix_b200, *args)
            elif sched == "wrt":
                from test_call_schedules import _pretrain_buffer
                _bulk(cmix_b200, "full_wrt", 2048, 2048, args[0], _pretrain_buffer(args[0]))
            elif sched == "wav":
                _wav(cmix_b200, *args)
            elif sched == "awkward":
                _awkward(cmix_b200, *args)
            elif sched == "batch":
                _batch(cmix_b200, *args)
            elif sched == "round_trip":
                if port is None:
                    from oracle_io import load_port
                    port = load_port()
                _round_trip(cmix_b200, port, *args)
            else:
                raise ValueError(sched)
            msg = None
        except BaseException as e:      # pytest.fail raises an exception outside pytest's Exception tree
            msg = "%s: %s" % (type(e).__name__, e)
        print(json.dumps({"cfg": cfg, "sched": sched, "args": args, "s": round(time.perf_counter() - t0, 2), "fail": msg}), flush=True)
        if msg and ("CUDA" in msg or "cuda" in msg):
            break                        # the context may be gone: report, do not go on
    lib.cmixb200_jitter_config(MODES["JIT_OFF"], 0, 0, 0, 0)
    n = len(_files()) * MAX_LINE
    counts = np.zeros(n, dtype=np.uint32)
    if lib.cmixb200_jitter_counts(counts.ctypes.data, n) == 0:
        print("FIRED " + json.dumps({int(i): int(counts[i]) for i in np.nonzero(counts)[0]}), flush=True)


def _describe(cfg):
    mode, seed, a, b, c = cfg
    if mode == "random":
        return "mode random, seed %#x, density %d/65536" % (seed, a)
    if mode == "entry":
        return "mode entry, kernel %s, %d us every %d launches" % (a, b, c)
    return "mode %s, group %s" % (mode, a)


FIRED = {}          # site -> sleeps, over every GPU test of this module
RAN = set()


def _run(jitter_lib, label, jobs, env=None, timeout=1500):
    """The jobs in a child interpreter; fails with every failing job's configuration and first difference."""
    import gc
    import torch
    gc.collect()
    torch.cuda.empty_cache()
    e = dict(os.environ, CMIXB200_LIB=jitter_lib, **(env or {}))
    e.setdefault("CMIXB200_PPMD_MB", "512")
    code = "import sys; sys.path[:0] = sys.argv[1:4]; import test_schedule_jitter as m; m._child(sys.argv[4])"
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [
        "-c", code, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools"), ROOT, json.dumps(jobs)]
    t0 = time.perf_counter()
    r = subprocess.run(cmd, env=e, cwd=ROOT, capture_output=True, text=True, timeout=timeout)
    results, fails = [], []
    for line in r.stdout.splitlines():
        if line.startswith("{"):
            results.append(json.loads(line))
        elif line.startswith("FIRED "):
            for k, v in json.loads(line[6:]).items():
                FIRED[int(k)] = FIRED.get(int(k), 0) + v
    for x in results:
        print("%-40s %-10s %-45s %6.1f s%s" % (x["cfg"], x["sched"], x["args"][:3] if x["sched"] != "wrt" else "full_wrt", x["s"],
                                              "  FAIL" if x["fail"] else ""))
        if x["fail"]:
            fails.append("%s, schedule %s %s: %s" % (_describe(x["cfg"]), x["sched"], x["args"] if x["sched"] != "wrt" else "full_wrt", x["fail"]))
    print("%s: %d runs in %.0f s" % (label, len(results), time.perf_counter() - t0))
    assert r.returncode == 0, "%s: child failed:\n%s\n%s" % (label, r.stdout[-3000:], r.stderr[-3000:])
    assert not fails, "%s: %d of %d runs differ from the reference:\n%s" % (label, len(fails), len(results), "\n".join(fails))
    assert len(results) == len(jobs), "%s: %d of %d runs reported" % (label, len(results), len(jobs))
    RAN.add(label)


def _random(seed):
    return ["random", seed, DENSITY, 0, 0]


@pytest.mark.gpu
@pytest.mark.timeout(1800)
def test_random_jitter_bulk(jitter_lib, dict_path):
    """Bulk calls of 2048 bytes on every fixture: the seven reach_*, stress_mixed, overflow_random6k (mixers past their
    10 000-row cap), near_mp3_tag, full_wrt with the dictionary and pretraining (in bulk, then bit by bit), and a WAV
    stream that must stop at its first sample with an identical prefix."""
    jobs = []
    for seed in SEEDS:
        jobs += [[_random(seed), "bulk", [n]] for n in REACH + ["stress_mixed", "overflow_random6k", "near_mp3_tag"]]
        jobs += [[_random(seed), "wav", [WAV]]]
    jobs += [[_random(seed), "wrt", [dict_path]] for seed in (SEEDS if SLOW else SEEDS[:1])]
    _run(jitter_lib, "random, bulk", jobs)


@pytest.mark.gpu
@pytest.mark.timeout(1800)
def test_random_jitter_call_schedules(jitter_lib, port):
    """Awkward bulk pieces around a lock-step stretch over each reach_* target; three streams in one code_batch_device;
    device encoder -> device decoder."""
    jobs = []
    for k, seed in enumerate(SEEDS):
        jobs += [[_random(seed), "awkward", [n]] for n in REACH]
        jobs += [[_random(seed), "batch", [[REACH[(3 * k + i) % 7] for i in range(3)]]]]
        jobs += [[_random(seed), "round_trip", [["dbase", "stress_mixed", "fxwiki"][k], 512]]]
    _run(jitter_lib, "random, call schedules", jobs)


STARVE_GROUPS = [g for g in GROUPS if g.startswith(("JG_P8_", "JG_MIX_C", "JG_MIX_T", "JG_MIX_MOVERS", "JG_LSTM_"))]


@pytest.mark.gpu
@pytest.mark.timeout(2400)
def test_starve_and_hurry_each_warp_group(jitter_lib):
    """Each warp group of PAQ8's model CTA (and its mixer CTA), of mix_kernel_v3 and of the LSTM cluster alone slow, then
    alone fast, on two reach_* fixtures and overflow_random6k."""
    jobs = []
    for g in STARVE_GROUPS:
        for mode in ("starve", "hurry"):
            cfg = [mode, 0, g, 0, 0]
            jobs += [[cfg, "bulk", [n]] for n in ("x86", "english", "overflow_random6k")]
    _run(jitter_lib, "starve / hurry", jobs, timeout=2300)


@pytest.mark.gpu
@pytest.mark.timeout(1800)
def test_late_kernel_entry(jitter_lib, port):
    """Each kernel on a side stream starts 200 us late (every launch of a bulk kernel, every third of a per-bit kernel): in
    bulk calls, in lock-step and in the decoder's graphs; and the coder's flush behind the last bulk call."""
    jobs = []
    for k in ["JK_PPMD", "JK_SMALL", "JK_LSTM", "JK_FXCM", "JK_PAQ8"]:
        jobs += [[["entry", 0, k, 200, 1], "bulk", ["dbase", 1024, 128]]]
    for k in ["JK_FXCM_BIT", "JK_PAQ8_BIT", "JK_SMALL_PERCEIVE", "JK_PPMD_BYTE", "JK_LSTM_BYTE"]:
        jobs += [[["entry", 0, k, 200, 3], "awkward", ["xml"]], [["entry", 0, k, 200, 3], "round_trip", ["fxwiki", 256]]]
    jobs += [[["entry", 0, "JK_ENCODE_FLUSH", 200, 1], "round_trip", ["dbase", 256]]]     # once per archive
    _run(jitter_lib, "late entry", jobs)


@pytest.mark.gpu
@pytest.mark.timeout(1200)
def test_late_mixer_with_producers_many_sub_chunks_ahead(jitter_lib):
    """mix_kernel_v3 starts 200 us late on every launch, with 16-byte sub-chunks in one launch group: the producers of
    sub-chunk k+1 and later run while the mixer of sub-chunk k has not started."""
    jobs = [[["entry", 0, "JK_MIX", 200, 1], "bulk", [n, 2048]] for n in ["english", "stress_mixed"]]
    _run(jitter_lib, "late mixer, sub-chunk 16", jobs, env={"CMIXB200_SUBCHUNK": "16", "CMIXB200_GROUP": "1"})


@pytest.mark.gpu
def test_every_site_slept():
    """After the module's runs every site slept at least once, or is in NEVER_FIRES with its reason: a site on a path no
    run reaches would otherwise give false comfort."""
    want = {"random, bulk", "random, call schedules", "starve / hurry", "late entry", "late mixer, sub-chunk 16"}
    if RAN != want:
        pytest.skip("needs every GPU test of this module in the same session (ran: %s)" % sorted(RAN))
    files = _files()
    allowed = {(f, text) for f, text, _ in NEVER_FIRES}
    silent = []
    for f, line in _sites():
        text = open(os.path.join(CSRC, f)).read().split("\n")[line - 1].strip()
        if FIRED.get(files.index(f) * MAX_LINE + line, 0) == 0 and (f, text) not in allowed:
            silent.append("%s:%d: %s" % (f, line, text))
    print("%d sites, %d slept" % (len(_sites()), sum(1 for f, l in _sites() if FIRED.get(files.index(f) * MAX_LINE + l))))
    assert not silent, "%d sites never slept:\n%s" % (len(silent), "\n".join(silent))
