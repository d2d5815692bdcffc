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
import os
import re

import pytest

from harness import CSRC, GROUPS, MAX_LINE, jitter_files, jitter_lib, run_jitter, sass_by_function  # noqa: F401  (jitter_lib: fixture)

SLOW = os.environ.get("CMIXB200_SLOW") == "1"
SEEDS = [0x5EED0001, 0x5EED0002, 0x5EED0003]
DENSITY = 16384                                   # random mode: a quarter of the visits sleep
KERNELS = ["fill_f32", "fill_u32", "fill_sse_rows", "fill_u16", "encode_kernel", "encode_flush_kernel", "decode_begin_kernel",
           "decode_step_kernel", "fxcm_kernel", "fxcm_bit_kernel", "lstm_kernel", "lock_predict_inputs_kernel",
           "lstm_byte_kernel", "mix_kernel_v3", "mix_predict_rows_kernel", "mix_predict_final_kernel", "mix_perceive_kernel",
           "paq8_kernel", "paq8_bit_kernel", "ppmd_init_kernel", "ppmd_kernel", "ppmd_byte_kernel", "small_kernel",
           "small_predict_kernel", "small_perceive_kernel"]
REACH = ["reach_english", "reach_europe", "reach_xml", "reach_x86", "reach_dbase", "reach_bmp", "reach_fxwiki"]
WAV = "wav_pcm16_mono"

# Sites no run of this module sleeps at, each with the reason: (file, stripped text of the line, reason).
NEVER_FIRES = []


def _sass_by_kernel(lib):
    """{kernel name: its SASS}, the functions of a template kernel together."""
    out = {}
    for mangled, body in sass_by_function(lib).items():
        name = next((k for k in KERNELS if re.search(r"\d%s[A-Z]" % k, mangled)), mangled)
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
    files = jitter_files()
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
FIRED = {}          # site -> sleeps, over every GPU test of this module
RAN = set()


def _run(jitter_lib, label, jobs, env=None, timeout=1500):
    """The jobs in a child interpreter (harness.run_jitter); records the run and the sites that slept for the last test."""
    for k, v in run_jitter(jitter_lib, label, jobs, env, timeout).items():
        FIRED[k] = FIRED.get(k, 0) + v
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
        jobs += [[_random(seed), "round_trip", [["reach_dbase", "stress_mixed", "reach_fxwiki"][k], 512]]]
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
            jobs += [[cfg, "bulk", [n]] for n in ("reach_x86", "reach_english", "overflow_random6k")]
    _run(jitter_lib, "starve / hurry", jobs, timeout=2300)


@pytest.mark.gpu
@pytest.mark.timeout(1800)
def test_late_kernel_entry(jitter_lib, port):
    """Each kernel on a side stream starts 200 us late (every launch of a bulk kernel, every third of a per-bit kernel): in
    bulk calls, in lock-step and in the decoder's graphs; and the coder's flush behind the last bulk call."""
    jobs = []
    for k in ["JK_PPMD", "JK_SMALL", "JK_LSTM", "JK_FXCM", "JK_PAQ8"]:
        jobs += [[["entry", 0, k, 200, 1], "bulk", ["reach_dbase", 1024, 128]]]
    for k in ["JK_FXCM_BIT", "JK_PAQ8_BIT", "JK_SMALL_PERCEIVE", "JK_PPMD_BYTE", "JK_LSTM_BYTE"]:
        jobs += [[["entry", 0, k, 200, 3], "awkward", ["reach_xml"]], [["entry", 0, k, 200, 3], "round_trip", ["reach_fxwiki", 256]]]
    jobs += [[["entry", 0, "JK_ENCODE_FLUSH", 200, 1], "round_trip", ["reach_dbase", 256]]]     # once per archive
    _run(jitter_lib, "late entry", jobs)


@pytest.mark.gpu
@pytest.mark.timeout(1200)
def test_late_mixer_with_producers_many_sub_chunks_ahead(jitter_lib):
    """mix_kernel_v3 starts 200 us late on every launch, with 16-byte sub-chunks in one launch group: the producers of
    sub-chunk k+1 and later run while the mixer of sub-chunk k has not started."""
    jobs = [[["entry", 0, "JK_MIX", 200, 1], "bulk", [n, 2048]] for n in ["reach_english", "stress_mixed"]]
    _run(jitter_lib, "late mixer, sub-chunk 16", jobs, env={"CMIXB200_SUBCHUNK": "16", "CMIXB200_GROUP": "1"})


@pytest.mark.gpu
def test_every_site_slept():
    """After the module's runs every site slept at least once, or is in NEVER_FIRES with its reason: a site on a path no
    run reaches would otherwise give false comfort."""
    want = {"random, bulk", "random, call schedules", "starve / hurry", "late entry", "late mixer, sub-chunk 16"}
    if RAN != want:
        pytest.skip("needs every GPU test of this module in the same session (ran: %s)" % sorted(RAN))
    files = jitter_files()
    allowed = {(f, text) for f, text, _ in NEVER_FIRES}
    silent = []
    for f, line in _sites():
        text = open(os.path.join(CSRC, f)).read().split("\n")[line - 1].strip()
        if FIRED.get(files.index(f) * MAX_LINE + line, 0) == 0 and (f, text) not in allowed:
            silent.append("%s:%d: %s" % (f, line, text))
    print("%d sites, %d slept" % (len(_sites()), sum(1 for f, l in _sites() if FIRED.get(files.index(f) * MAX_LINE + l))))
    assert not silent, "%d sites never slept:\n%s" % (len(silent), "\n".join(silent))
