"""Line coverage of the host/device headers of PAQ8, FXCM and PPMD over the committed fixtures.

    python tools/coverage_report.py [--cap N] [--jobs J] [fixture ...]      # default: every tests/golden/*.npz with a stream

PAQ8 (paq8_*.h), FXCM (fxcm_model.h, fxcm_text.h) and PPMD (ppmd_model.h) are single sources: the CUDA kernels compile
the same headers that tools/paq8_check.cpp, tools/fxcm_check.cpp and tools/ppmd_host.cpp compile for the CPU. A line no
fixture runs on the host is therefore never checked on the device either. This builds the three tools with --coverage,
runs them over every fixture's stream (each run with its own GCOV_PREFIX, in parallel), merges the runs per tool with
gcov-tool and lists the executable lines of the shared headers that no run reached.

FXCM runs only where a fixture carries the LSTM feedback it consumed (`lstmfx`); a fixture recorded with the WRT
dictionary pretrains FXCM on it first, as the reference does. PAQ8 and PPMD code every fixture's stream without
pretraining. Streams longer than `cap` bytes (the long_text* fixtures) are cut to their first `cap` bytes.
"""
import argparse
import glob
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "cmix_b200", "csrc")
GOLDEN = os.path.join(ROOT, "tests", "golden")

# tool -> (source, extra flags, the shared headers it measures)
TOOLS = {
    "paq8": ("paq8_check.cpp", ["-ffp-contract=off"], ["paq8_model.h", "paq8_predict.h", "paq8_text.h", "paq8_top.h"]),
    "fxcm": ("fxcm_check.cpp", [], ["fxcm_model.h", "fxcm_text.h"]),
    "ppmd": ("ppmd_host.cpp", ["-ffp-contract=off", "-DPPMD_HOST_MAIN"], ["ppmd_model.h"]),
}
DEFAULT_CAP = 40000


def _fixtures(names=None):
    names = names or sorted(os.path.basename(f)[:-4] for f in glob.glob(os.path.join(GOLDEN, "*.npz")))
    out = {}
    for name in names:
        z = np.load(os.path.join(GOLDEN, name + ".npz"))
        if "stream" in z.files:
            out[name] = {k: z[k] for k in ("stream", "vocab", "lstmfx", "dictionary") if k in z.files}
    return out


def _build(work, tool):
    src, flags, _ = TOOLS[tool]
    d = os.path.join(work, "build", tool)
    os.makedirs(d)
    obj, exe = os.path.join(d, tool + ".o"), os.path.join(d, tool)
    subprocess.run(["g++", "-O1", "--coverage", "-std=c++17", *flags, "-I", CSRC, "-c", os.path.join(ROOT, "tools", src),
                    "-o", obj], check=True)
    subprocess.run(["g++", "--coverage", obj, "-o", exe], check=True)
    return d, exe


def _jobs(work, fixtures, cap, dict_file):
    """(tool, label, argv) of every run; inputs are written under work/in."""
    d = os.path.join(work, "in")
    os.makedirs(d)
    jobs = []
    for name, g in fixtures.items():
        s = g["stream"][:cap]
        prefix = os.path.join(d, name)
        s.tofile(prefix + ".stream")
        np.ascontiguousarray(g["vocab"], dtype=np.uint8).tofile(prefix + ".vocab")
        jobs.append(("paq8", name, [prefix, "-", str(s.size), prefix + ".p8crc"]))
        jobs.append(("ppmd", name, [prefix + ".stream", prefix + ".vocab"]))
        if "lstmfx" in g:
            g["lstmfx"][:s.size * 8].tofile(prefix + ".lstmfx.u32")
            use_dict = "dictionary" in g and bool(g["dictionary"][0])
            jobs.append(("fxcm", name, [prefix, dict_file if use_dict else "-", str(s.size), prefix + ".fxcrc"]))
    return jobs


def _gcov_lines(build_dir, tool):
    """{header: {line: count}} of the merged .gcda next to the tool's .gcno (a line inlined twice counts once per copy)."""
    r = subprocess.run(["gcov", "--json-format", "--stdout", tool + ".o"], cwd=build_dir, capture_output=True, text=True, check=True)
    want = set(TOOLS[tool][2])
    lines = {}
    for doc in r.stdout.splitlines():
        if not doc.strip():
            continue
        for f in json.loads(doc)["files"]:
            base = os.path.basename(f["file"])
            if base not in want:
                continue
            per = lines.setdefault(base, {})
            for ln in f["lines"]:
                per[ln["line_number"]] = per.get(ln["line_number"], 0) + ln["count"]
    return lines


def measure(fixtures=None, cap=DEFAULT_CAP, jobs=None, work=None):
    """Runs every fixture through the coverage builds. Returns {tool: {header: {line: count}}} and a dict of run failures
    (label -> output) for runs that exited with anything other than 0 or PAQ8's 3 (unsupported block)."""
    fixtures = fixtures if isinstance(fixtures, dict) else _fixtures(fixtures)
    own = work is None
    work = work or tempfile.mkdtemp(prefix="cov_")
    try:
        builds = {t: _build(work, t) for t in TOOLS}
        sys.path.insert(0, os.path.join(ROOT, "tools"))
        from gen_synth import dictionary
        dict_file = os.path.join(work, "english.dic")
        with open(dict_file, "wb") as f:
            f.write(dictionary())
        runs = _jobs(work, fixtures, cap, dict_file)

        def run(job):
            tool, label, argv = job
            d, exe = builds[tool]
            prefix = os.path.join(work, "gcda", tool, label)
            env = dict(os.environ, GCOV_PREFIX=prefix, GCOV_PREFIX_STRIP=str(len(d.strip(os.sep).split(os.sep))))
            r = subprocess.run([exe, *argv], capture_output=True, text=True, env=env)
            ok = r.returncode == 0 or (tool == "paq8" and r.returncode == 3)
            return tool, prefix, None if ok else "%s %s: exit %d\n%s" % (tool, label, r.returncode, (r.stdout + r.stderr)[-2000:])

        with ThreadPoolExecutor(jobs or os.cpu_count() or 4) as ex:
            results = list(ex.map(run, runs))
        failures = {}
        coverage = {}
        for tool, (d, _) in builds.items():
            dirs = [p for t, p, _ in results if t == tool and os.path.isdir(p)]
            failures.update({p: e for t, p, e in results if t == tool and e})
            if not dirs:
                continue
            merged = dirs[0]
            os.makedirs(os.path.join(work, "merge", tool))
            for i, other in enumerate(dirs[1:]):
                out = os.path.join(work, "merge", tool, str(i))
                subprocess.run(["gcov-tool", "merge", "-o", out, merged, other], check=True, capture_output=True)
                merged = out
            shutil.copy(os.path.join(merged, tool + ".gcda"), os.path.join(d, tool + ".gcda"))
            coverage[tool] = _gcov_lines(d, tool)
        return coverage, failures
    finally:
        if own:
            shutil.rmtree(work, ignore_errors=True)


def unexecuted(coverage):
    """[(tool, header, line number, text)] of every executable line of the shared headers that no run reached."""
    out = []
    for tool, files in coverage.items():
        for header, lines in sorted(files.items()):
            text = open(os.path.join(CSRC, header)).read().split("\n")
            out += [(tool, header, n, text[n - 1].strip()) for n, c in sorted(lines.items()) if c == 0]
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--cap", type=int, default=DEFAULT_CAP, help="bytes of each stream to run (default %(default)s)")
    ap.add_argument("--jobs", type=int, default=None)
    ap.add_argument("fixtures", nargs="*")
    a = ap.parse_args()
    t0 = time.time()
    coverage, failures = measure(a.fixtures or None, a.cap, a.jobs)
    for e in failures.values():
        print(e)
    missed = unexecuted(coverage)
    for tool, header, n, text in missed:
        print("%s:%d: %s" % (header, n, text))
    for tool, files in coverage.items():
        total = sum(len(v) for v in files.values())
        miss = sum(1 for t, *_ in missed if t == tool)
        print("%-5s %5d executable lines, %3d unexecuted (%s)" % (tool, total, miss, ", ".join(sorted(files))))
    print("%.0f s" % (time.time() - t0))
    return 1 if failures else 0


if __name__ == "__main__":
    sys.exit(main())
