"""Fixtures of the coverage streams (tools/gen_reach.py) from dumps of the UNMODIFIED reference (build container only).

    python tools/make_reach_goldens.py [name ...]         # default: every entry of gen_reach.STREAMS

Recipe and layout of every committed tests/golden/reach_<name>.npz are those of the stress fixtures
(tools/make_stress_goldens.py), with (n_bytes, seed) from gen_reach.STREAMS:
    python tools/gen_reach.py <name> <n_bytes> s.bin <seed>;  oracle_dump dump n s.bin <prefix> 1 <n_bytes>
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import gen_reach  # noqa: E402
from make_stress_goldens import main  # noqa: E402

if __name__ == "__main__":
    main(gen_reach, "reach")
