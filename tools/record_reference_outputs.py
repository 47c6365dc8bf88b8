#!/usr/bin/env python3
"""Re-records tests/golden/reference_outputs.npz (see tests/ref_record.py): runs the tests that compare with the reference's
own sources with MPLB_RECORD_REFERENCE=1.  Needs oracle/_ref/libmplref.so, which __graft_entry__.build() makes where the
reference tree exists.  The GPU tests among them take the reference's side before any GPU call, so their values are
recorded on a machine without a GPU too (their GPU part then fails there, which does not matter for the recording).

  python tools/record_reference_outputs.py"""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TESTS = ["tests/test_oracle_vs_reference.py", "tests/test_oracle_fuzz_vs_reference.py", "tests/test_gpu_vs_reference.py",
         "tests/test_oracle_trajsolver.py::test_oracle_equals_reference_sources",
         "tests/test_oracle_trajsolver_edges.py::test_oracle_equals_reference_sources",
         "tests/test_oracle_lpa.py::test_oracle_equals_reference_sources"]


def main():
    path = os.path.join(ROOT, "tests", "golden", "reference_outputs.npz")
    if os.path.exists(path):
        os.remove(path)
    env = dict(os.environ, MPLB_RECORD_REFERENCE="1")
    subprocess.call([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider"] + TESTS, cwd=ROOT, env=env)
    if not os.path.exists(path):
        raise SystemExit("nothing was recorded (is oracle/_ref/libmplref.so built?)")
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
