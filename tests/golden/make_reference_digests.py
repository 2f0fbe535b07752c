#!/usr/bin/env python
"""Records tests/golden/reference_digests.json: the reference's side of every parity test (tests/refgold.py).

Runs the parity tests with MAB_RECORD_REFERENCE=1: the unmodified reference (oracle/_ref, built by oracle/Makefile from its
sources) computes what each comparison compares against, the oracle port and the reference binary stand in for the CUDA
library and the command line, and the digests are written when the run ends.  No GPU is needed.

usage: python tests/golden/make_reference_digests.py
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
TESTS = ["tests/test_asg_gpu.py", "tests/test_clean_gpu.py", "tests/test_hit_gpu.py", "tests/test_cli_gpu.py", "tests/test_switches_gpu.py",
         "tests/test_shard_gpu.py", "tests/test_oracle_cpu.py", "tests/test_abi_cpu.py::test_struct_layouts_match_ctypes_and_reference"]
# tests of the CUDA library alone: nothing of the reference to record
PRODUCT_ONLY = ["tests/test_hit_gpu.py::test_streamed_ingest_equals_two_calls", "tests/test_asg_gpu.py::test_empty_graph",
                "tests/test_hit_gpu.py::test_empty_inputs"]


def main():
    if not os.path.exists(os.path.join(ROOT, "oracle", "_ref", "libminiasm_ref.so")):
        sys.exit("oracle/_ref is not built: run __graft_entry__.build() where the reference's sources are")
    path = os.path.join(HERE, "reference_digests.json")
    if os.path.exists(path):
        os.unlink(path)
    cmd = [sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", *TESTS] + [f"--deselect={t}" for t in PRODUCT_ONLY]
    sys.exit(subprocess.call(cmd, cwd=ROOT, env={**os.environ, "MAB_RECORD_REFERENCE": "1"}))


if __name__ == "__main__":
    main()
