"""Runtime switches of the CUDA library (DESIGN.md "Runtime switches"): every alternative code path must give the
reference's GFA.  The switches are read once per process, so each case runs the command-line tool in a fresh
process with the variable set and compares its output with the unmodified reference binary's (stored digests,
tests/refgold.py): exact bytes, or for the tie-ordered sets the sorted lines plus the order of the non-L lines and of the L
lines' unitig ends.

Sets: tips/bubbles/multi-arcs/hot spots/deep groups, i.e. every kernel variant (warp / CTA / device-wide) is reached."""
import os
import subprocess

import pytest

from miniasm_b200 import synth
from tests.refgold import RECORD

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "miniasm_b200", "miniasm-b200")
REF = os.path.join(ROOT, "oracle", "_ref", "miniasm_ref")
OURS = REF if RECORD else CLI

SETS = {
    "chaos": "chaos",
    "bubbles800": "bubbles800",
    "shuffled": "shuffled",
    "deep": "-n 1500 -l 3000 -L 12000 -c 400 -j 30 -s 77",      # several hundred hits per read: the CTA-per-read kernels
    "multi": "-n 5000 -s 5 -d 200000 -j 30",                          # 20 % duplicated overlaps -> multi-arcs (shared marks in the transitive reduction)
    "skew": "skew_small",                                             # hot spots: slabs beyond the warp kernels' limits
    "bubbly": "-n 60000 -l 9000 -L 11000 -j 800 -c 30 -s 21",     # thousands of bubbles/tips along sorted ids
}
# "multi": jitter 30 on 10 kb reads makes equal-length arcs out of one unitig end common; the order of the L lines of such
# ties is the order the reference's unstable in-place radix sort happens to leave (DESIGN.md "Tie order")
TIES = {"multi"}
SWITCHES = [{}, {"MAB_GPU_GFA": "0", "MAB_WRITER_THREADS": "3"}, {"MAB_GPU_GFA": "0"}, {"MAB_SG_SEGSORT": "0"},
            {"MAB_GPU_GFA": "0", "MAB_SG_SEGSORT": "0"}]


@pytest.fixture(scope="module")
def pafs(built, paf_dir):
    return {k: synth.generate(v, f"{paf_dir}/sw_{k}.paf") for k, v in SETS.items()}


def gfa_form(text, tie_order_free):
    """What is compared: the bytes, or (tie_order_free) the sorted line multiset, the non-L lines in order and the (from-unitig,
    orientation) keys of the L lines in order -- L lines may only permute within the block of one unitig end."""
    if not tie_order_free:
        return text
    lines = text.split(b"\n")
    return [sorted(lines), [x for x in lines if not x.startswith(b"L\t")], [x.split(b"\t")[1:3] for x in lines if x.startswith(b"L\t")]]


def _want(path, tie_order_free):
    r = subprocess.run([REF, path], stdout=subprocess.PIPE, stderr=subprocess.PIPE)
    assert r.returncode == 0
    return gfa_form(r.stdout, tie_order_free)


@pytest.mark.parametrize("name", list(SETS))
@pytest.mark.parametrize("env", SWITCHES, ids=lambda e: "+".join(f"{k}={v}" for k, v in e.items()) or "default")
def test_switch(env, name, pafs, gold):
    r = subprocess.run([OURS, pafs[name]], stdout=subprocess.PIPE, stderr=subprocess.PIPE, env={**os.environ, **env})
    assert r.returncode == 0, r.stderr.decode()[-2000:]
    ties = name in TIES
    gold.cli("GFA modulo tie order" if ties else "GFA", [pafs[name]], gfa_form(r.stdout, ties), lambda: _want(pafs[name], ties))
