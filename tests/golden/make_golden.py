#!/usr/bin/env python
"""Regenerates tests/golden/*.json (+ small .gfa.gz) by running the UNMODIFIED reference binary
(oracle/_ref/miniasm_ref, built from the reference's sources by oracle/Makefile) on deterministic synthetic PAFs.

The reference ships no tests or vectors of its own, so these files are the pinned known answers for the
CPU-only test tier: final GFA and the `-S k -p paf|sg|bed|ug` stage dumps the reference offers as debug
hooks (SURVEY.md section 4).  Inputs are not stored: (pafgen options, sha256 of the PAF) identify them.

usage: python tests/golden/make_golden.py        (needs oracle/_ref/miniasm_ref)
"""
import gzip
import hashlib
import json
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from miniasm_b200 import synth  # noqa: E402

REF = os.path.join(ROOT, "oracle", "_ref", "miniasm_ref")
SETS = ["tiny_exact", "chaos_small", "lowcov", "shuffled", "jitter30"]
KEEP_TEXT = {"chaos_small", "lowcov"}            # full GFA text kept for these (small)
DUMPS = [["-S2", "-p", "paf"], ["-S3", "-p", "paf"], ["-S4", "-p", "paf"], ["-S5", "-p", "paf"], ["-p", "bed"],
         ["-S5", "-p", "sg"], ["-S6", "-p", "sg"], ["-S7", "-p", "sg"], ["-S9", "-p", "sg"], ["-S10", "-p", "sg"], ["-p", "sg"],
         ["-S6", "-p", "ug"], ["-S7", "-p", "ug"], ["-c", "2", "-e", "2"], ["-1"], ["-2"], ["-b"], ["-R"]]


def sha_lines(text, sort):
    lines = text.split(b"\n")
    if sort:
        lines = sorted(lines)
    return hashlib.sha256(b"\n".join(lines)).hexdigest()


def run(args):
    r = subprocess.run([REF] + args, stdout=subprocess.PIPE, stderr=subprocess.PIPE, check=True)
    return r.stdout, r.stderr.decode()


def counts(stderr):
    keep = ("stored", "remain after", "read ", "reduced", "multi-arcs", "asymmetric", "tips", "bubbles", "short overlaps", "internal", "bi-loops")
    out = []
    for ln in stderr.splitlines():
        if ln.startswith("[M::") and any(k in ln for k in keep):
            tag, _, msg = ln.partition("] ")
            out.append(tag.split("::")[1] + ": " + msg)
    return out


def main():
    tmp = "/tmp/mab_golden"
    os.makedirs(tmp, exist_ok=True)
    for name in SETS:
        paf = synth.generate(name, os.path.join(tmp, name + ".paf"))
        gfa, err = run([paf])
        rec = {"pafgen_args": synth.CONFIGS[name], "paf_sha256": synth.sha256(paf), "paf_lines": sum(1 for _ in open(paf, "rb")),
               "gfa_sha256": hashlib.sha256(gfa).hexdigest(), "gfa_sorted_sha256": sha_lines(gfa, True), "stderr_counts": counts(err), "dumps": {}}
        for d in DUMPS:
            out, _ = run(d + [paf])
            rec["dumps"][" ".join(d)] = {"sha256": hashlib.sha256(out).hexdigest(), "sorted_sha256": sha_lines(out, True), "n_lines": out.count(b"\n")}
        with open(os.path.join(HERE, name + ".json"), "w") as f:
            json.dump(rec, f, indent=1, sort_keys=True)
        if name in KEEP_TEXT:
            with gzip.GzipFile(os.path.join(HERE, name + ".gfa.gz"), "wb", mtime=0) as f:
                f.write(gfa)
        print(name, rec["paf_lines"], "lines", len(gfa), "GFA bytes")
    next_rows(tmp)


NEXT_R = "-n 4000 -l 2000 -L 30000 -c 30 -j 100 -s 41"          # read lengths spread over a factor of 15: -R has something to drop
NEXT_F = ["fa_var_gaps_extra_dups_missing.fa", "fq_crlf_extra_dups.fq", "fq_multi.fq"]


def next_rows(tmp):
    """SURVEY.md 8f rows 2 and 3: `-R` on a length-skewed set, `-f reads` on three layouts of the reads file (written by the
    generator the tests use, tests/test_cli_gpu.py::_reads_file; the files are identified by their sha256)."""
    from tests.test_cli_gpu import _reads_file
    rec = {"R": {}, "f": {}}
    paf = synth.generate(NEXT_R, os.path.join(tmp, "next_R.paf"))
    gfa, err = run(["-R", paf])
    rec["R"] = {"pafgen_args": NEXT_R, "paf_sha256": synth.sha256(paf), "gfa_sha256": hashlib.sha256(gfa).hexdigest(),
                "dropped": [ln.partition("] ")[2] for ln in err.splitlines() if "dropped" in ln],
                "stderr_counts": [c for c in counts(err) if not c.startswith("main:")]}
    paf = synth.generate("chaos_small", os.path.join(tmp, "chaos_small.paf"))
    for fn in NEXT_F:
        style, ext = fn.rsplit(".", 1)
        reads = _reads_file(paf, os.path.join(tmp, "next_" + fn), style)
        gfa, _ = run(["-f", reads, paf])
        rec["f"][fn] = {"reads_sha256": hashlib.sha256(open(reads, "rb").read()).hexdigest(), "gfa_sha256": hashlib.sha256(gfa).hexdigest(),
                        "gfa_bytes": len(gfa)}
    with open(os.path.join(HERE, "next_rows.json"), "w") as f:
        json.dump(rec, f, indent=1, sort_keys=True)
    print("next rows:", rec["R"]["dropped"], {k: v["gfa_bytes"] for k, v in rec["f"].items()})


if __name__ == "__main__":
    if sys.argv[1:] == ["next"]:
        os.makedirs("/tmp/mab_golden", exist_ok=True)
        next_rows("/tmp/mab_golden")
    else:
        main()
