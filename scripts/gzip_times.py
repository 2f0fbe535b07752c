"""Gzipped PAF on the GPU: inflate phases and the cold command line for config 3 (1 M reads, 50 M lines).

Writes config 3's PAF plain and as gzip -1 / -6 members (Python's zlib: the same deflate levels as gzip) to a temporary
directory, then runs `miniasm-b200 FILE > /dev/null` cold, in alternating order, on
  - the .gz files with this build (MAB_TRACE=1: the [T::gunzip] line gives the per-phase split, chunk counts and scratch peak),
  - the .gz files with another build (--parent, e.g. the previous commit's CLI: it inflates with gzread on the host),
  - the plain file with this build,
and checks every run's GFA against the sha256 of tests/golden/configs.json.  Prints one JSON object.

    python scripts/gzip_times.py [--parent DIR_WITH_miniasm-b200] [--runs 3]
"""
import argparse
import ctypes as C
import hashlib
import json
import os
import re
import statistics
import subprocess
import sys
import tempfile
import time
import zlib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402

GOLD = json.load(open(os.path.join(ROOT, "tests", "golden", "configs.json")))["c3_1m"]


def gzip_bytes(data, level):
    co = zlib.compressobj(level, zlib.DEFLATED, 31)
    return co.compress(data) + co.flush()


def run(cli, path, trace):
    env = dict(os.environ)
    if trace:
        env["MAB_TRACE"] = "1"
    t0 = time.perf_counter()
    r = subprocess.run([cli, path], stdout=subprocess.PIPE, stderr=subprocess.PIPE, env=env)
    wall = time.perf_counter() - t0
    assert r.returncode == 0, r.stderr[-2000:]
    assert hashlib.sha256(r.stdout).hexdigest() == GOLD["gfa_sha256"], f"GFA digest differs: {cli} {path}"
    m = re.search(rb"\[T::gunzip\] (\S+) rc (-?\d+): raw\+h2d ([\d.]+) find ([\d.]+) decode ([\d.]+) chain ([\d.]+) window ([\d.]+) "
                  rb"resolve ([\d.]+) crc ([\d.]+) ms; (\d+) chunks, (\d+) units, (\d+) chained, (\d+) confirmed, (\d+) members, "
                  rb"(\d+) bytes out, scratch peak (\d+)", r.stderr)
    ph = None
    if m:
        g = m.groups()
        ph = dict(rc=int(g[1]), raw_h2d_ms=float(g[2]), find_ms=float(g[3]), decode_ms=float(g[4]), chain_ms=float(g[5]),
                  window_ms=float(g[6]), resolve_ms=float(g[7]), crc_ms=float(g[8]), chunks=int(g[9]), units=int(g[10]),
                  chained=int(g[11]), confirmed=int(g[12]), members=int(g[13]), out_bytes=int(g[14]), scratch_peak=int(g[15]))
        dev = ph["find_ms"] + ph["decode_ms"] + ph["chain_ms"] + ph["window_ms"] + ph["resolve_ms"] + ph["crc_ms"]
        ph["inflate_gbps"] = ph["out_bytes"] / dev / 1e6 if dev else None
        ph["confirmed_share"] = ph["confirmed"] / max(ph["chunks"] - 1, 1)
    return wall, ph


def summary(xs):
    return dict(median_s=statistics.median(xs), min_s=min(xs), max_s=max(xs), runs=xs)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent", default=None, help="directory holding another build's miniasm-b200 (and its library)")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--levels", default="1,6")
    a = ap.parse_args()
    cli = os.path.join(ROOT, "miniasm_b200", "miniasm-b200")
    out = {"gpu": subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE,
                                 text=True).stdout.strip()}
    with tempfile.TemporaryDirectory() as td:
        buf, n_bytes, n_lines, free = bench.generate(1_000_000, 3)
        try:
            data = bytes((C.c_char * n_bytes).from_address(buf.value))
        finally:
            free()
        plain = os.path.join(td, "c3.paf")
        with open(plain, "wb") as f:
            f.write(data)
        for lvl in [int(x) for x in a.levels.split(",")]:
            t0 = time.perf_counter()
            gz = gzip_bytes(data, lvl)
            host_s = time.perf_counter() - t0
            path = os.path.join(td, f"c3.l{lvl}.paf.gz")
            with open(path, "wb") as f:
                f.write(gz)
            t0 = time.perf_counter()
            assert len(zlib.decompress(gz, 31)) == n_bytes
            res = {"gz_bytes": len(gz), "ratio": n_bytes / len(gz), "host_zlib_compress_s": host_s,
                   "host_zlib_inflate_s": time.perf_counter() - t0}
            del gz
            walls = {"gz_this": [], "gz_parent": [], "plain_this": []}
            phases = []
            for _ in range(a.runs):
                w, ph = run(cli, path, True)
                walls["gz_this"].append(w)
                phases.append(ph)
                if a.parent:
                    walls["gz_parent"].append(run(os.path.join(a.parent, "miniasm-b200"), path, False)[0])
                walls["plain_this"].append(run(cli, plain, False)[0])
            res["cold_cli"] = {k: summary(v) for k, v in walls.items() if v}
            res["inflate_phases"] = phases
            out[f"gzip_{lvl}"] = res
            os.unlink(path)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
