"""Windowed against resident ingest on config 3 (1 M reads, 50 M lines, 3.06 GB of PAF in a plain file).

Writes config 3's PAF to a temporary directory, then, in alternating order and --runs times each,
  - ingests the file through the library (mab_load_paf_file + mab_ingest against mab_ingest_file_windowed): host wall time of
    Step 1 ending in a device synchronise, and the high-water mark of the context's device allocator (mab_mem_peak),
  - runs `miniasm-b200 FILE > /dev/null` cold with MINIASM_B200_INGEST=resident and =windowed, checking every GFA against the
    sha256 of tests/golden/configs.json.
Prints one JSON object; the card and its power limit are part of it.

    python scripts/windowed_times.py [--runs 3] [--window BYTES]
"""
import argparse
import ctypes as C
import hashlib
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from miniasm_b200 import capi  # noqa: E402

GOLD = json.load(open(os.path.join(ROOT, "tests", "golden", "configs.json")))["c3_1m"]


def ingest(lib, path, window):
    """(wall seconds, allocator peak in bytes, hits stored) of Step 1 on a fresh context; window None = the resident ingest"""
    opt = lib.default_opt()
    ctx = lib.mab_create(0)
    lib.mab_sync(ctx)
    t0 = time.perf_counter()
    if window is None:
        assert lib.mab_load_paf_file(ctx, path.encode()) == 0
        lib.mab_ingest(ctx, opt.min_span, opt.min_match, 1)
    else:
        assert lib.mab_ingest_file_windowed(ctx, path.encode(), window, opt.min_span, opt.min_match, 1) == 0
    lib.mab_sync(ctx)
    wall = time.perf_counter() - t0
    peak, n_hits = lib.mab_mem_peak(ctx, 0), lib.mab_stats(ctx).contents.n_hits_stored
    lib.mab_destroy(ctx)
    return wall, peak, n_hits


def cold(cli, path, mode, window):
    env = dict(os.environ, MINIASM_B200_INGEST=mode, MINIASM_B200_WINDOW=str(window))
    t0 = time.perf_counter()
    r = subprocess.run([cli, path], stdout=subprocess.PIPE, stderr=subprocess.PIPE, env=env)
    wall = time.perf_counter() - t0
    assert r.returncode == 0, r.stderr[-2000:]
    assert hashlib.sha256(r.stdout).hexdigest() == GOLD["gfa_sha256"], f"GFA digest differs: {mode}"
    return wall


def summary(xs):
    return dict(median_s=statistics.median(xs), min_s=min(xs), max_s=max(xs), runs=xs)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--window", type=int, default=256 << 20)
    a = ap.parse_args()
    cli = os.path.join(ROOT, "miniasm_b200", "miniasm-b200")
    lib = capi.load_product()
    lib.set_verbose(0)
    out = {"gpu": subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                 stdout=subprocess.PIPE, text=True).stdout.strip(), "window_bytes": a.window}
    with tempfile.TemporaryDirectory() as td:
        plain = os.path.join(td, "c3.paf")
        buf, n_bytes, n_lines, free = bench.generate(1_000_000, 3)
        try:
            with open(plain, "wb") as f:
                f.write((C.c_char * n_bytes).from_address(buf.value))
        finally:
            free()
        out["paf_bytes"] = n_bytes
        ingest(lib, plain, None)                               # warm-up: module load, page cache
        walls = {"resident": [], "windowed": []}
        peaks = {"resident": set(), "windowed": set()}
        for _ in range(a.runs):
            for mode, window in (("resident", None), ("windowed", a.window)):
                w, peak, n_hits = ingest(lib, plain, window)
                walls[mode].append(w)
                peaks[mode].add(peak)
        out["n_hits"] = n_hits
        out["ingest_wall"] = {k: summary(v) for k, v in walls.items()}
        out["ingest_device_peak_bytes"] = {k: sorted(v) for k, v in peaks.items()}
        cw = {"resident": [], "windowed": []}
        for _ in range(a.runs):
            for mode in cw:
                cw[mode].append(cold(cli, plain, mode, a.window))
        out["cold_cli"] = {k: summary(v) for k, v in cw.items()}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
