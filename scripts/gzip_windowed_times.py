"""The windowed ingest of gzipped PAF: GPU inflate a segment at a time against zlib on the host, on config 3 (1 M reads, 50 M
lines, 3.06 GB of PAF) written as gzip -1 and gzip -6 files.

In alternating order and --runs times each, for each file:
  - Step 1 through the library in a fresh process: the resident GPU route (mab_load_paf_file + mab_ingest), the windowed GPU
    route (mab_ingest_file_windowed, window 0 = the gzip default) and, from the library of an earlier build passed by --parent
    (a directory holding its libminiasm_b200.so and miniasm-b200), its windowed route, which inflates with zlib on the host twice:
    host wall time of Step 1 ending in a device synchronise, and the high-water mark of the device allocator (mab_mem_peak);
  - `miniasm-b200 FILE > /dev/null` cold for the same three (MINIASM_B200_INGEST=resident / windowed), every GFA checked against the
    sha256 of tests/golden/configs.json;
  - the streaming inflater's phase times summed over its segments and both passes (MAB_TRACE's [T::gzstream] line).
Then, on the gzip -1 file, --runs windowed GPU Step 1 runs per window size and chunk size (MAB_GZ_CHUNK), alternating (--sweep).
Prints one JSON object; the card and its power limit are part of it.

    python scripts/gzip_windowed_times.py --parent DIR [--runs 3] [--levels 1,6] [--no-cold] [--sweep]
                                          [--sweep-windows 268435456,1073741824,2147483648] [--sweep-chunks 16384,65536,0]
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

GOLD = json.load(open(os.path.join(ROOT, "tests", "golden", "configs.json")))["c3_1m"]
TRACE = re.compile(rb"\[T::gzstream\] .*?read ([\d.]+) find ([\d.]+) decode ([\d.]+) chain ([\d.]+) window ([\d.]+) resolve ([\d.]+) "
                   rb"crc ([\d.]+) ms; (\d+) segments \((\d+) grown\), (\d+) chunks, (\d+) units, (\d+) chained, (\d+) bytes out, "
                   rb"scratch peak (\d+)")


def one(lib_path, route, path, window):
    """Step 1 in this process: (wall seconds, allocator peak, hits stored)"""
    from miniasm_b200 import capi
    lib = capi.Lib(lib_path, product=True, strict=False) if lib_path else capi.load_product()
    lib.set_verbose(0)
    opt = lib.default_opt()
    ctx = lib.mab_create(0)
    lib.mab_sync(ctx)
    t0 = time.perf_counter()
    if route == "resident":
        assert lib.mab_load_paf_file(ctx, path.encode()) == 0
        lib.mab_ingest(ctx, opt.min_span, opt.min_match, 1)
    else:
        assert lib.mab_ingest_file_windowed(ctx, path.encode(), window, opt.min_span, opt.min_match, 1) == 0
    lib.mab_sync(ctx)
    wall = time.perf_counter() - t0
    print(json.dumps(dict(wall=wall, peak=lib.mab_mem_peak(ctx, 0), n_hits=lib.mab_stats(ctx).contents.n_hits_stored)))
    lib.mab_destroy(ctx)


def step1(lib_path, route, path, window=0, env=None):
    r = subprocess.run([sys.executable, __file__, "--one", lib_path or "", route, path, str(window)], stdout=subprocess.PIPE,
                       stderr=subprocess.PIPE, env=dict(os.environ, MAB_TRACE="1", **(env or {})))
    assert r.returncode == 0, r.stderr[-2000:]
    res = json.loads(r.stdout.decode().strip().splitlines()[-1])
    m = TRACE.search(r.stderr)
    if m:
        g = m.groups()
        res["phases_ms"] = dict(zip(["read", "find", "decode", "chain", "window", "resolve", "crc"], map(float, g[:7])))
        res["counts"] = dict(zip(["segments", "grown", "chunks", "units", "chained", "bytes_out", "scratch_peak"], map(int, g[7:])))
    return res


def cold(cli, path, mode):
    env = dict(os.environ, MINIASM_B200_INGEST=mode)
    env.pop("MINIASM_B200_WINDOW", None)
    t0 = time.perf_counter()
    r = subprocess.run([cli, path], stdout=subprocess.PIPE, stderr=subprocess.PIPE, env=env)
    wall = time.perf_counter() - t0
    assert r.returncode == 0, r.stderr[-2000:]
    assert hashlib.sha256(r.stdout).hexdigest() == GOLD["gfa_sha256"], f"GFA digest differs: {cli} {mode}"
    return wall


def summary(xs):
    return dict(median_s=statistics.median(xs), min_s=min(xs), max_s=max(xs), runs=xs)


def write_gz(path, data, level):
    co = zlib.compressobj(level, zlib.DEFLATED, 31)
    with open(path, "wb") as f:
        for i in range(0, len(data), 64 << 20):
            f.write(co.compress(data[i:i + (64 << 20)]))
        f.write(co.flush())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--parent", required=True)
    ap.add_argument("--sweep", action="store_true")
    ap.add_argument("--sweep-only", action="store_true", help="only the gzip -1 file and the sweep")
    ap.add_argument("--levels", default="1,6")
    ap.add_argument("--no-cold", action="store_true", help="skip the cold command lines")
    ap.add_argument("--sweep-windows", default="268435456,1073741824,2147483648")
    ap.add_argument("--sweep-chunks", default="16384,65536,0", help="0 = the default chunk size")
    a = ap.parse_args()
    import bench
    cli = os.path.join(ROOT, "miniasm_b200", "miniasm-b200")
    parent_lib, parent_cli = os.path.join(a.parent, "libminiasm_b200.so"), os.path.join(a.parent, "miniasm-b200")
    out = {"gpu": subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                 stdout=subprocess.PIPE, text=True).stdout.strip()}
    routes = [("resident_gpu", None, "resident"), ("windowed_gpu", None, "windowed"), ("windowed_zlib_parent", parent_lib, "windowed")]
    with tempfile.TemporaryDirectory() as td:
        buf, n_bytes, n_lines, free = bench.generate(1_000_000, 3)
        try:
            data = (C.c_char * n_bytes).from_address(buf.value)
            files = {}
            levels = sorted({int(x) for x in a.levels.split(",")} | {1})
            for lvl in ((1,) if a.sweep_only else levels):
                files[lvl] = os.path.join(td, f"c3.l{lvl}.paf.gz")
                write_gz(files[lvl], memoryview(data), lvl)
        finally:
            free()
        out["paf_bytes"] = n_bytes
        for lvl, path in ([] if a.sweep_only else [(k, v) for k, v in files.items() if str(k) in a.levels.split(",")]):
            res = {"gz_bytes": os.path.getsize(path)}
            step1(None, "windowed", path)                          # warm-up: module load, page cache
            walls = {k: [] for k, _, _ in routes}
            peaks = {k: set() for k, _, _ in routes}
            phases = []
            for _ in range(a.runs):
                for name, lib, route in routes:
                    r = step1(lib, route, path)
                    walls[name].append(r["wall"])
                    peaks[name].add(r["peak"])
                    if name == "windowed_gpu":
                        phases.append(dict(r.get("phases_ms", {}), **r.get("counts", {})))
            res["step1_wall"] = {k: summary(v) for k, v in walls.items()}
            res["step1_device_peak_bytes"] = {k: sorted(v) for k, v in peaks.items()}
            res["gzstream_phases"] = phases
            cw = {"resident_gpu": [], "windowed_gpu": [], "windowed_zlib_parent": []}
            for _ in range(0 if a.no_cold else a.runs):
                cw["resident_gpu"].append(cold(cli, path, "resident"))
                cw["windowed_gpu"].append(cold(cli, path, "windowed"))
                cw["windowed_zlib_parent"].append(cold(parent_cli, path, "windowed"))
            if not a.no_cold:
                res["cold_cli"] = {k: summary(v) for k, v in cw.items()}
            out[f"gzip-{lvl}"] = res
            print(json.dumps({f"gzip-{lvl}": res}), file=sys.stderr, flush=True)
        if a.sweep or a.sweep_only:
            cells = {(int(w), int(c)): [] for w in a.sweep_windows.split(",") for c in a.sweep_chunks.split(",")}
            for _ in range(a.runs):
                for (window, chunk), runs in cells.items():
                    r = step1(None, "windowed", files[1], window, {"MAB_GZ_CHUNK": str(chunk)} if chunk else None)
                    runs.append(dict(wall=r["wall"], peak=r["peak"], phases_ms=r.get("phases_ms")))
                    print(json.dumps(dict(window_bytes=window, chunk=chunk or "auto", **runs[-1])), file=sys.stderr, flush=True)
            out["sweep_gzip-1"] = [dict(window_bytes=w, chunk=c or "auto", wall=summary([x["wall"] for x in v]), peak=sorted({x["peak"] for x in v}))
                                   for (w, c), v in cells.items()]
    print(json.dumps(out))


if __name__ == "__main__":
    if len(sys.argv) > 1 and sys.argv[1] == "--one":
        one(sys.argv[2] or None, sys.argv[3], sys.argv[4], int(sys.argv[5]))
    else:
        main()
