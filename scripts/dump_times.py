"""Wall clocks of the -p paf | bed | sg outputs, against another build of the command line.

  python scripts/dump_times.py OUT_DIR --other DIR [--workload c3_1m] [--runs 3] [--commands 0,1,2,3,4] [--no-calls]

DIR holds another build's `miniasm-b200` (with its libminiasm_b200.so beside it), e.g. the parent commit built in a directory
of its own.  On one generated PAF of the workload this measures (--commands: a subset of the five, by index):
  * the cold command-line wall clock of -S 2 -p paf, -p paf, -p bed, -S 5 -p sg and -p sg with stdout to /dev/null, each build
    `--runs` times, the two builds alternating;
  * the sha256 of each command's stdout for both builds (one more run each, stdout piped into the hash);
  * the device scratch and pinned memory of this build's writer (its MAB_TRACE line, from the hashing run);
  * the time of each mab_write_* call alone, in this process: host clock around the call after a device synchronise.
Prints one JSON document and writes it to OUT_DIR/dump_times_<workload>_<commands>.json, with the GPU's name and power limit.
"""
import argparse
import ctypes as C
import hashlib
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from miniasm_b200 import capi, synth  # noqa: E402

CLI = os.path.join(ROOT, "miniasm_b200", "miniasm-b200")
COMMANDS = [["-S", "2", "-p", "paf"], ["-p", "paf"], ["-p", "bed"], ["-S", "5", "-p", "sg"], ["-p", "sg"]]


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip()
    except Exception:
        return None


def wall(binary, args, paf):
    t0 = time.perf_counter()
    r = subprocess.run([binary] + args + [paf], stdout=subprocess.DEVNULL, stderr=subprocess.PIPE)
    t = time.perf_counter() - t0
    if r.returncode != 0:
        raise RuntimeError(f"{binary} {' '.join(args)} exited {r.returncode}: {r.stderr.decode()[-2000:]}")
    return t


def digest(binary, args, paf, trace):
    env = dict(os.environ, MAB_TRACE="1") if trace else None
    with tempfile.TemporaryFile() as err:
        p = subprocess.Popen([binary] + args + [paf], stdout=subprocess.PIPE, stderr=err, env=env)
        h, n = hashlib.sha256(), 0
        for blk in iter(lambda: p.stdout.read(1 << 22), b""):
            h.update(blk)
            n += len(blk)
        if p.wait() != 0:
            raise RuntimeError(f"{binary} {' '.join(args)} exited {p.returncode}")
        err.seek(0)
        mem = [ln for ln in err.read().decode(errors="replace").splitlines() if ln.startswith("[T::dg_dump_write]")]
    return {"sha256": h.hexdigest(), "bytes": n, "writer_memory": mem}


def writer_calls(paf, reps):
    """ms of each mab_write_* call to /dev/null, after the stages the command line runs before it"""
    lib = capi.load_product()
    lib.set_verbose(0)
    devnull = capi._libc.fopen(b"/dev/null", b"w")
    capi._libc.fflush.argtypes = [C.c_void_p]
    out = {}
    for label, stage, layout, fn in (("-S 2 -p paf", 2, False, "mab_write_paf"), ("-p paf", 100, False, "mab_write_paf"),
                                     ("-p bed", 100, False, "mab_write_bed"), ("-S 5 -p sg", 5, True, "mab_write_sg"),
                                     ("-p sg", 100, True, "mab_write_sg")):
        opt = lib.default_opt()
        ctx = lib.mab_create(0)
        assert lib.mab_load_paf_file(ctx, paf.encode()) == 0
        lib.mab_ingest(ctx, opt.min_span, opt.min_match, 1)
        lib.mab_select(ctx, C.byref(opt), 0, 0, stage)
        if layout:
            lib.mab_layout(ctx, C.byref(opt), stage)
        ms, n = [], 0
        for _ in range(reps):
            lib.mab_sync(ctx)
            t0 = time.perf_counter()
            n = getattr(lib, fn)(ctx, devnull)
            capi._libc.fflush(devnull)
            ms.append((time.perf_counter() - t0) * 1e3)
        out[label] = {"call": fn, "bytes": n, "ms": [round(x, 2) for x in ms]}
        lib.mab_destroy(ctx)
    capi._libc.fclose(devnull)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--other", required=True, help="directory with the other build's miniasm-b200")
    ap.add_argument("--workload", default="c3_1m", choices=sorted(synth.CONFIGS))
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--commands", default="0,1,2,3,4", help="indices into " + repr([" ".join(c) for c in COMMANDS]))
    ap.add_argument("--no-calls", action="store_true", help="skip the in-process timing of the mab_write_* calls")
    a = ap.parse_args()
    other = os.path.join(a.other, "miniasm-b200")
    os.makedirs(a.out_dir, exist_ok=True)
    res = {"gpu": gpu_info(), "workload": a.workload, "runs": a.runs, "wall_s": {}, "stdout": {}}
    with tempfile.TemporaryDirectory() as td:
        paf = synth.generate(a.workload, os.path.join(td, f"{a.workload}.paf"))
        res["paf_bytes"] = os.path.getsize(paf)
        print(json.dumps({"gpu": res["gpu"], "paf": a.workload, "paf_bytes": res["paf_bytes"]}), flush=True)
        for args in [COMMANDS[int(i)] for i in a.commands.split(",") if i]:
            key = " ".join(args)
            w = {"this": [], "other": []}
            for k in range(a.runs):
                order = (("this", CLI), ("other", other)) if k % 2 == 0 else (("other", other), ("this", CLI))
                for name, binary in order:
                    w[name].append(round(wall(binary, args, paf), 3))
                    print(json.dumps({"command": key, "build": name, "wall_s": w[name][-1]}), flush=True)
            res["wall_s"][key] = w
            mine, theirs = digest(CLI, args, paf, True), digest(other, args, paf, False)
            res["stdout"][key] = {"this": mine, "other": theirs, "identical": mine["sha256"] == theirs["sha256"]}
            print(json.dumps({key: {"wall_s": w, "stdout": res["stdout"][key]}}), flush=True)
        if not a.no_calls:
            res["writer_call_ms"] = writer_calls(paf, a.runs)
    print(json.dumps(res, indent=1))
    with open(os.path.join(a.out_dir, f"dump_times_{a.workload}_{a.commands.replace(',', '')}.json"), "w") as f:
        json.dump(res, f, indent=1)
    if not all(v["identical"] for v in res["stdout"].values()):
        sys.exit("stdout differs from the other build")


if __name__ == "__main__":
    main()
