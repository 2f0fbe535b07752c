"""Per-kernel GPU times of the single-GPU pipeline, from torch.profiler (CUDA activities).

  python scripts/kernel_times.py OUT_DIR [--workload c3_1m] [--steps 3] [--warmup 2]

Each step is what bench.py times per step, preceded by the text load: mab_load_paf_text, mab_ingest, mab_select,
mab_layout, mab_unitigs.  The warm-up steps run unprofiled; the timed steps run under the profiler, which sees the
library's kernels because they run in this process.  Prints total and mean ms per step for every kernel name, largest
first, and writes the same table to OUT_DIR/kernel_times_<workload>.json.  The profiler slows the host side: take step
times from bench.py, not from here.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
from collections import defaultdict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (workload table and the in-memory PAF generator)


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip()
    except Exception:
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--workload", default="c3_1m", choices=sorted(bench.WORKLOADS))
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile
    from miniasm_b200 import capi
    if not torch.cuda.is_available():
        sys.exit("kernel_times.py: no CUDA device")
    torch.cuda.set_device(0)
    lib = capi.load_product()
    lib.set_verbose(0)
    ctx = lib.mab_create(0)
    opt = lib.default_opt()
    buf, n_bytes, n_lines, free = bench.generate_args(bench.WORKLOADS[a.workload]["args"])
    pinned = torch.empty(max(n_bytes, 1), dtype=torch.uint8, pin_memory=True)
    C.memmove(pinned.data_ptr(), buf, n_bytes)
    free()

    def step():
        lib.mab_load_paf_text(ctx, pinned.data_ptr(), n_bytes)
        lib.mab_ingest(ctx, opt.min_span, opt.min_match, 1)
        lib.mab_select(ctx, C.byref(opt), 0, 0, 100)
        lib.mab_layout(ctx, C.byref(opt), 100)
        lib.mab_unitigs(ctx)
        lib.mab_sync(ctx)

    for _ in range(a.warmup):
        step()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for _ in range(a.steps):
            step()
        torch.cuda.synchronize()

    tot_us, calls = defaultdict(float), defaultdict(int)
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA:
            tot_us[ev.name] += ev.time_range.elapsed_us()
            calls[ev.name] += 1
    rows = sorted(({"kernel": k, "total_ms": tot_us[k] / 1e3, "ms_per_step": tot_us[k] / 1e3 / a.steps, "calls_per_step": calls[k] / a.steps}
                   for k in tot_us), key=lambda r: -r["total_ms"])
    all_ms = sum(r["ms_per_step"] for r in rows)
    print(f"{a.workload}: {n_lines} PAF lines, {a.steps} profiled steps, {all_ms:.2f} ms of device activity per step")
    print(f"{'ms/step':>9} {'total ms':>9} {'calls':>6}  kernel")
    for r in rows:
        print(f"{r['ms_per_step']:9.3f} {r['total_ms']:9.3f} {r['calls_per_step']:6.1f}  {r['kernel'][:150]}")
    os.makedirs(a.out_dir, exist_ok=True)
    with open(os.path.join(a.out_dir, f"kernel_times_{a.workload}.json"), "w") as f:
        json.dump({"workload": a.workload, "paf_lines": n_lines, "steps": a.steps, "warmup": a.warmup, "gpu": gpu_info(),
                   "device_ms_per_step": all_ms, "kernels": rows}, f, indent=1)
    lib.mab_destroy(ctx)


if __name__ == "__main__":
    main()
