"""The voxel grid (K1) alone on the 23 bench scans: per-kernel device times, per-call device span, launches, leaf statistics.

    python tools/vg_probe.py [--lib path/to/liblsdreg.so] [--repeats 20] [--out file.json]

Per scan: 3 warm calls, then `repeats` calls of lsd_voxelgrid_filter_dev (device-resident input, leaf 0.5 m) traced with
torch.profiler (CUDA activity only).  A call's span runs from its first kernel's start to its last kernel's end on the device
timeline; per kernel and per span the median over the repeats is taken, then the median (and max) over the scans.  The host
clock over the same repeats, ended by a device synchronise, is reported beside it.  Leaf statistics are counted on the CPU."""
import argparse
import ctypes as C
import json
import os
import statistics
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
import lsdreg  # noqa: E402
import torch  # noqa: E402

SMALL, CAP = 8, 512     # kVgSmall, kVgCap in csrc/voxelgrid.cu


def leaf_stats(p, leaf=0.5):
    p = p[np.isfinite(p[:, :3]).all(1), :3]
    inv = np.float32(1.0 / leaf)
    mn, mx = p.min(0), p.max(0)
    minb, maxb = np.floor(mn * inv).astype(np.int64), np.floor(mx * inv).astype(np.int64)
    div = maxb - minb + 1
    ijk = np.floor(p * inv).astype(np.int64) - minb
    _, c = np.unique(ijk[:, 0] + ijk[:, 1] * div[0] + ijk[:, 2] * div[0] * div[1], return_counts=True)
    c = c.astype(np.int64)
    return {"points": int(p.shape[0]), "leaves": int(c.size), "mean_k": round(float(c.mean()), 2), "max_k": int(c.max()),
            "sum_k2": int((c * c).sum()), "leaves_gt_small": int((c > SMALL).sum()), "points_in_gt_small": int(c[c > SMALL].sum()),
            "leaves_gt_32": int((c > 32).sum()), "points_in_gt_32": int(c[c > 32].sum()), "leaves_gt_cap": int((c > CAP).sum())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", help="liblsdreg.so to load instead of the package's")
    ap.add_argument("--repeats", type=int, default=20)
    ap.add_argument("--scans", type=int, default=23)
    ap.add_argument("--out")
    a = ap.parse_args()
    if a.lib:
        lsdreg.capi.lib = lsdreg.capi.load_library(os.path.abspath(a.lib))
        lsdreg.lib = lsdreg.capi.lib
    lib = lsdreg.capi.lib
    lsdreg.init(0)
    dev = torch.device("cuda", 0)
    vg = lsdreg.VoxelGrid(max_points=131072)
    per_kernel, spans, host_us, stats, missed, launches_per_call = {}, [], [], [], [], 0
    out = torch.empty((131072, 4), dtype=torch.float32, device=dev)
    m = torch.zeros(16, dtype=torch.int32, device=dev)
    for s in range(a.scans):
        scan = np.ascontiguousarray(np.asarray(bench.make_step(s)[0], np.float32))
        stats.append(leaf_stats(scan))
        x = torch.from_numpy(scan).to(dev)

        def call():
            st = lib.lsd_voxelgrid_filter_dev(vg.h, C.c_void_p(x.data_ptr()), x.shape[0], C.c_float(0.5), C.c_void_p(out.data_ptr()),
                                              C.c_void_p(m.data_ptr()))
            lsdreg.capi.check(st)
        for _ in range(3):
            call()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(a.repeats):
            call()
        torch.cuda.synchronize()
        host_us.append(1e6 * (time.perf_counter() - t0) / a.repeats)
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(a.repeats):
                call()
            torch.cuda.synchronize()
        with tempfile.TemporaryDirectory() as td:
            path = os.path.join(td, "t.json")
            prof.export_chrome_trace(path)
            ev = [e for e in json.load(open(path))["traceEvents"] if e.get("cat") == "kernel"]
        ev.sort(key=lambda e: e["ts"])
        calls, kern = [], {}
        for e in ev:
            name = e["name"].split("(")[0].split("<")[0].replace("void ", "").replace("lsd::", "")
            if name == "vg_minmax_kernel":
                calls.append([e["ts"], e["ts"] + e["dur"], 0])
            if calls:
                calls[-1][1] = e["ts"] + e["dur"]
                calls[-1][2] += 1
            kern.setdefault(name, []).append(e["dur"])
        if not calls:      # nothing traced for this scan (the profiler returned no kernel events): reported, not guessed
            missed.append(s)
            continue
        spans.append(statistics.median(c[1] - c[0] for c in calls))
        for k, v in kern.items():
            per_kernel.setdefault(k, []).append(statistics.median(v))
        launches_per_call = statistics.median(c[2] for c in calls)
    res = {"tool": "vg_probe", "lib": a.lib or "package", "gpu": torch.cuda.get_device_name(0), "scans": a.scans, "repeats": a.repeats,
           "scans_not_traced": missed, "launches_per_call": launches_per_call,
           "span_us_median": round(statistics.median(spans), 2), "span_us_max": round(max(spans), 2),
           "host_us_per_call_median": round(statistics.median(host_us), 2),
           "kernels_us_median": {k: round(statistics.median(v), 2) for k, v in per_kernel.items()},
           "kernels_us_max": {k: round(max(v), 2) for k, v in per_kernel.items()},
           "leaf_stats": {k: [st[k] for st in stats] for k in stats[0]}}
    print(json.dumps(res), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            f.write(json.dumps(res) + "\n")


if __name__ == "__main__":
    main()
