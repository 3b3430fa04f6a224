"""Cost of the whole-target scan that GICP takes on a target whose point map refused points, beside an ordinary pair.

    python tools/gicp_fallback_probe.py OUT.json [--lib-b path/to/other/liblsdreg.so] [--reps R]

Two pairs of 64-beam synth scans 0.5 m apart (source ~19 k points: the thread-per-point search shape; a second, every
4th point, for the warp shape): the ordinary pair, and the same pair with a 3000-point blob in one voxel 1 m from the
target's sensor (a wall beside the sensor: that voxel overflows the map's 896 points, so every correspondence update
scans the whole target).  For each pair and library: the host time of set_target + set_source and of align() from a
perturbed guess (align ends in a device synchronise), the iterations, and the final pose.  With --lib-b the two builds
alternate rep by rep in one process; the ordinary pair must give the same pose bits from both."""
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def opt(name, default):
    return sys.argv[sys.argv.index(name) + 1] if name in sys.argv else default


def scenes():
    from lsdreg import synth
    c0 = synth.block_center(0, 0)
    R = synth.rot_from_rpy(0.0, 0.0, 0.4)
    tgt = synth.scan64(31, 250, R, c0)
    src = synth.scan64(32, 300, R, c0 + np.array([0.5, 0.0, 0.0]))
    rng = np.random.default_rng(3)
    blob = np.zeros((3000, tgt.shape[1]), np.float32)
    blob[:, :3] = rng.uniform(-0.2, 0.2, (3000, 3)) + [1.0, 0.0, 0.0]
    guess = np.eye(4, dtype=np.float32)
    guess[0, 3] = -0.4
    return {"ordinary": (tgt, src), "overfull": (np.concatenate([tgt, blob]), src)}, guess


def run(capi, lib, tgt, src, guess):
    import lsdreg
    capi.lib = lib
    t0 = time.perf_counter()
    g = lsdreg.Matcher("FAST_GICP")
    g.set_target(tgt); g.set_source(src)
    t1 = time.perf_counter()
    out = g.align(guess)
    t2 = time.perf_counter()
    it = g.iterations
    g.close()
    return t1 - t0, t2 - t1, it, out


def main():
    import lsdreg
    from lsdreg import capi
    libs = {"a": capi.lib}
    if "--lib-b" in sys.argv:
        libs["b"] = capi.load_library(os.path.abspath(opt("--lib-b", "")))
    reps = int(opt("--reps", "7"))
    sc, guess = scenes()
    pairs = {}
    for name, (tgt, src) in sc.items():
        pairs[name + "/thread"] = (tgt, src)
        pairs[name + "/warp"] = (tgt, np.ascontiguousarray(src[::4]))
    res = {}
    for key, (tgt, src) in pairs.items():
        for ln, lib in libs.items():
            run(capi, lib, tgt, src, guess)                      # warm-up: module load, allocations
        rows = {ln: [] for ln in libs}
        for _ in range(reps):
            for ln, lib in libs.items():                         # alternate the builds
                rows[ln].append(run(capi, lib, tgt, src, guess))
        for ln, r in rows.items():
            poses = [x[3] for x in r]
            res[f"{key}/{ln}"] = dict(n_tgt=int(tgt.shape[0]), n_src=int(src.shape[0]),
                                      set_ms=float(np.median([x[0] for x in r]) * 1e3),
                                      align_ms=float(np.median([x[1] for x in r]) * 1e3),
                                      align_ms_min=float(np.min([x[1] for x in r]) * 1e3),
                                      align_ms_max=float(np.max([x[1] for x in r]) * 1e3),
                                      iterations=int(r[0][2]), same_pose_every_rep=bool(all(np.array_equal(p, poses[0]) for p in poses)),
                                      pose=poses[0].tolist())
        if "b" in libs:
            res[f"{key}/same_pose_a_b"] = bool(np.array_equal(res[f"{key}/a"]["pose"], res[f"{key}/b"]["pose"]))
    capi.lib = libs["a"]
    try:
        res["gpu"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                    capture_output=True, text=True).stdout.strip()
    except OSError:
        res["gpu"] = "unknown"
    with open(sys.argv[1], "w") as f:
        json.dump(res, f, indent=1)
    for k, v in res.items():
        print(k, {kk: vv for kk, vv in v.items() if kk != "pose"} if isinstance(v, dict) else v)


if __name__ == "__main__":
    main()
