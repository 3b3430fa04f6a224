"""Bit identity of the matcher and the loop detector between two builds of the library (same C ABI).

    python tools/reg_ab.py OUT.npz [--lib path/to/liblsdreg_variant.so] [--small]
    python tools/reg_ab.py --compare A.npz B.npz [--loose KEY_REGEX]

Runs seeded synth scenes through every matcher entry point and writes every result to one .npz:
NDT with 1 / 7 / 27 neighbours, GICP with a source below and one above the thread-shape switch (16 384 points), VGICP with
1 and 7 neighbours; for each, cost with update + derivatives at two poses, then error only, the correspondences, n_voxels,
align (pose, H, flags, iteration log) and fitness at 25 and 0.25.  Then LoopDetector.match over mixed cloud sizes, detect and
fitness(DBL_MAX).  --small uses 16-beam scans of a few thousand points (for the SIMT emulator build, tests/simt; both GICP
sources then sit below the switch).  --compare asserts np.array_equal on every array; keys matching --loose are compared
at rtol 1e-9 instead (results that come from double atomicAdd sums, which need not repeat bit for bit on the GPU)."""
import os
import re
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def opt(name, default):
    return sys.argv[sys.argv.index(name) + 1] if name in sys.argv else default


def compare(a, b):
    A, B = np.load(a), np.load(b)
    loose = re.compile(opt("--loose", "^$"))
    bad = sorted(set(A.files) ^ set(B.files))
    for k in sorted(set(A.files) & set(B.files)):
        x, y = A[k], B[k]
        same = x.shape == y.shape and (np.allclose(x, y, rtol=1e-9, atol=0) if loose.search(k) else np.array_equal(x, y))
        if not same:
            bad.append(k)
    print(f"{len(A.files)} arrays, {len(bad)} differ" + (": " + " ".join(bad) if bad else ""))
    return not bad


def run(out):
    import lsdreg
    from lsdreg import synth
    if "--lib" in sys.argv:
        lsdreg.capi.lib = lsdreg.capi.load_library(os.path.abspath(opt("--lib", "")))
        lsdreg.lib = lsdreg.capi.lib
    lsdreg.init(0)
    small = "--small" in sys.argv
    beams = 16 if small else 64
    c0 = synth.block_center(0, 0)
    R0 = synth.rot_from_rpy(0.0, 0.0, 0.3)
    tgt = synth.scan64(11, 300 if small else 400, R0, c0, n_beams=beams)
    src_lo = synth.scan64(12, 150 if small else 200, R0, c0 + np.array([0.4, -0.2, 0.0]), n_beams=beams)
    src_hi = synth.scan64(13, 200 if small else 400, R0, c0 + np.array([0.4, -0.2, 0.0]), n_beams=beams)
    dR, dt = synth.perturb(3)
    guess = np.eye(4); guess[:3, :3] = dR; guess[:3, 3] = dt
    poses = [guess, np.eye(4)]
    res = {}
    cases = [("ndt1", "NDT_CUDA", dict(ndt_neighbors=1), src_lo), ("ndt7", "NDT_CUDA", {}, src_lo),
             ("ndt27", "NDT_CUDA", dict(ndt_neighbors=27), src_lo), ("gicp_lo", "FAST_GICP", {}, src_lo),
             ("gicp_hi", "FAST_GICP", {}, src_hi), ("vgicp1", "FAST_VGICP", {}, src_lo),
             ("vgicp7", "FAST_VGICP", dict(ndt_neighbors=7), src_lo)]
    for name, kind, kw, src in cases:
        m = lsdreg.Matcher(kind, **kw)
        m.set_target(tgt); m.set_source(src)
        for j, T in enumerate(poses):
            e, H, b, nc = m.cost(T, update=True, deriv=True)
            res.update({f"{name}/cost{j}/err": e, f"{name}/cost{j}/H": H, f"{name}/cost{j}/b": b, f"{name}/cost{j}/n": nc})
        e, _, _, nc = m.cost(guess, update=False, deriv=False)
        res.update({f"{name}/err_only": e, f"{name}/err_only_n": nc, f"{name}/corr": m.correspondences(),
                    f"{name}/n_voxels": m.stats()["n_voxels"]})
        T32 = m.align(guess.astype(np.float32))
        T, H = m.final()
        res.update({f"{name}/align32": T32, f"{name}/align": T, f"{name}/align_H": H, f"{name}/converged": m.converged,
                    f"{name}/iterations": m.iterations, f"{name}/iter_log": m.iteration_log(),
                    f"{name}/fit25": m.fitness(25.0), f"{name}/fit025": m.fitness(0.25)})
        m.close()
    # loop detector: key frames on a short arc, mixed sizes (both fitness shapes unless --small)
    d = lsdreg.LoopDetector()
    est = []
    for i in range(6):
        th = 0.15 * i
        R = synth.rot_from_rpy(0.0, 0.0, th + np.pi / 2)
        t = c0 + np.array([6.0 * np.cos(th), 6.0 * np.sin(th), 0.0])
        d.add_keyframe(synth.scan64(100 + i, (150, 200, 300)[i % 3] if small else (200, 250, 400)[i % 3], R, t, n_beams=beams),
                       30.0 * i)
        T = np.eye(4); T[:3, :3] = synth.rot_from_rpy(0.0, 0.0, 0.02 * i) @ R; T[:3, 3] = t + 0.1 * i
        est.append(T)
    est = np.array(est)
    cands = [0, 1, 2, 3, 4]
    guesses = np.array([np.linalg.inv(est[5]) @ est[k] for k in cands])
    mt = d.match(5, cands, guesses)
    for k in ("final", "converged", "iterations", "fitness"):
        res[f"loop/match/{k}"] = mt[k]
    for i, lg in enumerate(mt["iteration_logs"]):
        res[f"loop/match/iter_log{i}"] = lg
    loops = d.detect(est, [0, 1, 2, 3], [5])
    res["loop/detect/n"] = len(loops)
    for i, lp in enumerate(loops):
        for k in ("key1", "key2", "relpose", "coarse_score", "score", "information"):
            res[f"loop/detect/{i}/{k}"] = lp[k]
    res["loop/reports"] = np.array([[r["decision"], r["n_candidates"], r["best_slot"], r["best_score"]] for r in d.reports()])
    res["loop/fitness_max"] = np.array(d.fitness(5, 2, guesses[2].astype(np.float32)))
    d.close()
    np.savez(out, **{k: np.asarray(v) for k, v in res.items()})
    print(f"wrote {len(res)} arrays to {out}")


if __name__ == "__main__":
    if "--compare" in sys.argv:
        i = sys.argv.index("--compare")
        sys.exit(0 if compare(sys.argv[i + 1], sys.argv[i + 2]) else 1)
    run(sys.argv[1])
