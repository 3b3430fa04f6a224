#!/usr/bin/env python
"""bench_overlap.py — the overlap detector of map merging (lsd_overlap_detect) on one fragment of 10 new key frames against a
loaded map of 100 key frames of ~25 k points, three ways:
  batched    lsd_overlap_detect: every pair's prescreen in one launch, every pair's NDT in one launch per LM round.  Each
             call builds the tables of its new key frames and releases them when it returns, as on a real merge, where
             every fragment is new; only the first call also allocates the buffers, and it is reported apart
  serial     the reference's loop order through the library's single-pair paths: per pair one prescreen launch and an
             lsd_reg NDT_CUDA alignment and getFitnessScore, then one lsd_reg FAST_GICP per new key frame with a best
             candidate; with one NDT handle per new key frame (target set once, as the reference's registration object)
             and with a fresh handle per pair (which also pays a stream, allocations and a target table every pair)
  reference  (when oracle/_ref holds the compiled reference) NDTCuda of the same pairs, one object per new key frame
Median and p95 wall time around the synchronous calls, kernel launches and host round trips of the batched path, and the
card's name and power limit read in the same run.  Prints one JSON object; --out writes it to a file too.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def _pose(R, t):
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = R, t
    return T


def world(n_kf: int, n_new: int, n_az: int):
    from lsdreg import synth
    c0 = synth.block_center(0, 0)
    clouds, poses, ids = [], [], []
    for i in range(n_kf):   # a drive through the block, 1 m apart
        R = synth.rot_from_rpy(0.0, 0.0, 0.02 * i)
        t = c0 + np.array([-0.5 * n_kf + 1.0 * i, 1.0, 0.0])
        clouds.append(synth.scan64(1000 + i, n_az, R, t)); poses.append(_pose(R, t)); ids.append(i)
    new = []
    first = n_kf // 2 - n_new // 2
    for j in range(n_new):  # a second drive beside it, turned
        i = first + j
        R = synth.rot_from_rpy(0.0, 0.0, 0.02 * i + 0.3)
        t = poses[i][:3, 3] + np.array([0.3, -0.5, 0.0])
        new.append(len(clouds)); clouds.append(synth.scan64(5000 + j, n_az, R, t)); poses.append(_pose(R, t)); ids.append(2010 + j)
    edges = [(a, a + 1) for a in range(n_kf - 1)] + [(a, a + 1) for a in range(2000, 2040)]
    return dict(clouds=clouds, poses=np.array(poses), ids=ids, kfs=list(range(n_kf)), new=new, edges=edges)


def gpu_info() -> dict:
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        name, power, clk = [v.strip() for v in r.stdout.splitlines()[0].split(",")]
        return dict(gpu=name, power_limit=power, max_sm_clock=clk)
    except Exception as e:  # noqa: BLE001
        return dict(gpu=f"unknown ({e})")


def stats(ms):
    a = np.array(ms)
    return dict(median_ms=float(np.median(a)), p95_ms=float(np.percentile(a, 95)), reps=len(a))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--keyframes", type=int, default=100)
    ap.add_argument("--new", type=int, default=10)
    ap.add_argument("--n-az", type=int, default=400)          # x 64 beams: ~25 k points per key frame
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()

    import lsdreg
    import overlap_oracle as OO
    lsdreg.init(0)
    W = world(a.keyframes, a.new, a.n_az)
    d = lsdreg.OverlapDetector()
    for c, i in zip(W["clouds"], W["ids"]):
        d.add_keyframe(c, i)
    P, kfs, new, edges = W["poses"], W["kfs"], W["new"], W["edges"]

    t0 = time.perf_counter()
    ov = d.detect(P, kfs, new, edges)
    first_ms = (time.perf_counter() - t0) * 1e3   # allocates the target buffers
    reps, st = d.reports(), d.stats()
    batched = []
    for _ in range(a.reps):
        t0 = time.perf_counter()
        d.detect(P, kfs, new, edges)
        batched.append((time.perf_counter() - t0) * 1e3)

    # the serial path over the same candidates
    cands = {ns: list(d.find_candidates(P, kfs, ns, edges)) for ns in new}
    pairs = [(ns, k) for ns in new for k in cands[ns]]

    def serial_once(per_pair: bool):
        """The reference's loop through the library's single-pair paths.  per_pair: a fresh lsd_reg NDT handle (stream,
        allocations, target table) for every pair; else one handle per new key frame whose target is set once, as the
        reference's one registration object does (overlap_merge.hpp:157-166)."""
        launches, trips = 0, 0
        for ns in new:
            best, best_score, rel = None, OO.DBL_MAX, None
            m = None
            for k in cands[ns]:
                g = lsdreg.overlap_guess(P[ns], P[k])
                launches += 1; trips += 1
                if d.fitness(ns, k, g, 1.0)["inlier_ratio"] < 0.2:
                    continue
                if per_pair or m is None:
                    m = lsdreg.Matcher("NDT_CUDA")
                    m.set_target(W["clouds"][ns])
                l0 = m.stats()["launches"]
                m.set_source(W["clouds"][k])
                m.align(g)
                sc = m.fitness(25.0) if m.converged else OO.DBL_MAX
                launches += m.stats()["launches"] - l0; trips += m.stats()["launches"] - l0
                if not m.converged or sc > best_score:
                    continue
                best, best_score, rel = k, sc, m.final()[0].astype(np.float32)
            if best is None:
                continue
            acc = OO.accumulate(W["clouds"], P, W["ids"], kfs, edges, best)
            gm = lsdreg.Matcher("FAST_GICP", max_corr_dist=0.5, transformation_epsilon=0.001)
            gm.set_target(acc); gm.set_source(W["clouds"][ns])
            gm.align(lsdreg.overlap_finetune_guess(rel))
        d.release_targets()   # the prescreen's filtered targets are rebuilt on every repetition, as in detect
        return launches, trips

    serial = {}
    for per_pair in (False, True):
        serial_once(per_pair)
        ms = []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            sl, strips = serial_once(per_pair)
            ms.append((time.perf_counter() - t0) * 1e3)
        serial["serial_handle_per_pair" if per_pair else "serial_handle_per_keyframe"] = dict(
            **stats(ms), prescreen_and_ndt_launches=sl, round_trips=strips)

    out = dict(config="overlap_detect", keyframes=a.keyframes, new_keyframes=a.new,
               points_per_keyframe=int(np.mean([len(c) for c in W["clouds"]])), pairs=len(pairs),
               decisions=[r["decision"] for r in reps], overlaps=len(ov),
               batched=dict(**stats(batched), first_call_ms=first_ms, launches=st["launches"], ndt_round_trips=st["rounds"],
                            target_buffers=st["target_buffers"]),
               **serial, **gpu_info())
    try:
        from oracle.reg import RefNdtCuda
        ref = []
        for _ in range(max(2, a.reps // 2)):
            t0 = time.perf_counter()
            for ns in new:
                r = RefNdtCuda()
                r.set_target(W["clouds"][ns])
                for k in cands[ns]:
                    r.set_source(W["clouds"][k])
                    r.align(lsdreg.overlap_guess(P[ns], P[k]).astype(np.float64))
            ref.append((time.perf_counter() - t0) * 1e3)
        out["reference_ndt_pairs"] = stats(ref)
    except Exception as e:  # noqa: BLE001  (oracle/_ref absent: not measured)
        out["reference_ndt_pairs"] = f"not measured: {type(e).__name__}: {e}"
    line = json.dumps(out)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
