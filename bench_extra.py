#!/usr/bin/env python
"""bench_extra.py — the other BASELINE.json configs (parity-test cases, not the headline bench line):
  config[2]  NDT scan-to-map: 100 k-pt scan vs a 50 M-pt map voxelised at 0.5 m
  config[3]  GICP loop-closure batch: submap pairs x 200 k pts (per-GPU share of the 256-pair batch)
  config[4]  detection voxelizer: 200 k pts, 4-frame window
  loop       loop-closure detection: one new key frame vs C candidates (C = 4, 16, 32), ~30 k pts each
  galign     global-alignment closure search: 72 reference x 100 new key frames, ~13 k pts each, hundreds of pairs
  floor      floor detection, mapping preset, on ~100 k-return scans (device and host input)
Prints one JSON object per config with device times (CUDA events via torch on the default stream are
NOT used: the library runs on its own stream, so wall time around synchronous C-ABI calls is reported)
and the CPU restatement timed on a bounded sample.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

os.environ.setdefault("NCCL_DEBUG_FILE", "/dev/stderr")


class _QuietStdout:
    """Route fd 1 to stderr while libraries may chat (NCCL prints its version banner with printf at the first
    communicator), and give it back for the one JSON line: stdout must carry nothing else."""

    def __enter__(self):
        sys.stdout.flush()
        self.saved = os.dup(1)
        os.dup2(2, 1)
        return self

    def __exit__(self, *exc):
        sys.stdout.flush()
        os.dup2(self.saved, 1)
        os.close(self.saved)
        return False


ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)


def t_ms(f, n=1):
    t0 = time.perf_counter()
    for _ in range(n):
        r = f()
    return (time.perf_counter() - t0) * 1e3 / n, r


def ndt(args):
    import lsdreg
    from lsdreg import synth
    from oracle.reg import OracleMatcher
    if int(os.environ.get("WORLD_SIZE", 1)) > 1:
        return ndt_sharded(args)
    bx = args.ndt_blocks
    t0 = time.time()
    m = synth.block_map(31, bx, bx, 0.25 * (240711 * bx * bx / args.ndt_points) ** 0.5)
    gen_s = time.time() - t0
    bi = bx // 2
    Rgt = synth.rot_from_rpy(0.01, -0.02, 0.3)
    tgt = synth.block_center(bi, bi) + np.array([1.0, -2.0, 0.0])
    scan = synth.scan64(32, 1920, Rgt, tgt, bi, bi)
    dR, dt = synth.perturb(33, 0.5, 3.0)
    guess = np.eye(4); guess[:3, :3] = Rgt @ dR; guess[:3, 3] = tgt + dt
    g = lsdreg.Matcher("NDT_CUDA", resolution=0.5, map_log2_lines=25)
    build_ms, _ = t_ms(lambda: g.set_target(m))
    src_ms, _ = t_ms(lambda: g.set_source(scan))
    g.align(guess)
    align_ms, T = t_ms(lambda: g.align(guess), 5)
    Tg, _ = g.final()
    cost_ms, _ = t_ms(lambda: g.cost(Tg), 20)
    st = g.stats()
    out = dict(config="NDT 100k vs %.1fM-pt map @0.5 m" % (m.shape[0] / 1e6), map_points=int(m.shape[0]), voxels=st["n_voxels"],
               scan_points=int(scan.shape[0]), target_build_ms=build_ms, set_source_ms=src_ms, align_ms=align_ms,
               iterations=g.iterations, converged=bool(g.converged), cost_eval_us=cost_ms * 1e3,
               pos_err_m=float(np.abs(Tg[:3, 3] - tgt).max()), map_gen_s=gen_s,
               last_steps_m_deg=[[float("%.3g" % v) for v in row[:2]] for row in g.iteration_log()[-6:]],   # what is_converged saw (eps 0.01 m / 0.1 deg)
               alg_bytes_per_eval=float(scan.shape[0] * (16 + 7 * 16 + 3 * 52)),
               cost_gbs=float(scan.shape[0] * (16 + 7 * 16 + 3 * 52) / (cost_ms * 1e-3) / 1e9))
    if not args.no_ref_cuda and os.path.exists(os.path.join(ROOT, "oracle", "_ref", "libref_cuda.so")):
        # the reference's own CUDA NDT (NDTCudaCore + kernels, recompiled for sm_90a) on the same clouds, same GPU
        try:
            from oracle.reg import RefNdtCuda
            r = RefNdtCuda(0.5, 7)
            rb, _ = t_ms(lambda: r.set_target(m)); rs, _ = t_ms(lambda: r.set_source(scan))
            r.align(guess)
            ra, Tr = t_ms(lambda: r.align(guess), 3)
            r.linearize(Tg)
            rl, _ = t_ms(lambda: r.linearize(Tg), 10)
            out["reference_cuda_sm90a"] = dict(target_build_ms=rb, set_source_ms=rs, align_ms=ra, cost_eval_us=rl * 1e3, voxels=int(r.n_voxels),
                                                converged=bool(r.converged), pos_err_m=float(np.abs(Tr[:3, 3] - tgt).max()))
            del r
        except Exception as e:  # the comparator must never take the measurement down
            out["reference_cuda_sm90a"] = dict(error=repr(e)[:200])
    if not args.no_cpu:
        near = (np.abs(m[:, 0] - tgt[0]) < 130) & (np.abs(m[:, 1] - tgt[1]) < 130)
        sub = np.ascontiguousarray(m[near])             # bounded CPU sample: the map within 130 m of the scan, full density
        o = OracleMatcher("ndt", resolution=0.5)
        cb, _ = t_ms(lambda: o.set_target(sub)); o.set_source(scan)
        ca, _ = t_ms(lambda: o.align(guess))
        out["cpu"] = dict(kind="port", cores=1, sample="same scan vs the %d map points within 130 m of it" % sub.shape[0], target_build_ms=cb, align_ms=ca,
                          iterations=o.iterations)
    print(json.dumps(out))


def ndt_sharded(args):
    """Config 3 on N GPUs (SURVEY.md section 8e row C3): the 50 M-point map voxelised per x-y tile on its owner GPU (every rank
    uploads only the points of its own tiles), every rank holds the scan, [H, b, err] all-reduced inside the cost kernel
    through peer memory.  Reports the same fields as the 1-GPU leg plus the 1-GPU align on rank 0's GPU for comparison."""
    import torch
    import torch.distributed as dist
    import lsdreg
    from lsdreg import shard, synth
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    bx = args.ndt_blocks
    m = synth.block_map(31, bx, bx, 0.25 * (240711 * bx * bx / args.ndt_points) ** 0.5)
    bi = bx // 2
    Rgt = synth.rot_from_rpy(0.01, -0.02, 0.3)
    tgt = synth.block_center(bi, bi) + np.array([1.0, -2.0, 0.0])
    scan = synth.scan64(32, 1920, Rgt, tgt, bi, bi)
    dR, dt = synth.perturb(33, 0.5, 3.0)
    guess = np.eye(4); guess[:3, :3] = Rgt @ dR; guess[:3, 3] = tgt + dt
    TILE = 64                                              # 32 m tiles at 0.5 m voxels
    g = lsdreg.Matcher("NDT_CUDA", resolution=0.5, map_log2_lines=25 if world <= 2 else 24)
    blob = torch.from_numpy(g.shard_export(rank, world, TILE)).cuda()
    blobs = [torch.empty_like(blob) for _ in range(world)]
    dist.all_gather(blobs, blob)
    g.shard_connect(np.stack([b.cpu().numpy() for b in blobs]))
    # host-side ownership (mirrors ndt_coord + tile_owner): upload only this rank's tiles
    c = np.floor(m[:, :2] / np.float32(0.5) - np.float32(0.5)).astype(np.int32)
    mine = np.ascontiguousarray(m[shard.tile_owner(c[:, 0], c[:, 1], TILE, world) == rank])
    dist.barrier()
    build_ms, _ = t_ms(lambda: g.set_target(mine))
    g.set_source(scan)
    dist.barrier()
    g.align(guess)
    dist.barrier()
    t0 = time.perf_counter()
    for _ in range(5):
        g.align(guess)
    torch.cuda.synchronize()
    align_ms = (time.perf_counter() - t0) * 1e3 / 5
    Tg, _ = g.final()
    dist.barrier()
    t0 = time.perf_counter()
    for _ in range(20):
        g.cost(Tg)
    cost_us = (time.perf_counter() - t0) * 1e6 / 20
    st = g.stats()
    t = torch.tensor([build_ms, align_ms, cost_us, float(st["n_voxels"]), float(mine.shape[0])], dtype=torch.float64, device="cuda")
    tmax = t.clone(); dist.all_reduce(tmax, op=dist.ReduceOp.MAX)
    tsum = t.clone(); dist.all_reduce(tsum, op=dist.ReduceOp.SUM)
    poses = [torch.empty(16, dtype=torch.float64, device="cuda") for _ in range(world)]
    dist.all_gather(poses, torch.from_numpy(Tg.reshape(-1)).cuda())
    if rank == 0:
        out = dict(config="NDT 100k vs %.1fM-pt map @0.5 m, target tile-sharded over %d GPUs" % (m.shape[0] / 1e6, world), n_gpus=world,
                   map_points=int(m.shape[0]), voxels_total=int(tsum[3]), voxels_this_rank=st["n_voxels"], points_uploaded_max=int(tmax[4]),
                   scan_points=int(scan.shape[0]), target_build_ms=float(tmax[0]), align_ms=float(tmax[1]), cost_eval_us=float(tmax[2]),
                   iterations=g.iterations, converged=bool(g.converged), pos_err_m=float(np.abs(Tg[:3, 3] - tgt).max()),
                   ranks_bit_identical=bool(all(torch.equal(poses[0], p) for p in poses[1:])),
                   collective="28 doubles all-reduced per cost evaluation inside ndt_cost_kernel (peer-memory inbox, rank-ordered fold)")
        # the unsharded matcher on this rank's GPU, same clouds: what one GPU does alone
        one = lsdreg.Matcher("NDT_CUDA", resolution=0.5, map_log2_lines=25)
        b1, _ = t_ms(lambda: one.set_target(m)); one.set_source(scan); one.align(guess)
        a1, _ = t_ms(lambda: one.align(guess), 5)
        T1, _ = one.final()
        c1, _ = t_ms(lambda: one.cost(T1), 20)
        out["one_gpu"] = dict(target_build_ms=b1, align_ms=a1, cost_eval_us=c1 * 1e3, iterations=one.iterations, converged=bool(one.converged),
                              pose_diff_vs_sharded_m=float(np.abs(T1[:3, 3] - Tg[:3, 3]).max()))
        print(json.dumps(out))
    dist.barrier()
    dist.destroy_process_group()


def gicp(args):
    """Config 4: a batch of loop-closure pairs.  Pairs are independent, so with N ranks (torchrun) rank r takes pairs
    r, r+N, ... — no collective on the data path; the wall time is the max over ranks."""
    import lsdreg
    from lsdreg import synth
    from oracle.reg import OracleMatcher
    rank = int(os.environ.get("RANK", 0)); world = int(os.environ.get("WORLD_SIZE", 1))
    dist = None
    if world > 1:
        import torch
        import torch.distributed as dist
        torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", 0)))
        dist.init_process_group("nccl", device_id=torch.device("cuda", int(os.environ.get("LOCAL_RANK", 0))))
    pairs = args.gicp_pairs
    method = args.gicp_method
    g = lsdreg.Matcher(method, max_corr_dist=2.0)
    distinct = min(4, max(1, pairs // world))
    data = []
    for d in range(distinct):                                 # a few distinct pairs per rank, cycled: the work per pair is the same
        p = rank * distinct + d
        m = synth.block_map(41 + p, 1, 1, 0.22)
        m = np.ascontiguousarray(m[np.linspace(0, m.shape[0] - 1, 200000).astype(np.int64)]) if m.shape[0] > 200000 else m
        Rgt = synth.rot_from_rpy(0.0, 0.0, 0.2 + 0.01 * p)
        tgt = synth.block_center(0, 0) + np.array([1.0 + 0.3 * (p % 7), -2.0, 0.0])
        src = synth.scan64(50 + p, 3800, Rgt, tgt)            # a dense submap seen from the unknown pose
        src = np.ascontiguousarray(src[np.linspace(0, src.shape[0] - 1, 200000).astype(np.int64)]) if src.shape[0] > 200000 else src
        dR, dt = synth.perturb(60 + p, args.gicp_perturb_m, args.gicp_perturb_deg)   # SURVEY.md section 8d: guess perturbed by <= 1 m, <= 5 deg
        guess = np.eye(4); guess[:3, :3] = Rgt @ dR; guess[:3, 3] = tgt + dt
        data.append((m, src, guess, tgt))
    g.set_target(data[0][0]); g.set_source(data[0][1]); g.align(data[0][2])    # warm-up
    times, errs, its, build = [], [], [], []
    if dist is not None:
        dist.barrier()
    t_all = time.perf_counter()
    for q in range(rank, pairs, world):
        m, src, guess, tgt = data[(q // world) % distinct]
        b1, _ = t_ms(lambda: g.set_target(m)); b2, _ = t_ms(lambda: g.set_source(src))
        a, T = t_ms(lambda: g.align(guess))
        Tg, _ = g.final()
        build.append(b1 + b2); times.append(a); its.append(g.iterations); errs.append(float(np.abs(Tg[:3, 3] - tgt).max()))
    wall = time.perf_counter() - t_all
    if dist is not None:
        import torch
        t = torch.tensor([wall, max(errs)], dtype=torch.float64, device="cuda")
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        wall, err_max = float(t[0]), float(t[1])
    else:
        err_max = max(errs)
    if rank == 0:
        out = dict(config="%s pairs x 200k pts" % method, pairs=pairs, n_gpus=world, points_per_cloud=200000,
                   covariance_build_ms=float(np.mean(build)), align_ms=float(np.mean(times)), pairs_per_s=pairs / wall,
                   guess_perturbation="<= %.1f m, <= %.1f deg" % (args.gicp_perturb_m, args.gicp_perturb_deg),
                   wall_s=wall, iterations=float(np.mean(its)), pos_err_m=err_max,
                   note="host clouds in, H2D + index build + covariances + align inside the timed region; rank r takes pairs r, r+N, ...")
        if (method == "FAST_VGICP" and world == 1 and not args.no_ref_cuda
                and os.path.exists(os.path.join(ROOT, "oracle", "_ref", "libref_cuda_vgicp.so"))):
            # the reference's own CUDA VGICP (FastVGICPCuda + FastVGICPCudaCore, recompiled for sm_90a; "FAST_VGICP_CUDA",
            # registrations.cpp:43-55: neighbours from its CPU k-d tree, covariances / voxel map / LM loop on the GPU), same pair
            try:
                from oracle.reg import RefVgicpCuda
                m, src, guess, tgt = data[-1]
                r = RefVgicpCuda(1.0, 64, 0.01, 0)
                rb, _ = t_ms(lambda: (r.set_target(m), r.set_source(src)))
                r.align(guess)
                ra, Tr = t_ms(lambda: r.align(guess), 3)
                out["reference_cuda_sm90a"] = dict(method="FAST_VGICP_CUDA", covariance_build_ms=rb, align_ms=ra, converged=bool(r.converged),
                                                    pos_err_m=float(np.abs(Tr[:3, 3] - tgt).max()),
                                                    note="first run on hardware pending (compiled after round 1's GPU budget was spent)")
                del r
            except Exception as e:  # the comparator must never take the measurement down
                out["reference_cuda_sm90a"] = dict(error=repr(e)[:200])
        if not args.no_cpu and world == 1:
            m, src, guess, tgt = data[-1]
            from oracle import oracle as O
            if O.HAVE_REF_REG:      # the reference's own classes (fast_gicp::FastGICP / FastVGICP compiled unmodified, oracle/_ref/libref_reg.so)
                from oracle.reg import RefMatcher
                nt = 4              # registrations.cpp:36,59: setNumThreads(4)
                o = RefMatcher("gicp", nthreads=nt) if method == "FAST_GICP" else RefMatcher("vgicp", neighbors=1, trans_eps=0.1, rot_eps=0.1, nthreads=nt)
                cb, _ = t_ms(lambda: (o.set_target(m), o.set_source(src)))
                ca, To = t_ms(lambda: o.align(guess))
                out["cpu"] = dict(kind="reference", cores=nt, sample="one pair", covariance_build_ms=cb, align_ms=ca, pairs_per_s=1e3 / (cb + ca),
                                  converged=bool(o.converged), pos_err_m=float(np.abs(To[:3, 3] - tgt).max()),
                                  what="fast_gicp::%s compiled unmodified, 4 OpenMP threads (the reference's setting)" % ("FastGICP" if method == "FAST_GICP" else "FastVGICP"))
            else:
                o = (OracleMatcher("gicp", nthreads=min(16, os.cpu_count() or 1)) if method == "FAST_GICP" else
                     OracleMatcher("vgicp", neighbors=1, trans_eps=0.1, rot_eps=0.1, nthreads=min(16, os.cpu_count() or 1)))
                cb, _ = t_ms(lambda: (o.set_target(m), o.set_source(src)))
                ca, _ = t_ms(lambda: o.align(guess))
                out["cpu"] = dict(kind="port", cores=min(16, os.cpu_count() or 1), sample="one pair", covariance_build_ms=cb, align_ms=ca,
                                  iterations=o.iterations, pos_err_m=float(np.abs(o.final[:3, 3] - tgt).max()))
        print(json.dumps(out))
    if dist is not None:
        dist.destroy_process_group()


def vfe(args):
    import lsdreg
    from lsdreg import synth
    from oracle.vfe import OracleVoxelizer
    frames = []
    for f in range(8):
        s = synth.scan64(300 + f, 800, synth.rot_from_rpy(0, 0, 0.05 * f), synth.block_center(0, 0) + np.array([0.8 * f, 0.1 * f, 0.0]))[:50000]
        p = np.zeros((s.shape[0], 5), np.float32); p[:, :4] = s; p[:, 2] -= 1.8
        frames.append(p)
    M = np.eye(4, dtype=np.float32); M[:3, 3] = [0.8, 0.1, 0.0]
    res = {}
    for mode in (1, 0):   # 1 = voxel ids in atomic order (the reference kernels' contract, 2 kernels); 0 = deterministic ids (3 kernels)
        g = lsdreg.Voxelizer(max_frame_num=4, unordered_ids=mode)
        for f in range(4):
            g.accumulate(frames[f], M)
        acc, vox = [], []
        for f in range(4, 8):
            a, tot = t_ms(lambda: g.accumulate(frames[f], M))
            v, r = t_ms(lambda: g.voxelize(True))
            acc.append(a); vox.append(v)
        res[mode] = (float(np.mean(acc)) * 1e3, float(np.mean(vox)) * 1e3, r[0].shape[0], tot)
        g.close()
    acc, vox = [res[1][0] / 1e3], [res[1][1] / 1e3]
    V, tot = res[1][2], res[1][3]
    out = dict(config="VFE voxelizer 4 x 50k pts", window_points=int(tot), voxels=int(V), accumulate_us=float(np.mean(acc)) * 1e3,
               voxelize_us=float(np.mean(vox)) * 1e3, ids="atomic order (the reference's contract)",
               deterministic_ids=dict(accumulate_us=res[0][0], voxelize_us=res[0][1]),
               alg_bytes=float(20 * tot + 16 * tot + V * 26), gbs=float((20 * tot + 16 * tot + V * 26) / (np.mean(vox) * 1e-3) / 1e9))
    if not args.no_cpu:
        o = OracleVoxelizer(max_frames=4)
        for f in range(4):
            o.accumulate(frames[f], M)
        ca, _ = t_ms(lambda: o.accumulate(frames[4], M)); cv, _ = t_ms(lambda: o.voxelize())
        out["cpu"] = dict(kind="port", cores=1, sample="one frame", accumulate_us=ca * 1e3, voxelize_us=cv * 1e3)
    print(json.dumps(out))


def _card():
    """Card name and power limit, read in the same run (both are part of any number measured on it)."""
    import subprocess
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=20).stdout.strip().splitlines()
        name, pl = [x.strip() for x in q[int(os.environ.get("LOCAL_RANK", 0))].split(",")]
        return dict(card=name, power_limit=pl)
    except Exception as e:  # the measurement does not depend on it
        return dict(card="unknown", power_limit="unknown (%s)" % repr(e)[:80])


def loop(args):
    """LoopDetector on one new key frame and C candidates: batched (lsd_loop_detect / lsd_loop_match) against the per-pair
    lsd_reg loop a user writes without it, and the reference's own CUDA NDT run candidate after candidate where built."""
    import lsdreg
    from lsdreg import synth
    c0 = synth.block_center(0, 0)
    card = _card()
    for C in (4, 16, 32):
        clouds, poses, accum = [], [], []
        for i in range(C):
            th = 2 * np.pi * i / C
            R = synth.rot_from_rpy(0.0, 0.0, th)
            t = c0 + np.array([8.0 * np.cos(th), 8.0 * np.sin(th), 0.0])
            clouds.append(synth.scan64(500 + i, 470, R, t))
            dR, dt = synth.perturb(600 + i, 0.5, 3.0)
            T = np.eye(4); T[:3, :3] = R @ dR; T[:3, 3] = t + dt
            poses.append(T); accum.append(2.0 * i)
        clouds.append(synth.scan64(499, 470, np.eye(3), c0))
        poses.append(np.eye(4)); poses[-1][:3, 3] = c0; accum.append(2.0 * C + 30.0)
        P = np.array(poses)
        new, kfs = C, list(range(C))
        d = lsdreg.LoopDetector()
        for c, a in zip(clouds, accum):
            d.add_keyframe(c, a)
        cand, G = d.find_candidates(P, kfs, new)
        assert len(cand) == C
        # batched: warm up every shape, then time
        d.match(new, cand, G)
        match_ms, m = t_ms(lambda: d.match(new, cand, G), args.loop_reps)
        d.last_edge_accum_distance = 0.0
        d.detect(P, kfs, [new])
        def det():
            d.last_edge_accum_distance = 0.0
            return d.detect(P, kfs, [new])
        detect_ms, loops = t_ms(det, args.loop_reps)
        # serial: one lsd_reg NDT handle, one pair after another (loop_detector.hpp:158-191 written against lsd_reg)
        g = lsdreg.Matcher("NDT_CUDA")
        def serial():
            g.set_target(clouds[new])
            out = []
            for k, gk in zip(cand, G):
                g.set_source(clouds[k])
                g.align(gk.astype(np.float32))
                out.append((g.final()[0], g.converged, g.fitness(25.0)))
            return out
        serial()
        l0 = g.stats()["launches"]
        serial_ms, ser = t_ms(serial, args.loop_reps)
        serial_launches = (g.stats()["launches"] - l0) / args.loop_reps
        same = all(np.array_equal(m["final"][i], ser[i][0]) and bool(m["converged"][i]) == ser[i][1] and m["fitness"][i] == ser[i][2]
                   for i in range(C))
        out = dict(config="loop detection: 1 new key frame vs %d candidates" % C, candidates=C,
                   points_per_keyframe=int(np.mean([c.shape[0] for c in clouds])), **card,
                   batched=dict(detect_ms=detect_ms, match_ms=match_ms, candidates_per_s=C / (match_ms * 1e-3),
                                match_launches=m["launches"], match_round_trips=m["rounds"] + 1, loops_found=len(loops)),
                   serial=dict(ms=serial_ms, candidates_per_s=C / (serial_ms * 1e-3), launches=serial_launches,
                               round_trips=serial_launches),   # every cost / fitness launch of lsd_reg waits for its result
                   batched_equals_serial=bool(same),
                   alg_bytes_per_round=float(sum(c.shape[0] for c in clouds[:C]) * (16 + 7 * (8 + 40))))
        if not args.no_ref_cuda and os.path.exists(os.path.join(ROOT, "oracle", "_ref", "libref_cuda.so")):
            try:
                from oracle.reg import RefNdtCuda
                r = RefNdtCuda(1.0, 7)
                def ref():
                    r.set_target(clouds[new])
                    for k, gk in zip(cand, G):
                        r.set_source(clouds[k]); r.align(gk)
                ref()
                rm, _ = t_ms(ref, args.loop_reps)
                out["reference_cuda_sm90a"] = dict(ms=rm, candidates_per_s=C / (rm * 1e-3))
                del r
            except Exception as e:  # the comparator must never take the measurement down
                out["reference_cuda_sm90a"] = dict(error=repr(e)[:200])
        d.close(); g.close()
        print(json.dumps(out))


def galign(args):
    """Global-alignment closure search: a reference map of R key frames and a new map of M key frames (a second drive around
    the same loop, plus a stretch in another block).  Batched search against the same (new, reference) pairs run serially
    through the single-pair kernels on the same tables (serial = 1), and the compiled reference FastVGICP (CPU) on a subset."""
    import math
    import lsdreg
    from lsdreg import synth
    card = _card()
    c0, c1 = synth.block_center(0, 0), synth.block_center(1, 0)
    R_kf, M_kf, M_other, radius = args.galign_refs, args.galign_news, 4, 14.0
    clouds_ref, clouds_new = [], []
    for i in range(R_kf):
        th = 2 * np.pi * i / R_kf
        clouds_ref.append(synth.scan64(1000 + i, 250, synth.rot_from_rpy(0.0, 0.0, th + np.pi / 2),
                                       c0 + np.array([radius * np.cos(th), radius * np.sin(th), 0.0])))
    for j in range(M_kf):
        th = 2 * np.pi * (j + 0.5) / M_kf
        clouds_new.append(synth.scan64(2000 + j, 250, synth.rot_from_rpy(0.0, 0.0, th - np.pi / 2),
                                       c0 + np.array([(radius + 0.8) * np.cos(th), (radius + 0.8) * np.sin(th), 0.0])))
    for j in range(M_other):
        clouds_new.append(synth.scan64(3000 + j, 250, np.eye(3), c1 + np.array([4.0 * j - 6.0, -5.0, 0.0]), bi=1))
    ga = lsdreg.GlobalAligner()
    refs = [ga.add_keyframe(c, True) for c in clouds_ref]
    news = [ga.add_keyframe(c, False) for c in clouds_new]
    cold_ms, closures = t_ms(lambda: ga.search(news))          # first search: builds every table it uses
    search_ms, closures = t_ms(lambda: ga.search(news), args.galign_reps)
    st = ga.stats()
    tried = ga.matches()
    groups = {}
    for m in tried:
        y = np.float32(-m["sc_yaw"])
        G = np.eye(4)
        G[0, 0] = G[1, 1] = float(np.float32(math.cos(float(y))))
        G[1, 0] = float(np.float32(math.sin(float(y)))); G[0, 1] = -G[1, 0]
        groups.setdefault(m["new_slot"], ([], []))
        groups[m["new_slot"]][0].append(m["ref_slot"]); groups[m["new_slot"]][1].append(G)
    def run(serial):
        return {q: ga.match(q, r, np.array(g), serial=serial) for q, (r, g) in groups.items()}
    run(False)
    per_kf_ms, bat = t_ms(lambda: run(False))
    serial_ms, ser = t_ms(lambda: run(True))
    same = all(all(np.array_equal(bat[q][k], ser[q][k]) for k in ("final", "converged", "iterations", "fitness")) for q in groups)
    pairs = len(tried)
    out = dict(config="global alignment search: %d reference x %d new key frames" % (R_kf, M_kf + M_other), **card,
               reference_keyframes=R_kf, new_keyframes=M_kf + M_other, pairs=pairs, closures=len(closures),
               points_per_keyframe=int(np.mean([c.shape[0] for c in clouds_ref + clouds_new])),
               batched=dict(search_ms=search_ms, first_search_ms=cold_ms, pairs_per_s=pairs / (search_ms * 1e-3), launches=st["launches"],
                            rounds=st["rounds"], batches=st["batches"], per_keyframe_match_ms=per_kf_ms),
               serial=dict(ms=serial_ms, pairs_per_s=pairs / (serial_ms * 1e-3), launches=sum(r["launches"] for r in ser.values()),
                           rounds=sum(r["rounds"] for r in ser.values())),
               batched_equals_serial=bool(same),
               # per round and live pair: source point (16 B) + covariance (32 B) + correspondence (4 B) + Mahalanobis (48 B)
               # + voxel line (128 B) per point, an upper bound reached by the linearising rounds
               alg_bytes_per_round_max=float(sum(clouds_new[m["new_slot"] - R_kf].shape[0] for m in tried) * (16 + 32 + 4 + 48 + 128)))
    if not args.no_cpu and os.path.exists(os.path.join(ROOT, "oracle", "_ref", "libref_reg.so")):
        try:
            from oracle.reg import RefMatcher
            sub = tried[:args.galign_ref_pairs]
            r = RefMatcher("vgicp", resolution=1.0, neighbors=1, max_iterations=64, trans_eps=0.1, rot_eps=0.1, k=20,
                           nthreads=args.galign_ref_threads)
            def ref():
                for m in sub:
                    G = groups[m["new_slot"]][1][groups[m["new_slot"]][0].index(m["ref_slot"])]
                    r.set_target(clouds_ref[m["ref_slot"]]); r.set_source(clouds_new[m["new_slot"] - R_kf])
                    r.align(G); r.fitness(25.0)
            rm, _ = t_ms(ref)
            out["reference_fast_vgicp_cpu"] = dict(pairs=len(sub), threads=args.galign_ref_threads, ms=rm, pairs_per_s=len(sub) / (rm * 1e-3))
        except Exception as e:  # the comparator must never take the measurement down
            out["reference_fast_vgicp_cpu"] = dict(error=repr(e)[:200])
    ga.close()
    print(json.dumps(out))


def floor(args):
    """Floor detection, LSD_FLOOR_MAPPING preset (VoxelGrid 0.2 + distance filter, clip, k = 10 normal filter, RANSAC) on
    BASELINE config[1]-size scans (~100 k returns, sensor 1.8 m above the ground), device-resident and host input.  Device
    kernel time by stage from torch.profiler; the CPU restatement (tests/floor_oracle.py, numpy + scipy) timed by stage,
    labelled as the restatement: PCL itself cannot be built here."""
    import torch
    import lsdreg
    from lsdreg import synth
    card = _card()
    scans = [synth.scan64(500 + i, 1563, synth.rot_from_rpy(0.0, 0.0, 0.4 * i), synth.block_center(0, 0) + np.array([1.5 * i - 3.0, -2.0, 0.0]))
             for i in range(args.floor_scans)]
    det = lsdreg.FloorDetector(lsdreg.FLOOR_MAPPING)
    dev = [torch.from_numpy(s).cuda() for s in scans]
    torch.cuda.synchronize()
    for s in dev:
        det.detect(s)                                   # warm-up: buffers sized
    out = dict(config="floor detection, mapping preset: %d scans x ~%d returns" % (len(scans), int(np.mean([s.shape[0] for s in scans]))), **card)
    for label, inputs in (("device_input", dev), ("host_input", scans)):
        ms, res = [], []
        for _ in range(args.floor_reps):
            for s in inputs:
                t0 = time.perf_counter()
                r = det.detect(s)
                ms.append((time.perf_counter() - t0) * 1e3)
                res.append(r)
        out[label] = dict(frames=len(ms), ms_median=float(np.median(ms)), ms_p95=float(np.percentile(ms, 95)),
                          launches_median=float(np.median([r["launches"] for r in res])),
                          round_trips_median=float(np.median([r["round_trips"] for r in res])),
                          hypotheses_scored_median=float(np.median([r["hypotheses_scored"] for r in res])),
                          iterations_median=float(np.median([r["iterations"] for r in res])),
                          found=int(sum(r["found"] for r in res)),
                          candidates_median=float(np.median([r["n_candidates"] for r in res])),
                          prefiltered_median=float(np.median([r["n_prefiltered"] for r in res])))
    try:   # device time by stage: kernel durations grouped by kernel name
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for s in dev:
                det.detect(s)
        stage_of = lambda n: ("voxelgrid" if n.startswith("vg_") or "vg_" in n else "clip+insert" if "floor_clip" in n  # noqa: E731
                              else "normals" if "normals" in n or "complete" in n else "ransac" if "sample" in n or "score" in n
                              else "compaction" if "compact" in n else "other")
        by = {}
        for e in prof.events():
            if getattr(e, "device_type", None) is not None and str(e.device_type).endswith("CUDA") and ("kernel" in str(getattr(e, "name", "")).lower() or "lsd" in e.name):
                by[stage_of(e.name)] = by.get(stage_of(e.name), 0.0) + e.device_time_total / 1e3
        out["device_kernel_ms_per_frame_by_stage"] = {k: v / len(dev) for k, v in sorted(by.items())}
    except Exception as e:  # the profiler must never take the measurement down
        out["device_kernel_ms_per_frame_by_stage"] = dict(error=repr(e)[:200])
    if not args.no_cpu:
        sys.path.insert(0, os.path.join(ROOT, "tests"))
        import floor_oracle as FO
        p = FO.default_params(FO.MAPPING)
        st = {"prefilter": [], "clip": [], "normals": [], "ransac": []}
        for s in scans:
            t0 = time.perf_counter(); pre = FO.prefilter(s, p)
            t1 = time.perf_counter(); cl = pre[FO.clip_mask(pre, p)]
            t2 = time.perf_counter(); nrm, _, _ = FO.normals(cl[:, :3]); cand = cl[np.abs(FO.normal_nz(nrm)).astype(np.float64) > np.cos(np.pi / 9)]
            t3 = time.perf_counter(); FO.ransac(cand, p["ransac_threshold"]) if cand.shape[0] >= p["floor_pts_thresh"] else None
            t4 = time.perf_counter()
            for k, a, b in (("prefilter", t0, t1), ("clip", t1, t2), ("normals", t2, t3), ("ransac", t3, t4)):
                st[k].append((b - a) * 1e3)
        out["restatement_cpu_ms_median_by_stage"] = {k: float(np.median(v)) for k, v in st.items()}
        out["restatement_cpu_ms_median"] = float(np.median(np.sum([st[k] for k in st], axis=0)))
        out["restatement_note"] = "numpy/scipy restatement of the PCL rules (single process), not PCL"
    det.close()
    print(json.dumps(out))


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--which", default="ndt,gicp,vfe")
    ap.add_argument("--ndt-points", type=float, default=50e6)
    ap.add_argument("--ndt-blocks", type=int, default=10)
    ap.add_argument("--gicp-pairs", type=int, default=4)
    ap.add_argument("--gicp-method", default="FAST_GICP", choices=["FAST_GICP", "FAST_VGICP"])
    ap.add_argument("--gicp-perturb-m", type=float, default=1.0)
    ap.add_argument("--gicp-perturb-deg", type=float, default=5.0)
    ap.add_argument("--loop-reps", type=int, default=5)
    ap.add_argument("--galign-refs", type=int, default=72)
    ap.add_argument("--galign-news", type=int, default=96)
    ap.add_argument("--galign-reps", type=int, default=3)
    ap.add_argument("--galign-ref-pairs", type=int, default=24)
    ap.add_argument("--galign-ref-threads", type=int, default=4, help="FastVGICP threads (setNumThreads(4), registrations.cpp:59)")
    ap.add_argument("--floor-scans", type=int, default=8)
    ap.add_argument("--floor-reps", type=int, default=5)
    ap.add_argument("--no-cpu", action="store_true")
    ap.add_argument("--no-ref-cuda", action="store_true", help="skip the legs that time the reference's own CUDA NDT / VGICP (oracle/_ref/libref_cuda*.so)")
    a = ap.parse_args()
    import contextlib
    import io
    import lsdreg
    buf = io.StringIO()
    with _QuietStdout():
        with contextlib.redirect_stdout(buf):
            lsdreg.init(int(os.environ.get("LOCAL_RANK", 0)))
            for w in a.which.split(","):
                {"ndt": ndt, "gicp": gicp, "vfe": vfe, "loop": loop, "galign": galign, "floor": floor}[w](a)
    sys.stdout.write(buf.getvalue())
    sys.stdout.flush()
