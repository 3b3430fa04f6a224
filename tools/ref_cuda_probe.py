"""Head-to-head on one GPU: the reference's CUDA NDT (recompiled for sm_90a, oracle/_ref/libref_cuda.so) against
liblsdreg, same clouds: agreement of one linearisation and wall time of target build / cost evaluation / align."""
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import lsdreg  # noqa: E402
from lsdreg import synth  # noqa: E402
from oracle.reg import RefNdtCuda  # noqa: E402

lsdreg.init(0)
blocks = int(sys.argv[1]) if len(sys.argv) > 1 else 3
m = synth.block_map(7, blocks, blocks, 0.25)
Rgt = synth.rot_from_rpy(0.01, -0.02, 0.3)
tgt = synth.block_center(blocks // 2, blocks // 2) + np.array([1.0, -2.0, 0.0])
scan = synth.scan64(2, 1563, Rgt, tgt, blocks // 2, blocks // 2)
dR, dt = synth.perturb(5, 0.3, 1.0)
guess = np.eye(4); guess[:3, :3] = Rgt @ dR; guess[:3, 3] = tgt + dt


def t_ms(f, n=1):
    t0 = time.perf_counter()
    for _ in range(n):
        r = f()
    return (time.perf_counter() - t0) * 1e3 / n, r


out = dict(map_points=int(m.shape[0]), scan_points=int(scan.shape[0]))
g = lsdreg.Matcher("NDT_CUDA")
r = RefNdtCuda(1.0, 7)
for name, mm in (("lsdreg", g), ("reference_cuda_sm90a", r)):
    mm.set_target(m[:1000]); mm.set_source(scan[:1000])                       # warm-up (module load, allocator)
    tb = min(t_ms(lambda: mm.set_target(m))[0] for _ in range(3))         # best of 3: allocator growth lands in the first call
    ts = min(t_ms(lambda: mm.set_source(scan))[0] for _ in range(3))
    lin = (lambda: mm.cost(guess)) if name == "lsdreg" else (lambda: mm.linearize(guess))
    lin()
    tl, res = t_ms(lin, 20)
    ta, T = t_ms(lambda: mm.align(guess))
    out[name] = dict(target_build_ms=tb, set_source_ms=ts, linearize_us=tl * 1e3, align_ms=ta, err=float(res[0]),
                     pos_err_m=float(np.abs(np.asarray(T)[:3, 3] - tgt).max()),
                     iterations=(g.iterations if name == "lsdreg" else None), n_voxels=(g.stats()["n_voxels"] if name == "lsdreg" else r.n_voxels))
eg, Hg, bg, nc = g.cost(guess)
er, Hr, br = r.linearize(guess)
out["agreement"] = dict(n_corr=[int(nc), int(r.n_corr)], err_rel=float(abs(eg - er) / abs(er)), H_rel=float(np.abs(Hg - Hr).max() / np.abs(Hr).max()),
                        b_rel=float(np.abs(bg - br).max() / np.abs(br).max()))
# ---- detection voxelizer: the reference's Preprocess + Voxelization kernels against lsd_vfe_*
from oracle.vfe import RefVoxelizer  # noqa: E402
frames = []
for f in range(8):
    sc = synth.scan64(300 + f, 800, synth.rot_from_rpy(0, 0, 0.05 * f), synth.block_center(0, 0) + np.array([0.8 * f, 0.1 * f, 0.0]))[:50000]
    pp = np.zeros((sc.shape[0], 5), np.float32); pp[:, :4] = sc; pp[:, 2] -= 1.8
    frames.append(pp)
M = np.eye(4, dtype=np.float32); M[:3, 3] = [0.8, 0.1, 0.0]
vg, vr = lsdreg.Voxelizer(max_frame_num=4, unordered_ids=1), RefVoxelizer(max_frame_num=4)   # same contract as the reference: ids in atomic order
vfe = {}
for name, v in (("lsdreg", vg), ("reference_cuda_sm90a", vr)):
    for f in range(4):
        v.accumulate(frames[f], M)
    v.voxelize(True)
    acc, vox = [], []
    for f in range(4, 8):
        a, tot = t_ms(lambda: v.accumulate(frames[f], M))
        b, res = t_ms(lambda: v.voxelize(True))
        acc.append(a); vox.append(b)
    vfe[name] = dict(window_points=int(tot), voxels=int(res[0].shape[0]), accumulate_us=float(np.mean(acc)) * 1e3, voxelize_us=float(np.mean(vox)) * 1e3)
out["vfe"] = vfe
print(json.dumps(out))
