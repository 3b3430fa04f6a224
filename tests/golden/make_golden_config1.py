"""Writes tests/golden/config1_ref.npz: what laserMapping.cpp compiled unmodified (oracle/_ref/libref_fastlio.so,
RefFastLioBench) computes for the first steps of bench.py's workload, for tests/test_gpu_lio_config1.py.  Needs the reference
tree at build time (oracle/_ref); run from the repository root:

  python tests/golden/make_golden_config1.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from oracle import eskf  # noqa: E402
from oracle import fastlio as FL  # noqa: E402

N_STEPS = 6

assert FL.HAVE_REF_FASTLIO, "oracle/_ref/libref_fastlio.so missing: run build() where the reference tree exists"
synth = bench.load_synth()
m = synth.block_map(bench.MAP_SEED, bench.BLOCKS_X, bench.BLOCKS_Y, bench.SPACING)
ref = FL.RefFastLioBench(capacity=1 << 30, threads=8)
ref.add_map_points(m)
P0 = eskf.init_P()
xs, Ps, counts = [], [], []
for s in range(N_STEPS):
    scan, Rgt, tgt, Rp, tp = bench.make_step(s)
    prior = eskf.State(); prior.rot = eskf.R_to_quat(Rp); prior.pos = tp.copy()
    xr, Pr, n_down = ref.process_scan(scan, prior, P0)
    c = ref.counts()
    xs.append(xr.to_vec()); Ps.append(Pr)
    counts.append([n_down, c["n_down"], c["n_eff"], c["degenerate"], c["map_cells"]])
np.savez_compressed(os.path.join(ROOT, "tests", "golden", "config1_ref.npz"), x=np.array(xs), P=np.array(Ps),
                    counts=np.array(counts, np.int64), map_points=m.shape[0])
print("wrote config1_ref.npz:", np.array(counts))
