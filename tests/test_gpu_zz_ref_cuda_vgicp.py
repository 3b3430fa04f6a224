"""GPU: the VGICP path against BOTH of the reference's own implementations of it, side by side:

  * fast_gicp::FastVGICP, the CPU/OpenMP class (fast_vgicp_impl.hpp, double precision) compiled unmodified into
    oracle/_ref/libref_reg.so — what registrations.cpp:56-66 selects on a build without CUDA, and what the product's
    VGICP follows;
  * fast_gicp::FastVGICPCuda over FastVGICPCudaCore recompiled for sm_90a (oracle/ref_cuda_vgicp.cu ->
    oracle/_ref/libref_cuda_vgicp.so) — what registrations.cpp:43-55 selects with USE_VGICP_CUDA.

Round 1 compared the product with the CUDA variant only, at 3 %, and failed (H off by 11 % on one diagonal entry, cost by
2.4 %).  The reason is inside the reference: its two variants do not agree with each other.  The CUDA one regularises the
k-NN covariances with Eigen's closed-form `SelfAdjointEigenSolver::computeDirect` in fp32 and rebuilds them as
V diag(1e-3, 1, 1) V^-1 (covariance_regularization.cu:15-52,105-116) where the CPU one uses a double-precision JacobiSVD
(fast_gicp_impl.hpp:283-300); it drops up to 1 % of the points from its voxel hash (gaussian_voxelmap.cu:283-288) and sums
fp32 moments with atomics.  So this test measures three distances on the same clouds and poses:
  product vs compiled CPU reference   — tight (1e-6 relative: same model, same precision),
  compiled CUDA reference vs compiled CPU reference — whatever it is (printed; the reference's own spread),
  product vs compiled CUDA reference  — must not exceed the reference's own spread by more than a third,
and the aligned poses of all three within 5 mm / 1e-3.  Runs in a subprocess (its own CUDA context).
"""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HAVE = os.path.exists(os.path.join(_ROOT, "oracle", "_ref", "libref_cuda_vgicp.so"))

_SCRIPT = r'''
import sys
sys.path.insert(0, %(root)r)
import numpy as np
import lsdreg
from lsdreg import synth
from oracle.reg import RefMatcher, RefVgicpCuda

lsdreg.init(0)
m = synth.block_map(1, 1, 1, 0.25)
m[:, :2] -= np.array([60, 40], np.float32)
Rgt = synth.rot_from_rpy(0.01, -0.02, 0.3)
tgt = np.array([1.0, -2.0, 1.8])
scan = synth.scan64(2, 200, Rgt, tgt + np.array([60, 40, 0]))[::2].copy()
dR, dt = synth.perturb(5, 0.5, 3.0)
guess = np.eye(4); guess[:3, :3] = Rgt @ dR; guess[:3, 3] = tgt + dt
Tgt = np.eye(4); Tgt[:3, :3] = Rgt; Tgt[:3, 3] = tgt
# registrations.cpp:43-55: eps 0.01, rotation epsilon left at LsqRegistration's default 1e-2 (lsq_registration_impl.hpp:24)
g = lsdreg.Matcher("FAST_VGICP_CUDA", transformation_epsilon=0.01, rotation_epsilon_deg=1e-2)
c = RefMatcher("vgicp", neighbors=1, trans_eps=0.01, rot_eps=1e-2)         # compiled CPU FastVGICP
r = RefVgicpCuda(1.0, 64, 0.01, 0)                                          # compiled CUDA FastVGICPCuda
for mm in (g, c, r):
    mm.set_target(m); mm.set_source(scan)

def rel(a, b):
    a, b = np.asarray(a, float), np.asarray(b, float)
    return float(np.abs(a - b).max() / np.abs(b).max())

for name, T in (("guess", guess), ("truth", Tgt)):
    er, Hr, br = r.linearize(T)
    eg, Hg, bg, ncg = g.cost(T)
    ec, Hc, bc = c.linearize(T)
    ours_cpu = (rel(eg, ec), rel(Hg, Hc), rel(bg, bc))
    cuda_cpu = (rel(er, ec), rel(Hr, Hc), rel(br, bc))
    ours_cuda = (rel(eg, er), rel(Hg, Hr), rel(bg, br))
    print(name, "cost / H / b, max-norm relative:  ours vs ref-CPU", ours_cpu, " ref-CUDA vs ref-CPU", cuda_cpu, " ours vs ref-CUDA", ours_cuda, " corr", ncg)
    assert max(ours_cpu) < 1e-6, ours_cpu                                   # the product IS the reference's CPU model
    assert max(cuda_cpu) < 0.25, cuda_cpu                                   # sanity: the two reference variants are the same method
    for a, b in zip(ours_cuda, cuda_cpu):
        assert a <= 1.34 * b + 1e-3, (name, ours_cuda, cuda_cpu)            # we are no further from the CUDA variant than its CPU sibling is
Tr = r.align(guess)
Tc = c.align(guess)
Tg = g.align(guess)
d = lambda A, B: (float(np.abs(A[:3, 3] - B[:3, 3]).max()), float(np.abs(A[:3, :3] - B[:3, :3]).max()))
print("align |dt|, |dR|: ours vs ref-CPU", d(Tg, Tc), " ref-CUDA vs ref-CPU", d(Tr, Tc), " ours vs ref-CUDA", d(Tg, Tr),
      " ours vs truth", float(np.abs(Tg[:3, 3] - tgt).max()), " converged", g.converged, c.converged, r.converged)
assert d(Tg, Tc)[0] < 1e-4 and d(Tg, Tc)[1] < 1e-5                           # float32 output of the reference's align()
assert d(Tg, Tr)[0] < 5e-3 and d(Tg, Tr)[1] < 1e-3
assert g.converged == c.converged
print("REF_VGICP_OK")
'''


@pytest.mark.skipif(not HAVE, reason="oracle/_ref/libref_cuda_vgicp.so not built (needs /root/reference + nvcc)")
def test_vgicp_matches_compiled_reference_cuda():
    r = subprocess.run([sys.executable, "-c", _SCRIPT % {"root": _ROOT}], cwd=_ROOT, capture_output=True, text=True, timeout=420)
    tail = (r.stdout[-3000:] + "\n" + r.stderr[-3000:])
    assert r.returncode == 0 and "REF_VGICP_OK" in r.stdout, tail
