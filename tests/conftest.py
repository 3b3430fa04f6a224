import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on the H100 with -m gpu)")
    # make sure the native artefacts exist (nvcc cross-compiles without a GPU)
    import __graft_entry__ as g
    g.build()   # no-op when liblsdreg.so, slam_wrapper and the oracle libraries are newer than their sources
    if os.environ.get("LSDREG_EMU"):
        # run the `gpu` tests against the SIMT emulator build (tests/simt): the same sources, kernels executed by fibers on
        # the CPU.  A debugging aid for kernels written without a GPU at hand; never a substitute for the H100 run.
        sys.path.insert(0, os.path.join(ROOT, "tests", "simt"))
        import build_emu
        import lsdreg
        lsdreg.capi.lib = lsdreg.capi.load_library(build_emu.build())
        lsdreg.lib = lsdreg.capi.lib


@pytest.fixture(scope="session")
def small_world():
    """2x2-block map (~240 k pts), a 16 k-pt scan with its ground-truth pose and a perturbed prior."""
    import numpy as np
    from lsdreg import synth
    m = synth.block_map(1, 2, 2, 0.5)
    Rgt = synth.rot_from_rpy(0.01, -0.02, 0.3)
    tgt = synth.block_center(0, 0) + np.array([1.0, -2.0, 0.0])
    scan = synth.scan64(2, 250, Rgt, tgt)
    dR, dt = synth.perturb(5)
    return dict(map=m, scan=scan, Rgt=Rgt, tgt=tgt, Rprior=Rgt @ dR, tprior=tgt + dt)
