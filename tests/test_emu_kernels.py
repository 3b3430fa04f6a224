"""CPU: the kernels that have not seen a GPU yet, executed by the SIMT emulator (tests/simt) against the oracle.

The four GPU tests written after round 1's GPU budget was spent (tests/test_gpu_zz_*.py: flat k-NN shape, ScanContext,
stale Nearest_Points rows, the LIO seam end to end) carry their bodies as scripts; here the same scripts run with
liblsdreg_emu.so — the product's CUDA sources compiled for the host, kernels executed by fibers — swapped in for liblsdreg.so.
This is a logic check (indices, capacities, phase structure, collectives, arithmetic), not a parity claim: see
tests/simt/README.md for what an emulator on one CPU thread can and cannot show.  The four run concurrently (~40 s)."""
import importlib.util
import os
import subprocess
import sys

import pytest

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)

_CASES = {
    "scancontext": ("test_gpu_zz_scancontext.py", "SC_OK"),
    "sequence": ("test_gpu_zz_sequence.py", "SEQUENCE_OK"),
    "fastlio_seam": ("test_gpu_zz_fastlio_seam.py", "SEAM_OK"),
    "pdl": ("test_gpu_zz_pdl.py", "PDL_OK"),      # control flow only: the emulator serialises launches, PDL on == off by construction
    "fuzz_knn": ("simt/fuzz_knn.py", "FUZZ_OK"),   # adversarial map / k-NN inputs, three shapes vs each other and the oracle
    "fuzz_misc": ("simt/fuzz_misc.py", "FUZZ_MISC_OK"),
    "fuzz_reforder": ("simt/fuzz_reforder.py", "FUZZ_REFORDER_OK"),   # reference-order rows on crowded / clustered maps, every path of the search kernel
    "fuzz_nth": ("simt/fuzz_nth.py", "FUZZ_NTH_OK"),   # std::nth_element as the search kernel replays it vs the restatement (warp path, depth-limit bail-out, serial path)
    "fuzz_map_contents": ("simt/fuzz_map_contents.py", "FUZZ_MAP_CONTENTS_OK"),   # the map's contents voxel by voxel: insert, box delete, LRU eviction
    "fuzz_pipeline": ("simt/fuzz_pipeline.py", "FUZZ_PIPELINE_OK"),   # random announce / register schedules: staging slots, deferred requests, buffer hand-over   # voxel grid, key-frame filters, ScanContext descriptor on degenerate inputs
    "fuzz_imu": ("simt/fuzz_imu.py", "FUZZ_IMU_OK"),   # the IMU stage's edge cases vs the compiled ImuProcess (tests/imu_edges.py)
}
# cases that compare with a compiled reference library under oracle/_ref, built only where the reference tree is readable
_NEEDS = {"fuzz_imu": "libref_ikfom.so"}


def _runnable(case):
    return case not in _NEEDS or os.path.exists(os.path.join(_ROOT, "oracle", "_ref", _NEEDS[case]))


_PROLOGUE = r'''
import sys
sys.path.insert(0, %(root)r); sys.path.insert(0, %(root)r + "/tests"); sys.path.insert(0, %(root)r + "/tests/simt")
import lsdreg, build_emu
lsdreg.capi.lib = lsdreg.capi.load_library(build_emu.build())
lsdreg.lib = lsdreg.capi.lib
'''


def _script(fname):
    if fname.startswith("simt/"):      # a plain script, not a test module
        return _PROLOGUE % {"root": _ROOT} + open(os.path.join(_HERE, fname)).read()
    spec = importlib.util.spec_from_file_location("zz_" + fname[:-3], os.path.join(_HERE, fname))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return (_PROLOGUE + m._SCRIPT) % {"root": _ROOT}


@pytest.fixture(scope="module")
def runs():
    sys.path.insert(0, os.path.join(_HERE, "simt"))
    import build_emu
    build_emu.build()                      # once, before the four start
    procs = {k: subprocess.Popen([sys.executable, "-c", _script(f)], cwd=_ROOT, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
             for k, (f, _) in _CASES.items() if _runnable(k)}
    out = {}
    for k, p in procs.items():
        try:
            so, se = p.communicate(timeout=1500)
        except subprocess.TimeoutExpired:
            p.kill(); so, se = p.communicate()
            se += "\nTIMEOUT"
        out[k] = (p.returncode, so, se)
    return out


@pytest.mark.parametrize("case", list(_CASES))
def test_kernel_logic_under_the_simt_emulator(runs, case):
    if not _runnable(case):
        pytest.skip(f"oracle/_ref/{_NEEDS[case]} not built (needs the reference tree)")
    rc, so, se = runs[case]
    assert rc == 0 and _CASES[case][1] in so, so[-3000:] + "\n" + se[-3000:]
