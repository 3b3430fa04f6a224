"""TEST INFRASTRUCTURE: the IMU stage's edge cases (tests/imu_edges.py: the earliest point's repeated compensation, ties
on IMU pose offsets, IMU past the scan end, stale samples and gaps, init paths, time-field edges, sizes, the 256-pose cap,
undistort = 0) at emulator sizes, the product's kernels against the compiled reference class.  Run by
tests/test_emu_kernels.py; the same cases run on the GPU in tests/test_gpu_imu_edges.py."""
import sys

import imu_edges
import lsdreg
from oracle import oracle as O

assert O.HAVE_REF_IKFOM, "oracle/_ref/libref_ikfom.so not built"
lsdreg.init(0)
for name, case in imu_edges.CASES.items():
    if name in imu_edges.NEEDS_TORCH:
        continue
    case(False)
    print("ok imu", name)
    sys.stdout.flush()
print("FUZZ_IMU_OK")
