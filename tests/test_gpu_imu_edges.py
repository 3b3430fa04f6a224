"""GPU parity, row N1 at the edges: the product's IMU stage (host forward propagation, imu_undistort_kernel and the
one-thread imu_first_point_kernel) against the COMPILED reference ImuProcess, with the numpy restatement run alongside so
a failure shows which of the two departs from the reference.  The cases and bars are in tests/imu_edges.py, whose
docstring also states the one specified divergence: among points tied at the earliest time past the first IMU pose, the
reference repeats the compensation on whichever std::sort put first, the product on the lowest input index."""
import imu_edges
import pytest

from oracle import oracle as O

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not O.HAVE_REF_IKFOM, reason="oracle/_ref/libref_ikfom.so not built (needs the reference tree)")]


@pytest.mark.parametrize("case", list(imu_edges.CASES))
def test_imu_stage_matches_compiled_reference(case):
    imu_edges.CASES[case](True)
