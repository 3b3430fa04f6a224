"""Generates tests/golden/esti_plane_edges.npz: about 5 000 five-point sets at the edges of esti_plane (common_lib.h:236-268,
Eigen's ColPivHouseholderQR in fp32) with the COMPILED reference's answers (oracle/_ref/libref_lio.so), so that the device's
esti_plane_dev can be pinned bit for bit where the reference tree is absent (tests/test_gpu_lio_edges.py).

Families (name -> what it reaches):
  plane_d*        well-conditioned planes at distance 0, +-1e-6, 1e-3, 1, 1e3 and 1e4 m from the origin, the patch at the foot
                  of the normal or slid 30 m / 1 km along the plane; noise so that the 0.1 m gate goes both ways
  zero_column     one coordinate exactly 0 in every point (a plane through the origin: A n = -1 has no exact solution),
                  a share of the zeros written as -0.0
  zero_mixed      -0.0 and +0.0 entries scattered through otherwise general sets
  collinear       points exactly on a line (dyadic coordinates, exact in fp32): rank 2, or 1 when the line runs through 0
  near_collinear  the same lines with offsets of 1e-7 .. 1e-2 m off the line
  coincident_k    k = 2..5 copies of one point among general points (k = 5: rank 1)
  all_zero        five copies of (0, 0, 0) and of (-0, -0, -0): no non-zero pivot
  threshold       sets whose worst residual sits within one fp32 step of the 0.1 m gate: for each base set, the offset of one
                  point off the plane is bisected over its fp32 bit patterns to where the compiled reference's ok flips,
                  and the sets one ulp below, at and one ulp above the flip are kept
  norm_ties       two columns of equal norm in Eigen's summation order (the pivot is the first of them), whose norms
                  another order would round apart
  non_finite      one entry +-inf, NaN, 1e19 (its square overflows) or a denormal
  far             clusters of 0.5 m at up to 1e4 m from the origin in every direction

Each set's columns are permuted at random so that Eigen's column pivoting takes every permutation.  Stored: pts [n,5,3]
float32, pabcd [n,4] float32 and ok [n] int8 from ref_esti_plane (threshold 0.1), nz [n] int8 and perm [n,3] int8 from
ref_esti_plane_qr (non-zero pivots, column permutation), family [n] int8 indexing `families`.  Where the compiled
reference is present, tests/test_gpu_lio_edges.py also draws the same families at scale 4 (about 1.3 10^5 sets)
and takes the answers from the reference itself.

Run from the repository root with oracle/_ref built: python tests/golden/make_golden_esti_plane.py"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
OUT = os.path.join(ROOT, "tests", "golden", "esti_plane_edges.npz")
FIXTURE_SCALE = 0.15        # the committed fixture: every family, about 5 000 sets (under 300 kB)


def _basis(rng, n):
    nrm = rng.normal(size=(n, 3)); nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    a = np.where(np.abs(nrm[:, :1]) < 0.9, [[1.0, 0, 0]], [[0, 1.0, 0]])
    u = np.cross(nrm, a); u /= np.linalg.norm(u, axis=1, keepdims=True)
    v = np.cross(nrm, u)
    return nrm, u, v


def planes(rng, n, dist, slide, spread=0.7, noise=0.03):
    nrm, u, v = _basis(rng, n)
    c = nrm * dist + u * slide
    t = rng.uniform(-spread, spread, (n, 5, 2))
    p = c[:, None] + t[..., :1] * u[:, None] + t[..., 1:] * v[:, None] + nrm[:, None] * rng.normal(scale=noise, size=(n, 5, 1))
    return p.astype(np.float32)


def dyadic(rng, shape, lo, hi, bits=4):
    return (rng.integers(lo << bits, hi << bits, shape) / float(1 << bits)).astype(np.float32)


def collinear(rng, n, through_origin):
    d = dyadic(rng, (n, 1, 3), -2, 3, 2)
    d[np.all(d == 0, axis=2)[:, 0]] = np.float32([1, 0, 0])
    t = dyadic(rng, (n, 5, 1), -4, 5, 2)
    a = np.zeros((n, 1, 3), np.float32) if through_origin else dyadic(rng, (n, 1, 3), -20, 20)
    return (a + t * d).astype(np.float32), d


def edge_sets(O, rng, scale=1.0):
    """-> (pts [n,5,3] float32, family [n] int8, family names): every family above, about 33 000 sets at scale 1.  The
    threshold family is bisected against the compiled reference O.ref_esti_plane."""
    k = lambda m: max(1, int(round(m * scale)))
    fams = []                                   # (name, sets)
    for dist in (0.0, 1e-6, -1e-6, 1e-3, 1.0, 1e3, 1e4):
        for slide in (0.0, 30.0, 1e3):
            fams.append((f"plane_d{dist:g}_s{slide:g}", planes(rng, k(400), dist, slide, noise=0.03 if slide < 1e3 else 0.01)))
    n = k(1500)
    p = planes(rng, n, 3.0, 5.0)
    ax = rng.integers(0, 3, n)
    p[np.arange(n), :, ax] = 0.0
    i, j = np.nonzero(rng.random((n, 5)) < 0.4)
    p[i, j, ax[i]] = -0.0
    fams.append(("zero_column", p))
    p = planes(rng, k(1000), 2.0, 3.0)
    z = rng.random(p.shape) < 0.25
    p[z] = np.where(rng.random(int(z.sum())) < 0.5, np.float32(0.0), np.float32(-0.0))
    fams.append(("zero_mixed", p))
    for origin in (False, True):
        c, d = collinear(rng, k(1500), origin)
        fams.append((f"collinear{'_origin' if origin else ''}", c))
    n = k(3000)
    c, d = collinear(rng, n, False)
    perp = np.cross(d[:, 0], rng.normal(size=(n, 3)))
    perp /= np.linalg.norm(perp, axis=1, keepdims=True)
    eps = np.array([1e-7, 1e-6, 1e-5, 1e-4, 1e-3, 1e-2])[np.arange(n) % 6]
    off = perp[:, None] * (eps[:, None, None] * rng.uniform(-1, 1, (n, 5, 1)))
    fams.append(("near_collinear", (c + off).astype(np.float32)))
    for m in (2, 3, 4, 5):
        p = planes(rng, k(1000), 4.0, 2.0)
        p[:, :m] = p[:, :1]
        p = p[:, rng.permutation(5)]
        fams.append((f"coincident_{m}", p))
    z = np.zeros((40, 5, 3), np.float32)
    z[20:] = -0.0
    fams.append(("all_zero", z))
    # two columns whose squared entries are the same up to swaps inside the pairs (0, 1) and (2, 3): equal norms in
    # Eigen's order ((t0 + t2) + (t1 + t3)) + t4, while another summation order would round them apart and pick another pivot
    n = k(6000)
    p = planes(rng, n, 1.5, 2.0, spread=1.0, noise=0.2)
    p[:, :, 1] = p[:, [1, 0, 3, 2, 4], 0] * rng.choice(np.float32([-1, 1]), (n, 5))
    fams.append(("norm_ties", p))
    n = k(200)
    p = planes(rng, n, 2.0, 1.0)
    r = np.arange(n)
    p[r, rng.integers(0, 5, n), rng.integers(0, 3, n)] = np.array([np.inf, -np.inf, np.nan, 1e19, 1e-40])[r % 5]
    fams.append(("non_finite", p))
    n = k(2000)
    far = rng.normal(size=(n, 3)); far /= np.linalg.norm(far, axis=1, keepdims=True)
    far *= np.array([1e2, 1e3, 5e3, 1e4])[np.arange(n) % 4, None]
    fams.append(("far", (far[:, None] + planes(rng, n, 0.0, 0.0, spread=0.5, noise=0.02)).astype(np.float32)))
    fams.append(("threshold", threshold_sets(O, rng, k(600))))
    names = [f for f, _ in fams]
    pts = np.concatenate([s for _, s in fams]).astype(np.float32)
    fam = np.concatenate([np.full(len(s), i, np.int8) for i, (_, s) in enumerate(fams)])
    # every set's columns in a random order: Eigen's pivoting then takes every permutation
    perm = np.argsort(rng.random((len(pts), 3)), axis=1)
    return np.ascontiguousarray(np.take_along_axis(pts, perm[:, None, :], axis=2)), fam, names


def main():
    from oracle import oracle as O
    assert O.HAVE_REF and hasattr(O.ref, "ref_esti_plane_qr"), "oracle/_ref/libref_lio.so not built (needs the reference tree)"
    pts, fam, names = edge_sets(O, np.random.default_rng(20261018), scale=FIXTURE_SCALE)
    pabcd, ok = O.ref_esti_plane(pts, 0.1)
    qr = O.ref_esti_plane_qr(pts)
    np.savez_compressed(OUT, pts=pts, pabcd=pabcd, ok=ok.astype(np.int8), nz=qr["nonzero_pivots"].astype(np.int8),
                        perm=qr["perm"].astype(np.int8), family=fam, families=np.array(names))
    print(f"{OUT}: {len(pts)} sets, {os.path.getsize(OUT) / 1e6:.2f} MB")


def _ord(f):
    """fp32 -> integers in the order of the values (adjacent floats are adjacent integers; -0.0 and +0.0 both 0)."""
    b = np.asarray(f, np.float32).view(np.int32).astype(np.int64)
    return np.where(b >= 0, b, -(b & 0x7FFFFFFF))


def _unord(o):
    o = np.asarray(o, np.int64)
    return np.where(o >= 0, o, (-o) | 0x80000000).astype(np.uint32).view(np.float32)


def threshold_sets(O, rng, n):
    """Sets on the 0.1 m gate: four points on a plane and a fifth moved off it along the coordinate axis closest to the
    normal.  That coordinate is bisected over its fp32 values (0 to 0.4 m off the plane) to where the compiled reference's
    ok flips, and the sets one value below the flip, at it and one above are kept."""
    out = []
    for dist, spread in ((1.0, 0.6), (40.0, 0.8), (800.0, 0.5)):
        base = planes(rng, n, dist, 10.0, spread=spread, noise=0.0)
        c = base.astype(np.float64)
        nrm = np.cross(c[:, 1] - c[:, 0], c[:, 2] - c[:, 0]); nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
        k = np.abs(nrm).argmax(1)
        r = np.arange(n)
        x0 = base[r, 4, k]
        lo = _ord(x0)                                          # accepted (on the plane up to rounding)
        hi = _ord((x0 + np.sign(nrm[r, k]) * 0.4 / np.abs(nrm[r, k])).astype(np.float32))   # rejected: 0.4 m off

        def at(o):
            s = base.copy()
            s[r, 4, k] = _unord(o)
            return s

        keep = (O.ref_esti_plane(at(lo), 0.1)[1] == 1) & (O.ref_esti_plane(at(hi), 0.1)[1] == 0)
        for _ in range(40):
            mid = lo + (hi - lo) // 2
            ok = O.ref_esti_plane(at(mid), 0.1)[1] == 1
            lo = np.where(ok, mid, lo); hi = np.where(ok, hi, mid)
        keep &= np.abs(hi - lo) == 1
        step = np.sign(hi - lo)
        for d in (-1, 0, 1):
            out.append(at(hi + d * step)[keep])
    return np.concatenate(out)


if __name__ == "__main__":
    main()
