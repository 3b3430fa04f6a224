"""Per-term restatement, in numpy, of the scan matcher's cost kernels (reg.cu), for tests/test_gpu_reg_cost_terms.py and
tests/test_reg_cost_ref_host.py.

Given the source cloud, the pose(s) and the target tables the matcher built (lsd_reg_get_voxels, lsd_reg_get_covariances),
every function returns the terms one source point contributes to each of the 28 outputs of a cost evaluation (21 upper-
triangle H, 6 b, err), one row per (stencil offset, source point), and the correspondence pattern.  The kernel expressions
are restated in their own order and precision:

* xform (Pose34f in fp32, Pose34d in double), ndt_coord (floorf(x / res - 0.5f) in fp32), vg_coord (floor in double), the
  DIRECT1 / 7 / 27 stencils, the `<= 6` point gate of ndt_point;
* ndt_point: C^-1 e = e + 999 n (n.e) and C^-1 J alike, the Cauchy weight k^2 / (k^2 + xn * xn) with xn = sqrtf(|e|^2),
  every product in fp32, each term cast to double as the kernel adds it;
* gicp_store_maha and vgicp_point: the cofactor inverse of C_B + R C_A R^T in double, stored as the kernel stores it;
* accum_d2d: e^T M e, J^T M J and J^T M e with VGICP's weight sqrt(voxel points).

Only element-wise numpy operations are used (no @, dot or einsum, whose BLAS kernels may reorder or fuse), and numpy keeps
float32 arithmetic in float32, so every term is the kernel's term bit for bit (the library is built with -fmad=false and
without fast math).  What is left free is the order of the double reduction over terms, bounded by reduction_bound().

math_check_ndt / math_check_gicp / math_check_vgicp are the independent float64 statement of the same quantities
(numpy.linalg.inv, textbook J^T M J): they hold the restatement to the mathematics, so that the restatement cannot copy a
kernel bug faithfully.
"""
import math

import numpy as np

F32 = np.float32
F64 = np.float64
U64 = 2.0 ** -53
U32 = 2.0 ** -24
OFF7 = np.array([[0, 0, 0], [1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1]], np.int64)
TRIU = np.triu_indices(6)          # (p, r), p <= r, row-major: the kernels' vals[0..21) order


def stencil(n_off):
    """Offsets of DIRECT1 / DIRECT7 / DIRECT27 in the order the kernels visit them (stencil_offset)."""
    if n_off == 27:
        o = np.arange(27)
        return np.stack([o // 9 - 1, (o // 3) % 3 - 1, o % 3 - 1], 1).astype(np.int64)
    return OFF7[:n_off]


def xform_f(T, a):
    """Pose34f xform: R a + t in fp32, each row ((r0 x + r1 y) + r2 z) + t.  a [n, >=3] float32; returns 3 float32 [n]."""
    R, t = np.asarray(T, F64)[:3, :3].astype(F32), np.asarray(T, F64)[:3, 3].astype(F32)
    x, y, z = (a[:, k].astype(F32) for k in range(3))
    return tuple(R[r, 0] * x + R[r, 1] * y + R[r, 2] * z + t[r] for r in range(3))


def xform_d(T, a):
    """Pose34d xform: R a + t in double from the float point."""
    T = np.asarray(T, F64)
    x, y, z = (a[:, k].astype(F32).astype(F64) for k in range(3))
    return tuple(T[r, 0] * x + T[r, 1] * y + T[r, 2] * z + T[r, 3] for r in range(3))


def rotate_d(T, n):
    """R n in double (gicp_store_maha / vgicp_point: rn)."""
    T = np.asarray(T, F64)
    return tuple(T[r, 0] * n[:, 0] + T[r, 1] * n[:, 1] + T[r, 2] * n[:, 2] for r in range(3))


class Table:
    """A voxel dump of Matcher.voxels() (or the same dict built from the oracle), looked up by coordinate."""

    def __init__(self, vox):
        self.coord = np.asarray(vox["coord"], np.int64).reshape(-1, 3)
        key = self._key(self.coord)
        self.order = np.argsort(key)
        self.sorted = key[self.order]
        self.count = np.asarray(vox["count"], np.int64)
        self.mean = np.asarray(vox["mean"], F64).reshape(-1, 3)
        self.second = np.asarray(vox["second"], F64).reshape(-1, 6)

    @staticmethod
    def _key(c):
        return ((c[:, 0] + (1 << 20)) << 42) | ((c[:, 1] + (1 << 20)) << 21) | (c[:, 2] + (1 << 20))

    def lookup(self, c):
        """Row of every coordinate c [m, 3] in the dump, -1 where the table has no such voxel."""
        if len(self.sorted) == 0:
            return np.full(len(c), -1, np.int64)
        k = self._key(np.asarray(c, np.int64))
        pos = np.minimum(np.searchsorted(self.sorted, k), len(self.sorted) - 1)
        return np.where(self.sorted[pos] == k, self.order[pos], -1)


def _accum_d2d(M, e, t, w, deriv):
    """accum_d2d for arrays of terms: M 6-tuple (xx xy xz yy yz zz), e / t 3-tuples, w (python float 1.0 or array).
    Returns [m, 28] double terms (H upper triangle, b, err)."""
    m00, m01, m02, m11, m12, m22 = M
    Mm = ((m00, m01, m02), (m01, m11, m12), (m02, m12, m22))
    ex, ey, ez = e
    cx = Mm[0][0] * ex + Mm[0][1] * ey + Mm[0][2] * ez
    cy = Mm[1][0] * ex + Mm[1][1] * ey + Mm[1][2] * ez
    cz = Mm[2][0] * ex + Mm[2][1] * ey + Mm[2][2] * ez
    out = np.zeros((len(ex), 28), F64)
    out[:, 27] = w * (ex * cx + ey * cy + ez * cz)
    if deriv:
        z, one = np.zeros_like(ex), np.ones_like(ex)
        tx, ty, tz = t
        J = ((z, -tz, ty, -one, z, z), (tz, z, -tx, z, -one, z), (-ty, tx, z, z, z, -one))
        MJ = [[Mm[r][0] * J[0][cc] + Mm[r][1] * J[1][cc] + Mm[r][2] * J[2][cc] for cc in range(6)] for r in range(3)]
        q = 0
        for p in range(6):
            for r in range(p, 6):
                out[:, q] = w * (J[0][p] * MJ[0][r] + J[1][p] * MJ[1][r] + J[2][p] * MJ[2][r])
                q += 1
            out[:, 21 + p] = w * (J[0][p] * cx + J[1][p] * cy + J[2][p] * cz)
    return out


class Terms:
    """Terms of one cost evaluation: vals [n_off, n, 28] (zero rows where no residual), found [n_off, n] (a
    correspondence: vals[28] counts it), used [n_off, n] (a residual was added), plus per-matcher extras."""

    def __init__(self, vals, found, used, **extra):
        self.vals, self.found, self.used = vals, found, used
        self.__dict__.update(extra)

    @property
    def n_corr(self):
        return int(self.found.sum())

    def flat(self):
        """The [m, 28] terms that enter the sums (the rows with a residual)."""
        return self.vals[self.used]

    def per_point(self):
        """[n, 28]: each point's terms summed in offset order into zeros, as a one-point source's evaluation does."""
        acc = np.zeros(self.vals.shape[1:], F64)
        for o in range(self.vals.shape[0]):
            acc = acc + self.vals[o]
        return acc


# ------------------------------------------------------------------ NDT (ndt_point)
def ndt_terms(src, vox, res, n_off, T_lin, T_ev, deriv=True):
    """NDT terms: correspondences looked up at T_lin (ndt_coord of the fp32 transformed point + stencil), residuals at T_ev.
    vox: the NDT dump (mean = float mean, second[:, :3] = float normal)."""
    tab = vox if isinstance(vox, Table) else Table(vox)
    a = np.ascontiguousarray(src[:, :3], F32)
    n = a.shape[0]
    r32 = F32(res)
    k_sq = r32 * r32
    tx, ty, tz = xform_f(T_ev, a)
    lx, ly, lz = xform_f(T_lin, a)
    half = F32(0.5)
    c = np.stack([np.floor(lx / r32 - half), np.floor(ly / r32 - half), np.floor(lz / r32 - half)], 1).astype(np.int64)
    off = stencil(n_off)
    vals = np.zeros((n_off, n, 28), F64)
    found = np.zeros((n_off, n), bool)
    used = np.zeros((n_off, n), bool)
    slot = np.full((n_off, n), -1, np.int64)
    mean32 = tab.mean.astype(F32)
    nrm32 = tab.second[:, :3].astype(F32)
    k999 = F32(999.0)
    for o in range(n_off):
        row = tab.lookup(c + off[o])
        slot[o] = row
        found[o] = row >= 0
        sel = np.nonzero(found[o])[0]
        sel = sel[tab.count[row[sel]] > 6]                  # ndt_compute_derivatives.cu:62-64
        used[o, sel] = True
        if sel.size == 0:
            continue
        rr = row[sel]
        mx, my, mz = mean32[rr, 0], mean32[rr, 1], mean32[rr, 2]
        nx, ny, nz = nrm32[rr, 0], nrm32[rr, 1], nrm32[rr, 2]
        px, py, pz = tx[sel], ty[sel], tz[sel]
        ex, ey, ez = mx - px, my - py, mz - pz
        ne = nx * ex + ny * ey + nz * ez
        cx, cy, cz = ex + k999 * nx * ne, ey + k999 * ny * ne, ez + k999 * nz * ne
        xn = np.sqrt(ex * ex + ey * ey + ez * ez)
        w = k_sq / (k_sq + xn * xn)
        v = vals[o, sel]
        v[:, 27] = (w * (ex * cx + ey * cy + ez * cz)).astype(F64)
        if deriv:
            z, one = np.zeros_like(px), np.ones_like(px)
            J = ((z, -pz, py, -one, z, z), (pz, z, -px, z, -one, z), (-py, px, z, z, z, -one))
            M = [[None] * 6 for _ in range(3)]
            for cc in range(6):
                nj = nx * J[0][cc] + ny * J[1][cc] + nz * J[2][cc]
                M[0][cc], M[1][cc], M[2][cc] = J[0][cc] + k999 * nx * nj, J[1][cc] + k999 * ny * nj, J[2][cc] + k999 * nz * nj
            q = 0
            for p in range(6):
                for r in range(p, 6):
                    v[:, q] = (w * (J[0][p] * M[0][r] + J[1][p] * M[1][r] + J[2][p] * M[2][r])).astype(F64)
                    q += 1
                v[:, 21 + p] = (w * (J[0][p] * cx + J[1][p] * cy + J[2][p] * cz)).astype(F64)
        vals[o, sel] = v
    return Terms(vals, found, used, slot=slot, table=tab, t=(tx, ty, tz), res=res, deriv=deriv)


# ------------------------------------------------------------------ GICP (gicp_store_maha, gicp_cost_kernel)
def gicp_maha(src_nrm, tgt_nrm, corr, T):
    """gicp_store_maha for every source point with a correspondence: [n, 6] (xx xy xz yy yz zz), NaN rows where corr < 0."""
    n = len(corr)
    out = np.full((n, 6), np.nan)
    sel = np.nonzero(corr >= 0)[0]
    if sel.size == 0:
        return out
    rn = rotate_d(T, np.asarray(src_nrm, F64)[sel, :3])
    nb = np.asarray(tgt_nrm, F64)[corr[sel], :3]
    nbv = (nb[:, 0], nb[:, 1], nb[:, 2])
    A = [(2.0 if p == q else 0.0) - 0.999 * (nbv[p] * nbv[q] + rn[p] * rn[q]) for p in range(3) for q in range(3)]
    c00 = A[4] * A[8] - A[5] * A[7]
    c01 = A[5] * A[6] - A[3] * A[8]
    c02 = A[3] * A[7] - A[4] * A[6]
    idet = 1.0 / (A[0] * c00 + A[1] * c01 + A[2] * c02)
    out[sel] = np.stack([c00 * idet, (A[2] * A[7] - A[1] * A[8]) * idet, (A[1] * A[5] - A[2] * A[4]) * idet,
                         (A[0] * A[8] - A[2] * A[6]) * idet, (A[2] * A[3] - A[0] * A[5]) * idet,
                         (A[0] * A[4] - A[1] * A[3]) * idet], 1)
    return out


def dist2f(q, p):
    """The kernels' fp32 dist2 of query rows q [m, 3] to point rows p [m, 3]: (dx*dx + dy*dy) + dz*dz."""
    d = p.astype(F32) - q.astype(F32)
    return d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1] + d[:, 2] * d[:, 2]


def gicp_nn(src, tgt, T, max_corr, k=8):
    """update_correspondences under the reference's gate: the 1-NN of the fp32 transformed source point by fp32 d2 (ties:
    lower index) among the k nearest by a float64 k-d tree, kept where (double) d2 < max_corr^2 (double).  Returns corr [n]
    and the fp32 d2 of the nearest [n].  Raises if a nearest point could lie outside the k candidates."""
    from scipy.spatial import cKDTree
    a = np.ascontiguousarray(src[:, :3], F32)
    q = np.stack(xform_f(T, a), 1)
    P = np.ascontiguousarray(tgt[:, :3], F32)
    k = min(k, len(P))
    d64, idx = cKDTree(P.astype(F64)).query(q.astype(F64), k=k)
    d64, idx = d64.reshape(len(q), k), idx.reshape(len(q), k)
    d2 = np.stack([dist2f(q, P[idx[:, j]]) for j in range(k)], 1)
    key = (d2.view(np.uint32).astype(np.uint64) << np.uint64(32)) | idx.astype(np.uint64)   # d2 >= 0: bits order like values
    best = np.argmin(key, axis=1)
    rows = np.arange(len(q))
    bd, bi = d2[rows, best], idx[rows, best]
    if k < len(P):
        # every point outside the candidates is at least d64[:, -1] away; its fp32 d2 is that squared to within
        # gamma_5(u32) relative (one rounding of each difference, three products, two sums)
        g5 = 5 * U32 / (1 - 5 * U32)
        assert np.all(d64[:, -1] ** 2 * (1 - g5) > bd.astype(F64) * (1 + 1e-15)), "raise k: a nearer point may be uncovered"
    corr = np.where(bd.astype(F64) < float(max_corr) * float(max_corr), bi, -1).astype(np.int64)
    return corr, bd


def gicp_terms(src, tgt, src_nrm, tgt_nrm, corr, T_lin, T_ev, deriv=True):
    """GICP terms at T_ev with the correspondences corr and the Mahalanobis matrices of T_lin (update: T_lin = T_ev)."""
    M = gicp_maha(src_nrm, tgt_nrm, corr, T_lin)
    n = len(corr)
    found = (corr >= 0)[None, :]
    vals = np.zeros((1, n, 28), F64)
    sel = np.nonzero(found[0])[0]
    a = np.ascontiguousarray(src[:, :3], F32)[sel]
    t = xform_d(T_ev, a)
    b = np.ascontiguousarray(tgt[:, :3], F32)[corr[sel]].astype(F64)
    e = (b[:, 0] - t[0], b[:, 1] - t[1], b[:, 2] - t[2])
    vals[0, sel] = _accum_d2d(tuple(M[sel, j] for j in range(6)), e, t, 1.0, deriv)
    return Terms(vals, found, found.copy(), maha=M, corr=corr, t=t, e=e, sel=sel, deriv=deriv)


# ------------------------------------------------------------------ VGICP (vgicp_point)
def vgicp_terms(src, src_nrm, vox, res, n_off, T_lin, T_ev, deriv=True):
    """VGICP terms: voxels looked up at T_lin (vg_coord of the double transformed point + stencil) with the Mahalanobis
    matrices of T_lin, residuals at T_ev (update: T_lin = T_ev).  vox: the VGICP dump (mean, second = cov xx xy xz yy yz zz)."""
    tab = vox if isinstance(vox, Table) else Table(vox)
    a = np.ascontiguousarray(src[:, :3], F32)
    n = a.shape[0]
    lt = xform_d(T_lin, a)
    c = np.stack([np.floor(lt[k] / float(res) - 0.5) for k in range(3)], 1).astype(np.int64)
    rn_all = rotate_d(T_lin, np.asarray(src_nrm, F64)[:, :3])
    t_all = xform_d(T_ev, a)
    off = stencil(n_off)
    vals = np.zeros((n_off, n, 28), F64)
    found = np.zeros((n_off, n), bool)
    maha = np.full((n_off, n, 6), np.nan)
    slot = np.full((n_off, n), -1, np.int64)
    for o in range(n_off):
        row = tab.lookup(c + off[o])
        slot[o] = row
        found[o] = row >= 0
        sel = np.nonzero(found[o])[0]
        if sel.size == 0:
            continue
        rr = row[sel]
        cv = [tab.second[rr, j] for j in range(6)]
        r0, r1, r2 = rn_all[0][sel], rn_all[1][sel], rn_all[2][sel]
        A0 = cv[0] + 1.0 - 0.999 * r0 * r0
        A1 = cv[1] - 0.999 * r0 * r1
        A2 = cv[2] - 0.999 * r0 * r2
        A4 = cv[3] + 1.0 - 0.999 * r1 * r1
        A5 = cv[4] - 0.999 * r1 * r2
        A8 = cv[5] + 1.0 - 0.999 * r2 * r2
        c00, c01, c02 = A4 * A8 - A5 * A5, A5 * A2 - A1 * A8, A1 * A5 - A4 * A2
        idet = 1.0 / (A0 * c00 + A1 * c01 + A2 * c02)
        M = (c00 * idet, c01 * idet, c02 * idet, (A0 * A8 - A2 * A2) * idet, (A2 * A1 - A0 * A5) * idet, (A0 * A4 - A1 * A1) * idet)
        maha[o, sel] = np.stack(M, 1)
        t = (t_all[0][sel], t_all[1][sel], t_all[2][sel])
        m = tab.mean[rr]
        e = (m[:, 0] - t[0], m[:, 1] - t[1], m[:, 2] - t[2])
        w = np.sqrt(tab.count[rr].astype(F64))
        vals[o, sel] = _accum_d2d(M, e, t, w, deriv)
    return Terms(vals, found, found.copy(), slot=slot, maha=maha, table=tab, t=t_all, deriv=deriv)


# ------------------------------------------------------------------ bounds and the independent check
def gamma(k, u=U64):
    return k * u / (1.0 - k * u)


def reduction_bound(terms):
    """For each of the 28 outputs: (exact sum fsum(t), gamma(m - 1) * sum |t|), the worst case of any order of m - 1 double
    additions of the m terms [m, 28]."""
    m = terms.shape[0]
    s = np.array([math.fsum(terms[:, j]) for j in range(28)])
    return s, gamma(max(m - 1, 0)) * np.abs(terms).sum(0)


def unpack(e, H, b):
    """A device result (err, H 6x6, b 6) as the 28-vector of the kernels' vals[0..28)."""
    out = np.zeros(28)
    out[:21] = np.asarray(H)[TRIU]
    out[21:27] = b
    out[27] = e
    return out


def check_sums(dev28, terms, deriv=True):
    """The device's 28 sums against the exact sum of the restated terms.  Returns the worst ratio |S - fsum| / bound (<= 1
    holds; 0 when every sum is exact) over the outputs the evaluation produced."""
    s, bnd = reduction_bound(terms)
    idx = np.arange(28) if deriv else np.array([27])
    diff = np.abs(dev28[idx] - s[idx])
    assert np.all(diff <= bnd[idx]), (idx[diff > bnd[idx]], diff[diff > bnd[idx]], bnd[idx][diff > bnd[idx]])
    m = terms.shape[0]
    unit = max(m - 1, 1) * U64 * np.abs(terms[:, idx]).sum(0)
    return float(np.max(np.where(unit > 0, diff / np.where(unit > 0, unit, 1.0), 0.0))) if idx.size else 0.0


def _math_d2d(Minv_in, e, t, w, norm_scale=False):
    """Textbook J^T M J, J^T M e, e^T M e in float64 with M = inv(Minv_in) per term, and the absolute-value scale of each.
    norm_scale: |M| in the scale is replaced by max|M_ij| in every entry, the size of the rounding error of an inverse."""
    M = np.linalg.inv(Minv_in)
    m = len(e)
    J = np.zeros((m, 3, 6))
    tx, ty, tz = t[:, 0], t[:, 1], t[:, 2]
    J[:, 0, 1], J[:, 0, 2], J[:, 1, 0], J[:, 1, 2], J[:, 2, 0], J[:, 2, 1] = -tz, ty, tz, -tx, -ty, tx
    J[:, 0, 3] = J[:, 1, 4] = J[:, 2, 5] = -1.0
    H = w[:, None, None] * np.einsum("mip,mij,mjr->mpr", J, M, J)
    b = w[:, None] * np.einsum("mip,mij,mj->mp", J, M, e)
    err = w * np.einsum("mi,mij,mj->m", e, M, e)
    aJ, aM, ae = np.abs(J), np.abs(M), np.abs(e)
    if norm_scale:
        aM = np.broadcast_to(aM.max(axis=(1, 2))[:, None, None], aM.shape)
    sH = w[:, None, None] * np.einsum("mip,mij,mjr->mpr", aJ, aM, aJ)
    sb = w[:, None] * np.einsum("mip,mij,mj->mp", aJ, aM, ae)
    se = w * np.einsum("mi,mij,mj->m", ae, aM, ae)
    out = np.concatenate([H[:, TRIU[0], TRIU[1]], b, err[:, None]], 1)
    scale = np.concatenate([sH[:, TRIU[0], TRIU[1]], sb, se[:, None]], 1)
    return out, scale


def _cols(deriv):
    return slice(0, 28) if deriv else slice(27, 28)


def math_check_d2d(terms, C_B, C_A_rot, t, e, w, rel=1e-10, deriv=True):
    """GICP / VGICP: the restated terms [m, 28] against inv(C_B + R C_A R^T) and the textbook products in float64, within
    rel of each term's scale: |M| by max|M_ij| (the inverse of a matrix of condition number up to 1000 is exact to about
    1e-13 of its largest entry, not of each entry).  C_B, C_A_rot [m, 3, 3]; t, e [m, 3]; w [m].  Returns the worst ratio."""
    ref, scale = _math_d2d(C_B + C_A_rot, e, t, w, norm_scale=True)
    k = _cols(deriv)
    r = np.abs(terms[:, k] - ref[:, k]) / np.maximum(scale[:, k], np.finfo(F64).tiny)
    assert np.all(r <= rel), (np.unravel_index(np.argmax(r), r.shape), r.max())
    return float(r.max())


def math_check_ndt(T, src, terms):
    """NDT: the restated terms against C^-1 = inv(I - 0.999 n n^T), the Cauchy weight and the textbook products in float64.
    The restatement works in fp32: its e carries the rounding of the fp32 transform, relative to |R||a| + |t| + |mean|
    rather than to |e|, and each output is an expression of at most 32 fp32 roundings along any path.  Bound: gamma_32(u32)
    times the absolute-value scale computed with that |e| bound, and with the weight's sensitivity to e (relative change
    at most |de| / k)."""
    tab = terms.table
    sel_o, sel_i = np.nonzero(terms.used)
    if sel_o.size == 0:
        return 0.0
    row = terms.slot[sel_o, sel_i]
    a = np.ascontiguousarray(src[:, :3], F32)[sel_i].astype(F64)
    Tf = np.asarray(T, F64).astype(F32).astype(F64)
    t = np.einsum("ij,mj->mi", Tf[:3, :3], a) + Tf[:3, 3]
    mean = tab.mean[row].astype(F32).astype(F64)
    nv = tab.second[row, :3].astype(F32).astype(F64)
    nv = nv / np.linalg.norm(nv, axis=1, keepdims=True)   # the unit eigenvector the float normal rounds: C^-1 = I + 999 n n^T
    e = mean - t
    k = float(F32(terms.res))
    w = k * k / (k * k + (e * e).sum(1))
    C = np.eye(3)[None] - 0.999 * nv[:, :, None] * nv[:, None, :]
    ref, _ = _math_d2d(C, e, t, w)
    # scale: t (in J) and e replaced by their rounding envelopes |R||a| + |t| and that + |mean|
    t_abs = np.einsum("ij,mj->mi", np.abs(Tf[:3, :3]), np.abs(a)) + np.abs(Tf[:3, 3])
    e_abs = t_abs + np.abs(mean)
    _, scale = _math_d2d(C, e_abs, t_abs, w)
    scale = scale * (1.0 + np.linalg.norm(e_abs, axis=1) / k)[:, None]
    k = _cols(terms.deriv)
    vals = terms.vals[sel_o, sel_i]
    r = np.abs(vals[:, k] - ref[:, k]) / np.maximum(scale[:, k], np.finfo(F64).tiny)
    g = gamma(32, U32)
    assert np.all(r <= g), (np.unravel_index(np.argmax(r), r.shape), r.max(), g)
    return float(r.max() / g)


def _rot_cov(T, nrm):
    """R (I - 0.999 n n^T) R^T [m, 3, 3] in float64."""
    R = np.asarray(T, F64)[:3, :3]
    C = np.eye(3)[None] - 0.999 * nrm[:, :, None] * nrm[:, None, :]
    return np.einsum("ij,mjk,lk->mil", R, C, R)


def math_check_gicp(terms, src_nrm, tgt_nrm, T_lin, rel=1e-10):
    """GICP terms against inv(C_B + R C_A R^T) at the linearisation pose, within rel of each term's scale."""
    sel = terms.sel
    nb = np.asarray(tgt_nrm, F64)[terms.corr[sel], :3]
    C_B = np.eye(3)[None] - 0.999 * nb[:, :, None] * nb[:, None, :]
    return math_check_d2d(terms.vals[0, sel], C_B, _rot_cov(T_lin, np.asarray(src_nrm, F64)[sel, :3]),
                          np.stack(terms.t, 1), np.stack(terms.e, 1), np.ones(len(sel)), rel, terms.deriv)


def math_check_vgicp(terms, src, src_nrm, T_lin, rel=1e-10):
    """VGICP terms against inv(cov_B + R C_A R^T) at the linearisation pose with weight sqrt(n), within rel of each term's
    scale."""
    o, i = np.nonzero(terms.used)
    if o.size == 0:
        return 0.0
    row = terms.slot[o, i]
    tab = terms.table
    cv = tab.second[row]
    C_B = np.stack([cv[:, [0, 1, 2]], cv[:, [1, 3, 4]], cv[:, [2, 4, 5]]], 1)
    t = np.stack([terms.t[k][i] for k in range(3)], 1)
    e = tab.mean[row] - t
    return math_check_d2d(terms.vals[o, i], C_B, _rot_cov(T_lin, np.asarray(src_nrm, F64)[i, :3]), t, e,
                          np.sqrt(tab.count[row].astype(F64)), rel, terms.deriv)
