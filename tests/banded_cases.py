"""Shared bodies of the banded-solver tests: the combine / factor / solve / matvec kernels on ragged batches against LAPACK
(scipy.linalg.lapack dgbtrf / dgbtrs) and long-double products, through the CPU emulation of the kernels (tests/test_emu_banded.py)
and on the GPU (tests/test_gpu_1b_banded.py).

The sizes cover every n from 1 to 9, a warp's width, the largest per-m system of the 512 x 256 shallow-water problem (n = 1530) and
a batch past n = 1536, where the solve drops from 8 to 4 right-hand-side columns per CTA."""
import ctypes as C
import numpy as np
from scipy.linalg import lapack
from dedalus_b200 import lib as dlib

EPS = np.finfo(np.float64).eps
NRHS_CYCLE = (1, 8, 9, 33)           # one column, exactly one chunk, one past a chunk, more than 32 columns in the row swap
SMALL_NS = tuple(range(1, 10)) + (31, 32, 33, 100)


def small_batch():
    """n = 1 .. 9, 31, 32, 33, 100, right-hand-side counts cycling through NRHS_CYCLE."""
    return list(SMALL_NS), [NRHS_CYCLE[i % len(NRHS_CYCLE)] for i in range(len(SMALL_NS))]


class Batch:
    """A ragged batch: operators M, L in operator storage (ld0 = kl + ku + 1), right-hand sides v1, v2, and the offsets of each system."""

    def __init__(self, ns, nrhs, kl, ku, seed, diag_scale=1e-3):
        self.ns, self.nrhs, self.kl, self.ku = list(ns), list(nrhs), kl, ku
        self.ld0, self.ldf = kl + ku + 1, 2 * kl + ku + 1
        self.sys = (dlib.BandedSys * len(ns))()
        op = lu = pv = vec = 0
        for i, (n, r) in enumerate(zip(ns, nrhs)):
            s = self.sys[i]
            s.n, s.nrhs, s.op_off, s.lu_off, s.piv_off, s.vec_off = n, r, op, lu, pv, vec
            op += n * self.ld0; lu += n * self.ldf; pv += n; vec += n * r
        self.n_op, self.n_lu, self.n_piv, self.n_vec = op, lu, pv, vec
        rng = np.random.default_rng(seed)
        # band entries outside the matrix stay zero; the main diagonal is scaled down so that the pivot search moves rows
        self.m_ab, self.l_ab = np.zeros(op), np.zeros(op)
        for i, n in enumerate(ns):
            for ab in (self.m_ab, self.l_ab):
                band = self.op_band(ab, i)
                for d in range(-kl, ku + 1):               # A(i, i + d) at band[ku - d, i + d]
                    rows = np.arange(max(0, -d), min(n, n - d))
                    band[ku - d, rows + d] = rng.standard_normal(len(rows)) * (diag_scale if d == 0 else 1.0)
        self.v1, self.v2 = rng.standard_normal(vec), rng.standard_normal(vec)
        self.a0, self.b0 = 1.0, 0.37
        self.c1, self.c2 = 2.0, -0.5

    def op_band(self, ab, i):
        """View (ld0, n) of system i's operator storage: A(r, c) at [ku + r - c, c]."""
        s = self.sys[i]
        return ab[s.op_off:s.op_off + s.n * self.ld0].reshape(s.n, self.ld0).T

    def lu_band(self, lu, i):
        """View (ldf, n) of system i's factor storage, LAPACK's dgbtrf layout."""
        s = self.sys[i]
        return lu[s.lu_off:s.lu_off + s.n * self.ldf].reshape(s.n, self.ldf).T

    def vec(self, v, i):
        s = self.sys[i]
        return v[s.vec_off:s.vec_off + s.n * s.nrhs].reshape(s.n, s.nrhs)

    def band_matvec(self, band, x):
        """A x in long double from operator storage (ld0, n); x (n, r).  Also returns |A| |x|."""
        n = x.shape[0]
        x = x.astype(np.longdouble)
        y, ya = np.zeros_like(x), np.zeros_like(x)
        for d in range(-self.kl, self.ku + 1):            # y(i) += A(i, i + d) x(i + d)
            rows = np.arange(max(0, -d), min(n, n - d))
            a = band[self.ku - d, rows + d].astype(np.longdouble)[:, None]
            y[rows] += a * x[rows + d]
            ya[rows] += np.abs(a) * np.abs(x[rows + d])
        return y, ya


def _run(B, bt, alias_x=False):
    """combine -> factor -> solve -> matvec; returns host copies of lu, ipiv, x, ym, yl."""
    lib, P = B.lib, B.ptr
    kl, ku, nsys = bt.kl, bt.ku, len(bt.ns)
    sysb = B.dev(np.frombuffer(bytes(bt.sys), dtype=np.uint8).copy())
    m_d, l_d = B.dev(bt.m_ab), B.dev(bt.l_ab)
    lu = B.dev(np.full(bt.n_lu, np.nan))
    ipiv, info = B.dev(np.full(bt.n_piv, -7, dtype=np.int32)), B.dev(np.full(nsys, -1, dtype=np.int32))
    v1, v2 = B.dev(bt.v1), B.dev(bt.v2)
    x = v1 if alias_x else B.dev(np.full(bt.n_vec, np.nan))
    ym, yl = B.dev(np.full(bt.n_vec, np.nan)), B.dev(np.full(bt.n_vec, np.nan))
    lib.call("db_banded_combine", P(sysb), nsys, kl, ku, bt.a0, P(m_d), bt.b0, P(l_d), P(lu), B.stream)
    lu_comb = B.host(lu).copy()
    lib.call("db_banded_factor", P(sysb), nsys, kl, ku, P(lu), P(ipiv), P(info), B.stream)
    vc = dlib.VecComb(); vc.nvec = 2
    vc.vec[0], vc.vec[1] = P(v1).value, P(v2).value
    vc.coef[0], vc.coef[1] = bt.c1, bt.c2
    lib.call("db_banded_solve", P(sysb), nsys, kl, ku, max(bt.ns), max(bt.nrhs), P(lu), P(ipiv), C.byref(vc), P(x), B.stream)
    lib.call("db_banded_matvec", P(sysb), nsys, kl, ku, P(m_d), P(l_d), P(x), P(ym), P(yl), B.stream)
    assert not B.host(info).any(), B.host(info)
    return dict(comb=lu_comb, lu=B.host(lu).copy(), ipiv=B.host(ipiv).copy(), x=B.host(x).copy(),
                ym=B.host(ym).copy(), yl=B.host(yl).copy())


def _check_against_lapack(bt, r):
    kl, ku, a0, b0 = bt.kl, bt.ku, bt.a0, bt.b0
    for i, (n, nr) in enumerate(zip(bt.ns, bt.nrhs)):
        tag = dict(n=n, nrhs=nr, kl=kl, ku=ku)
        M, L = bt.op_band(bt.m_ab, i), bt.op_band(bt.l_ab, i)
        # combine: a0 M + b0 L below kl rows of fill-in that are exactly zero
        comb = bt.lu_band(r["comb"], i)
        assert not comb[:kl].any(), tag
        exact = a0 * M.astype(np.longdouble) + b0 * L.astype(np.longdouble)
        bound = 2 * EPS * (np.abs(a0 * M) + np.abs(b0 * L))
        assert np.all(np.abs(comb[kl:] - exact) <= bound), (tag, "combine")
        # factor: the same pivot rows and LU as LAPACK's band LU with partial pivoting
        ab_ref = np.zeros((bt.ldf, n)); ab_ref[kl:] = comb[kl:]
        lu_ref, piv_ref, info = lapack.dgbtrf(ab_ref, kl, ku)
        assert info == 0, tag
        piv = r["ipiv"][bt.sys[i].piv_off:bt.sys[i].piv_off + n]
        assert np.array_equal(piv, piv_ref), (tag, "pivots", np.flatnonzero(piv != piv_ref)[:5])
        lu = bt.lu_band(r["lu"], i)
        err = np.abs(lu - lu_ref).max() / np.abs(lu_ref).max()
        assert err <= 1e-13, (tag, "lu", err)
        # solve: LAPACK's dgbtrs on the kernel's own factors, and the backward error of x
        b = bt.c1 * bt.vec(bt.v1, i) + bt.c2 * bt.vec(bt.v2, i)
        x = bt.vec(r["x"], i)
        x_ref, info = lapack.dgbtrs(lu, kl, ku, b, piv)
        assert info == 0, tag
        err = np.abs(x - x_ref).max() / np.abs(x_ref).max()
        assert err <= 1e-12, (tag, "solve vs dgbtrs", err)
        ax, aax = bt.band_matvec(comb[kl:], x)              # the matrix the kernels factored
        # backward error per right-hand-side column, max|b - A x| / max(|A| |x| + |b|): partial pivoting bounds it by a small
        # multiple of n eps, but not the componentwise form (|L| |U| may exceed |A| by far: LAPACK's own solutions of these batches
        # reach 1e7 n eps componentwise at kl = 40, and stay below 0.3 n eps in this form)
        resid = np.abs(b.astype(np.longdouble) - ax)
        berr = float((resid.max(axis=0) / (aax + np.abs(b)).max(axis=0)).max())
        assert berr <= 50 * n * EPS, (tag, "backward error", berr)
        # matvec: M x and L x against long-double products
        for name, band in (("ym", M), ("yl", L)):
            exact, mag = bt.band_matvec(band, x)
            got = bt.vec(r[name], i)
            assert np.all(np.abs(got - exact) <= (kl + ku + 2) * EPS * mag), (tag, name)


def check_banded(B, kl, ku, ns, nrhs, seed=0, alias=True):
    """One ragged batch, LAPACK-accurate.  With `alias`, x is also solved in place over a right-hand-side vector, which the ABI
    allows: each CTA stages its right-hand-side columns in shared memory before it writes any of x; the result must be bitwise equal."""
    bt = Batch(ns, nrhs, kl, ku, seed)
    run = _run(B, bt)
    _check_against_lapack(bt, run)
    if alias:
        r = _run(B, bt, alias_x=True)
        assert r["x"].tobytes() == run["x"].tobytes(), ("x solved over v1", _first_difference(bt, r["x"], run["x"]))


def _first_difference(bt, a, b):
    bad = np.flatnonzero(a.view(np.uint64) != b.view(np.uint64))
    if not len(bad):
        return None
    for i in range(len(bt.ns)):
        s = bt.sys[i]
        if s.vec_off <= bad[0] < s.vec_off + s.n * s.nrhs:
            return dict(system=i, n=s.n, nrhs=s.nrhs)
