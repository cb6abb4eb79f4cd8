"""Shared bodies of the kernel-level tests of the sphere and shell paths: the dense batch kernels (csrc/dense.cu), the matrix transform
on the FP64 tensor cores (k_mmt_dmma) and on the FMA pipe (k_mmt), the ragged colatitude products, the pair combinations, the index
moves and the max reductions, through the CPU emulation of the kernels (tests/test_emu_curvilinear_kernels.py) and on the GPU
(tests/test_gpu_1d_curvilinear_kernels.py).

The references are restated from the contract in include/dedalus_b200.h in np.longdouble, not from the kernels.  Products are compared
componentwise, |got - ref| <= c k eps (|A| |x|) with k the contraction length; moves and maxima are compared exactly.  Output buffers
start as NaN, and what the contract does not write must still be NaN afterwards.  Every case asserts the edge it was written for.

B is a small array backend: B.dev(numpy) -> device array, B.ptr(device array) -> c_void_p, B.host(device array) -> numpy, B.lib, B.stream,
B.sms (streaming multiprocessors: the grid caps of the grid-stride kernels), B.dev_at(numpy, off) -> device array whose first element
sits 8 bytes past a 16-byte boundary when off is true, and on one otherwise."""
import ctypes as C
import os
import numpy as np
import pytest
from dedalus_b200 import lib as dlib

EPS = np.finfo(np.float64).eps
LD = np.longdouble
DN_THREADS = 256          # csrc/dense.cu: threads of the factorisation's CTA
DENSE_SMEM_MAX_N = 800    # csrc/dense.cu: 32 columns of n doubles fit in 200 KB of shared memory up to here


def _nan(shape, dtype=np.float64):
    return np.full(shape, np.nan, dtype=dtype)


def _struct_bytes(arr):
    return np.frombuffer(bytes(arr), dtype=np.uint8).copy()


# ------------------------------------------------------------------------------------------------------------------------------
# csrc/dense.cu
# ------------------------------------------------------------------------------------------------------------------------------
def lu_reference(A, gap=1e-6, skip_gap=()):
    """Unblocked right-looking LU with partial pivoting in long double: pivot = largest |a| of the column, lowest row on ties.
    Returns (lu, ipiv).  With `gap`, asserts that the runner-up of every pivot search (steps in skip_gap excepted) is smaller by that
    relative margin, so that a float64 factorisation must choose the same rows."""
    a = np.array(A, dtype=LD)
    n = a.shape[0]
    ipiv = np.zeros(n, dtype=np.int32)
    for k in range(n):
        col = np.abs(a[k:, k])
        p = int(np.argmax(col))                                  # the first maximum: the lowest row
        if gap and k not in skip_gap and len(col) > 1:
            assert np.delete(col, p).max() <= (1 - gap) * col[p], ("pivot candidates too close", k)
        p += k
        ipiv[k] = p
        if p != k:
            a[[k, p]] = a[[p, k]]
        a[k + 1:, k] /= a[k, k]
        a[k + 1:, k + 1:] -= np.outer(a[k + 1:, k], a[k, k + 1:])
    return a, ipiv


def _permute_rows(A, ipiv):
    """P A for the interchanges ipiv applied in ascending order."""
    pa = np.array(A, dtype=LD)
    for k, p in enumerate(ipiv):
        if p != k:
            pa[[k, p]] = pa[[p, k]]
    return pa


def dense_factor(B, A):
    """db_dense_factor on the batch A (nsys, n, n); returns host copies of lu, ipiv, info."""
    nsys, n = A.shape[:2]
    lu, ipiv, info = B.dev(A), B.dev(np.full((nsys, n), -7, dtype=np.int32)), B.dev(np.full(nsys, -1, dtype=np.int32))
    B.lib.call("db_dense_factor", nsys, n, B.ptr(lu), B.ptr(ipiv), B.ptr(info), B.stream)
    return B.host(lu).copy(), B.host(ipiv).copy(), B.host(info).copy()


def check_factor_against_reference(A, lu, ipiv, skip_gap=()):
    """One healthy system: the pivot rows of the long-double LU exactly, its factors within a growth-aware bound, and P A = L U."""
    n = A.shape[0]
    lu_ref, piv_ref = lu_reference(A, skip_gap=skip_gap)
    assert np.array_equal(ipiv, piv_ref), ("pivots", n, np.flatnonzero(ipiv != piv_ref)[:5])
    Lr, Ur = np.tril(lu_ref, -1) + np.eye(n, dtype=LD), np.triu(lu_ref)
    # P A = L U + E with |E| <= gamma_n |L| |U| (Higham, Accuracy and Stability, thm 9.3); 2 n eps covers gamma_n and the reciprocal
    # pivot the kernel multiplies by instead of dividing
    Lg, Ug = np.tril(lu, -1).astype(LD) + np.eye(n, dtype=LD), np.triu(lu).astype(LD)
    resid = np.abs(_permute_rows(A, ipiv) - Lg @ Ug)
    bound = 2 * n * EPS * (np.abs(Lg) @ np.abs(Ug))
    assert np.all(resid <= bound + np.finfo(np.float64).tiny), ("P A = L U", n, float((resid / (bound + 1e-300)).max()))
    # the factors themselves: the error of an entry grows with the conditioning of the leading blocks, measured here by the
    # largest entry of U^{-1} (growth of the back-substitution) times the largest entry of U
    growth = float(np.abs(Ur).max() / np.abs(np.diag(Ur)).min())
    err = float(np.abs(lu - lu_ref).max() / np.abs(lu_ref).max())
    assert err <= 8 * n * EPS * max(growth, 1.0), ("factors", n, err, growth)


def pivoting_matrix(rng, n):
    """Standard-normal entries with the diagonal scaled down, so that nearly every pivot search moves a row."""
    A = rng.standard_normal((n, n))
    A[np.arange(n), np.arange(n)] *= 1e-3
    return A


def check_dense_factor_sizes(B, ns):
    """Healthy systems of each size in ns (one launch per size, two systems per launch)."""
    for n in ns:
        rng = np.random.default_rng(1000 + n)
        A = np.stack([pivoting_matrix(rng, n), rng.standard_normal((n, n))])
        lu, ipiv, info = dense_factor(B, A)
        assert not info.any(), (n, info)
        if n > 1:
            assert (ipiv[0] != np.arange(n)).any(), "the case is meant to interchange rows"
        for s in range(2):
            check_factor_against_reference(A[s], lu[s], ipiv[s])


def check_dense_factor_ties(B):
    """|a| equal at rows 2, 5 and 300 of the first column: threads 2, 5 and 300 - 256 = 44 of the strided search hold the same
    candidate value, and the tree reduction must return the lowest row."""
    n = 304
    assert n > DN_THREADS + 44
    rng = np.random.default_rng(7)
    A = pivoting_matrix(rng, n)
    A[:, 0] *= 0.1
    A[2, 0], A[5, 0], A[300, 0] = 3.0, -3.0, 3.0
    assert np.abs(A[:, 0]).max() == 3.0 and (np.abs(A[:, 0]) == 3.0).sum() == 3
    lu, ipiv, info = dense_factor(B, A[None])
    assert info[0] == 0
    assert ipiv[0, 0] == 2, ipiv[0, :3]
    check_factor_against_reference(A, lu[0], ipiv[0], skip_gap=(0,))


def padded_system(rng, n0, n):
    """A block of size n0 completed to n with identity rows and columns, as the shell systems pad every degree to a common n."""
    A = np.zeros((n, n))
    A[:n0, :n0] = pivoting_matrix(rng, n0)
    A[np.arange(n0, n), np.arange(n0, n)] = 1.0
    return A


class DenseVectors:
    """Right-hand-side columns of a dense batch: system s holds ncols[s] columns of n rows at vec_off[s], with `gap` doubles that
    belong to no system between consecutive systems (they must never be written)."""

    def __init__(self, n, ncols, gap=3):
        self.n, self.ncols = n, list(ncols)
        self.sys = (dlib.DenseSys * len(ncols))()
        off = gap
        for s, nc in enumerate(ncols):
            self.sys[s].ncols, self.sys[s].vec_off = nc, off
            off += n * nc + gap
        self.size = off
        self.owned = np.zeros(off, dtype=bool)
        for s, nc in enumerate(ncols):
            self.owned[self.sys[s].vec_off:self.sys[s].vec_off + n * nc] = True

    def view(self, v, s):
        o = self.sys[s].vec_off
        return v[o:o + self.n * self.ncols[s]].reshape(self.n, self.ncols[s])

    def random(self, rng):
        v = _nan(self.size)
        v[self.owned] = rng.standard_normal(int(self.owned.sum()))
        return v

    def check_unowned_nan(self, v, what):
        assert np.isnan(v[~self.owned]).all(), (what, "wrote outside the systems' rows")
        assert not np.isnan(v[self.owned]).any(), (what, "left rows of a system unwritten")


def dense_solve(B, dv, lu, ipiv, vecs, coefs, smem):
    """db_dense_solve with DB_DENSE_SOLVE_SMEM unset (smem = None) or "0"; returns the host copy of x (NaN where nothing is written).
    Asserts which template instance the launcher's size rule selects."""
    n, nsys = dv.n, len(dv.ncols)
    uses_smem = smem is None and n <= DENSE_SMEM_MAX_N
    assert uses_smem == (smem != "0" and n * 32 * 8 <= 200 * 1024)
    vc = dlib.VecComb()
    vc.nvec = len(vecs)
    keep = [B.dev(v) for v in vecs]
    for k, (d, c) in enumerate(zip(keep[:16], coefs)):
        vc.vec[k], vc.coef[k] = B.ptr(d).value, c
    x = B.dev(_nan(dv.size))
    sysb, lud, pivd = B.dev(_struct_bytes(dv.sys)), B.dev(lu), B.dev(ipiv)
    old = os.environ.pop("DB_DENSE_SOLVE_SMEM", None)
    try:
        if smem is not None:
            os.environ["DB_DENSE_SOLVE_SMEM"] = smem
        B.lib.call("db_dense_solve", B.ptr(sysb), nsys, n, max(max(dv.ncols), 1), B.ptr(lud), B.ptr(pivd), C.byref(vc), B.ptr(x), B.stream)
        out = B.host(x).copy()
    finally:
        os.environ.pop("DB_DENSE_SOLVE_SMEM", None)
        if old is not None:
            os.environ["DB_DENSE_SOLVE_SMEM"] = old
    return out, uses_smem


def check_solution(A, b, x, tag, c=8):
    """Normwise backward error of every column, max|b - A x| / (max(|A| |x|) + max|b|) <= c n eps (partial pivoting bounds this
    form, not the componentwise one).  A, b long double."""
    n = A.shape[0]
    if x.shape[1] == 0:
        return
    xl = x.astype(LD)
    resid = np.abs(b - A @ xl).max(axis=0)
    scale = (np.abs(A) @ np.abs(xl)).max(axis=0) + np.abs(b).max(axis=0)
    berr = float((resid / scale).max())
    assert berr <= c * n * EPS, (tag, "backward error", berr / (n * EPS))


def check_dense_solve(B, n, ncols, nvec, seed, mats=None, smem_modes=(None, "0")):
    """Factor and solve a batch with the given column counts and `nvec` right-hand-side terms, in both template instances of the
    solve: backward error of every column against the long-double combination, nothing written outside the systems, and the two
    instances bitwise equal (they perform the same operations in the same order; only where the columns live differs)."""
    rng = np.random.default_rng(seed)
    nsys = len(ncols)
    A = np.stack([pivoting_matrix(rng, n) for _ in range(nsys)]) if mats is None else mats
    lu, ipiv, info = dense_factor(B, A)
    assert not info.any(), info
    dv = DenseVectors(n, ncols)
    vecs = [dv.random(rng) for _ in range(nvec)]
    coefs = [(-1.0) ** k * 10.0 ** (((k + 2) % 5) - 2) * (1 + 0.1 * k) for k in range(nvec)]  # 1, -11, 120, ...: mixed sign and magnitude
    if nvec > 1:
        assert min(coefs) < 0 < max(coefs) and max(np.abs(coefs)) / min(np.abs(coefs)) >= 10
    runs = {}
    for smem in smem_modes:
        x, used = dense_solve(B, dv, lu, ipiv, vecs, coefs, smem)
        runs[smem] = x
        dv.check_unowned_nan(x, dict(n=n, smem=smem))
        for s, nc in enumerate(ncols):
            b = sum(LD(c) * dv.view(v, s).astype(LD) for c, v in zip(coefs, vecs))
            # the combination is rounded once per term: it enters the bound through |b|
            check_solution(A[s].astype(LD), b, dv.view(x, s), dict(n=n, ncols=nc, nvec=nvec, smem=smem), c=8 + nvec)
    if len(smem_modes) == 2:
        assert runs[None].tobytes() == runs["0"].tobytes(), "the two template instances of the solve differ"
    return A, lu, ipiv, dv, vecs, coefs, runs[smem_modes[0]]


def check_dense_solve_ragged(B, n=39):
    """Column counts 0, 1, 31, 32, 33, 64, 65 and 200 in one launch: empty systems, a full warp, one past it, several CTAs per system."""
    ncols = [0, 1, 31, 32, 33, 64, 65, 200]
    assert 0 in ncols and any(c % 32 == 0 and c > 0 for c in ncols) and any(c % 32 == 1 and c > 32 for c in ncols)
    check_dense_solve(B, n, ncols, nvec=2, seed=11)


def check_dense_solve_nvec(B):
    """1, 2 and 16 right-hand-side terms; 0 and 17 are rejected on the host with the documented message, before any launch."""
    for nvec in (1, 2, 16):
        check_dense_solve(B, 23, [5, 40], nvec=nvec, seed=20 + nvec)
    dv = DenseVectors(5, [3])
    lu, ipiv = np.eye(5)[None], np.arange(5, dtype=np.int32)[None]
    for nvec in (0, 17):
        vc = dlib.VecComb(); vc.nvec = nvec
        x, sysb, lud, pivd = B.dev(_nan(dv.size)), B.dev(_struct_bytes(dv.sys)), B.dev(lu), B.dev(ipiv)
        with pytest.raises(dlib.DedalusB200Error, match=r"code 1.*dense_solve: 1\.\.16 right-hand-side vectors"):
            B.lib.call("db_dense_solve", B.ptr(sysb), 1, 5, 3, B.ptr(lud), B.ptr(pivd), C.byref(vc), B.ptr(x), B.stream)
        assert np.isnan(B.host(x)).all()


def check_dense_solve_remainders(B):
    """n = 4k + {0, 1, 2, 3} against the four-chain unroll of both sweeps, from n = 1 up."""
    for n in (1, 2, 3, 4, 5, 6, 7, 8, 9, 31, 32, 33):
        check_dense_solve(B, n, [3, 33], nvec=2, seed=40 + n)


def check_dense_solve_long_cycle(B, n=37):
    """A matrix whose factorisation interchanges row k with row k + 1 at every step: the row-swap loop of the solve must apply the
    interchanges in ascending order (the composition is an n-cycle, and any other order is a different permutation)."""
    rng = np.random.default_rng(5)
    A = 0.01 * rng.standard_normal((n, n))
    A[np.arange(1, n), np.arange(n - 1)] = 10.0
    A[0, n - 1] = 10.0
    out = check_dense_solve(B, n, [7, 33], nvec=1, seed=6, mats=A[None].repeat(2, axis=0))
    ipiv = out[2]
    assert np.array_equal(ipiv[0, :n - 1], np.arange(1, n)), ipiv[0]


def check_dense_padded(B, n0=23, n=39):
    """Identity-padded systems: no pivot crosses into the pad, the pad of L and U is the identity, and with a single term of
    coefficient 1 the pad of the solution is the pad of the right-hand side bit for bit."""
    rng = np.random.default_rng(9)
    A = np.stack([padded_system(rng, n0, n), padded_system(rng, 1, n), padded_system(rng, n - 1, n)])
    sizes = (n0, 1, n - 1)
    out = check_dense_solve(B, n, [33, 2, 5], nvec=1, seed=10, mats=A)
    lu, ipiv, dv, vecs, coefs, x = out[1], out[2], out[3], out[4], out[5], out[6]
    assert coefs == [1.0]
    for s, k in enumerate(sizes):
        assert (ipiv[s, :k] < k).all() and np.array_equal(ipiv[s, k:], np.arange(k, n)), (s, ipiv[s])
        assert np.array_equal(lu[s, k:, :], np.eye(n)[k:]) and not lu[s, :k, k:].any(), s
        assert dv.view(x, s)[k:].tobytes() == dv.view(vecs[0], s)[k:].tobytes(), (s, "pad of the solution")


def check_dense_info(B, n=33):
    """Singular and non-finite systems next to healthy ones in one launch: info counts the zero / non-finite pivots (a zero column
    gives 1, two give 2, a NaN or an Inf entry gives at least 1) and the healthy systems keep info = 0 and correct factors."""
    rng = np.random.default_rng(13)
    A = np.stack([pivoting_matrix(rng, n) for _ in range(6)])
    A[1, :, 4] = 0.0
    A[2, :, 7] = 0.0; A[2, :, 20] = 0.0
    A[3, 10, 12] = np.nan
    A[4, 10, 12] = np.inf
    lu, ipiv, info = dense_factor(B, A)
    assert info[0] == 0 and info[5] == 0, info
    assert info[1] == 1 and info[2] == 2, info
    assert info[3] >= 1 and info[4] >= 1, info
    for s in (0, 5):
        check_factor_against_reference(A[s], lu[s], ipiv[s])
    return A


def check_singular_matrix_raises(B_unused=None):
    """matsolvers.B200Dense raises its error on a singular and on a non-finite matrix, and ShellSystems.check_info raises when a
    system of the batch reports a bad pivot."""
    import scipy.sparse as sp
    from dedalus_b200 import matsolvers
    rng = np.random.default_rng(3)
    A = rng.standard_normal((9, 9))
    matsolvers.B200Dense(sp.csr_matrix(A))
    for bad in ("zero", "nan"):
        Ab = A.copy()
        if bad == "zero":
            Ab[:, 3] = 0.0
        else:
            Ab[2, 3] = np.nan
        with pytest.raises(dlib.DedalusB200Error, match="matrix is singular to working precision"):
            matsolvers.B200Dense(sp.csr_matrix(Ab))


def shell_systems():
    """The per-degree dense systems (ShellSystems) of the 16 x 8 x 6 shell-convection problem, as an SBDF2 solver builds them."""
    import dedalus_b200 as d3
    from dedalus_b200 import examples
    solver = examples.shell_convection(16, 8, 6)['problem'].build_solver(d3.SBDF2)
    solver._init_device()
    solver._prepare_batches(1.0, 0.5)
    return solver.bset


def check_shell_systems_info_raises(bset):
    """ShellSystems.check_info on a batch whose operator L has a zero column in one system."""
    import torch
    bset.factor(0, 1.0, 0.5)
    bset.check_info()
    keep = bset.L_t.clone(), bset.M_t.clone()
    try:
        bset.L_t[2, :, 1] = 0.0; bset.M_t[2, :, 1] = 0.0
        bset.factor(0, 1.0, 0.5)
        assert int(bset.info[2]) == 1 and int((bset.info != 0).sum()) == 1
        with pytest.raises(dlib.DedalusB200Error, match="1 shell pencil systems hit a zero / non-finite pivot"):
            bset.check_info()
    finally:
        bset.L_t.copy_(keep[0]); bset.M_t.copy_(keep[1])


def _csr(mats):
    """CSR of a batch (nsys, n, n) as db_csr_matvec takes it: ptr (nsys, n + 1) with offsets global over the batch."""
    nsys, n = mats.shape[:2]
    nz = mats != 0
    counts = nz.sum(axis=2)
    ptr = np.zeros((nsys, n + 1), dtype=np.int64)
    ptr[:, 1:] = np.cumsum(counts, axis=1)
    ptr += np.concatenate([[0], np.cumsum(counts.sum(axis=1))[:-1]])[:, None]
    s_, r_, c_ = np.nonzero(nz)
    col, val = c_.astype(np.int32), mats[s_, r_, c_]
    if len(val) == 0:                                      # keep the arrays addressable
        col, val = np.zeros(1, dtype=np.int32), np.zeros(1)
    return ptr, col, val


def _check_product(got, Mx, x, k, what):
    """got = Mx x componentwise: |got - ref| <= (k + 1) eps (|M| |x|), k = longest row of the product."""
    ref = Mx.astype(LD) @ x.astype(LD)
    mag = np.abs(Mx).astype(LD) @ np.abs(x).astype(LD)
    assert np.all(np.abs(got - ref) <= (k + 1) * EPS * mag), (what, float((np.abs(got - ref) / (mag + 1e-300)).max() / EPS))


def check_dense_and_csr_matvec(B, Am, Bm, ncols, seed=0):
    """db_dense_matvec and db_csr_matvec on the operators Am, Bm (nsys, n, n): ya only, yb only and both, against long-double
    products; nothing outside the systems' rows is written; an output that is not asked for is not touched."""
    nsys, n = Am.shape[:2]
    rng = np.random.default_rng(seed)
    dv = DenseVectors(n, ncols)
    xh = dv.random(rng)
    sysb, x = B.dev(_struct_bytes(dv.sys)), B.dev(xh)
    Ad, Bd = B.dev(Am), B.dev(Bm)
    csr_a, csr_b = [tuple(B.dev(t) for t in _csr(m)) for m in (Am, Bm)]
    P = B.ptr
    for kind in ("dense", "csr"):
        for want_a, want_b in ((True, False), (False, True), (True, True)):
            ya, yb = B.dev(_nan(dv.size)), B.dev(_nan(dv.size))
            pa, pb = (P(ya) if want_a else None), (P(yb) if want_b else None)
            if kind == "dense":
                B.lib.call("db_dense_matvec", P(sysb), nsys, n, P(Ad) if want_a else None, P(Bd) if want_b else None, P(x), pa, pb, B.stream)
            else:
                # an absent matrix: NULL ptr / col / val with its y NULL
                a3 = [P(t) for t in csr_a] if want_a else [None] * 3
                b3 = [P(t) for t in csr_b] if want_b else [None] * 3
                B.lib.call("db_csr_matvec", P(sysb), nsys, n, *a3, *b3, P(x), pa, pb, B.stream)
            for want, y, Mx, name in ((want_a, ya, Am, "ya"), (want_b, yb, Bm, "yb")):
                yh = B.host(y)
                if not want:
                    assert np.isnan(yh).all(), (kind, name, "written though not asked for")
                    continue
                dv.check_unowned_nan(yh, (kind, name))
                for s in range(nsys):
                    k = n if kind == "dense" else int((Mx[s] != 0).sum(axis=1).max())
                    _check_product(dv.view(yh, s), Mx[s], dv.view(xh, s), k, (kind, name, s, want_a, want_b))


def check_matvec_edges(B, n=39):
    """Systems of 0 columns, n * ncols past 16 * 256 (the y-grid stride loops), CSR with empty rows and an empty matrix."""
    ncols = [0, 1, 33, 200]
    assert 0 in ncols and n * max(ncols) > 16 * 256
    rng = np.random.default_rng(17)
    Am = rng.standard_normal((len(ncols), n, n))
    Bm = rng.standard_normal((len(ncols), n, n)) * (rng.random((len(ncols), n, n)) < 0.1)
    Bm[:, 5, :] = 0.0; Bm[3, n - 1, :] = 0.0; Bm[0, 0, :] = 0.0          # empty rows: the first, the last, one inside
    Bm[2] = 0.0                                                           # a system whose matrix is empty
    ptr = _csr(Bm)[0]
    assert ptr[2, 0] == ptr[2, -1] and (np.diff(ptr, axis=1) == 0).any(axis=1).all()
    check_dense_and_csr_matvec(B, Am, Bm, ncols, seed=18)
    # a batch whose second operator is empty everywhere: ptr all equal
    Z = np.zeros_like(Am)
    assert len(set(_csr(Z)[0].ravel())) == 1
    check_dense_and_csr_matvec(B, Am, Z, ncols, seed=19)


def check_shell_operator_matvec(B, bset):
    """M and L of a shell-convection problem's pencil systems (identity-padded, mostly zeros): CSR, dense and long-double
    products agree."""
    Mall, Lall = bset.M_t.cpu().numpy(), bset.L_t.cpu().numpy()
    nsys, n = Mall.shape[:2]
    assert (nsys, n) == (bset.nsys, bset.n)
    density = (Lall != 0).mean()
    assert density < 0.5, density
    assert any(np.array_equal(Lall[s, -1], np.eye(n)[-1]) for s in range(nsys)), "no identity-padded system in the batch"
    ncols = [2 * (s + 1) for s in range(nsys)]
    check_dense_and_csr_matvec(B, Mall, Lall, ncols, seed=23)
    return n


def check_dense_combine(B, nsys, n):
    """out = a0 M + b0 L elementwise, at a0 = 0, b0 = 0 and both nonzero: one rounding of the fused product-sum at most."""
    rng = np.random.default_rng(29)
    M, L = rng.standard_normal((nsys, n, n)), rng.standard_normal((nsys, n, n))
    Md, Ld = B.dev(M), B.dev(L)
    for a0, b0 in ((0.0, 0.37), (1.5, 0.0), (1.0, -0.25), (0.0, 0.0)):
        out = B.dev(_nan((nsys, n, n)))
        B.lib.call("db_dense_combine", nsys, n, a0, B.ptr(Md), b0, B.ptr(Ld), B.ptr(out), B.stream)
        got = B.host(out)
        exact = LD(a0) * M.astype(LD) + LD(b0) * L.astype(LD)
        bound = 2 * EPS * (np.abs(a0 * M) + np.abs(b0 * L))
        assert np.all(np.abs(got - exact) <= bound), (a0, b0)
        if a0 == 0.0:
            assert np.array_equal(got, b0 * L + 0.0)
        if b0 == 0.0:
            assert np.array_equal(got, a0 * M + 0.0)
    return nsys * n * n


# ------------------------------------------------------------------------------------------------------------------------------
# db_mmt_apply: k_mmt_dmma (FP64 tensor cores) and k_mmt (FMA pipe)
# ------------------------------------------------------------------------------------------------------------------------------
def mmt_apply(B, mat, x, expect, offset=None):
    """db_mmt_apply(mat (m, n), x (outer, n, inner)) into a NaN buffer; `expect` in ("dmma", "fma") is asserted against the launch
    counter of the tensor-core kernel.  offset = "mat" | "in" | "out": that array starts 8 bytes past a 16-byte boundary."""
    m, n = mat.shape
    outer, n2, inner = x.shape
    assert n2 == n
    md, xd, od = B.dev_at(mat, offset == "mat"), B.dev_at(x, offset == "in"), B.dev_at(_nan((outer, m, inner)), offset == "out")
    ptrs = [B.ptr(t).value for t in (md, xd, od)]
    aligned = all(p % 16 == 0 for p in ptrs)
    rule = aligned and n % 2 == 0 and inner % 2 == 0
    assert rule == (expect == "dmma"), (dict(m=m, n=n, inner=inner, aligned=aligned), expect)
    before = B.lib._raw_db_mmt_dmma_launches()
    B.lib.call("db_mmt_apply", ptrs[0], m, n, ptrs[1], ptrs[2], outer, inner, B.stream)
    got = B.host(od).copy()
    assert B.lib._raw_db_mmt_dmma_launches() - before == (1 if expect == "dmma" else 0), (expect, m, n, inner)
    return got


def check_mmt(B, m, n, outer, inner, expect, offset=None, seed=0):
    """out(o, i, r) = sum_j mat[i][j] in(o, j, r) against the long-double contraction, componentwise."""
    rng = np.random.default_rng(seed + 7 * m + 13 * n + inner)
    mat = rng.standard_normal((m, n)) * 10.0 ** rng.integers(-3, 4, size=(m, 1))      # rows of very different scale
    x = rng.standard_normal((outer, n, inner))
    got = mmt_apply(B, mat, x, expect, offset)
    ref = np.einsum('ij,ojr->oir', mat.astype(LD), x.astype(LD))
    mag = np.einsum('ij,ojr->oir', np.abs(mat).astype(LD), np.abs(x).astype(LD))
    assert not np.isnan(got).any(), (m, n, inner, "unwritten output")
    assert np.all(np.abs(got - ref) <= (n + 1) * EPS * mag), (dict(m=m, n=n, outer=outer, inner=inner, expect=expect, offset=offset),
                                                              float((np.abs(got - ref) / mag).max() / EPS))
    return got


MMT_M = (1, 7, 8, 63, 64, 65, 130)
MMT_N = (2, 4, 14, 16, 18, 30, 32, 34, 256)
MMT_INNER = (2, 62, 64, 66, 130)


def mmt_tile_edge_shapes():
    """(m, n, outer, inner) around the 64 x 64 tiles and the k blocks of 16: every m, every n and every inner appears, without the
    full cross product."""
    shapes = []
    for i, m in enumerate(MMT_M):
        shapes.append((m, MMT_N[i % len(MMT_N)], 1 + 2 * (i % 2), MMT_INNER[i % len(MMT_INNER)]))
    for i, n in enumerate(MMT_N):
        shapes.append((MMT_M[(i + 3) % len(MMT_M)], n, 1 + 2 * ((i + 1) % 2), MMT_INNER[(i + 2) % len(MMT_INNER)]))
    for i, inner in enumerate(MMT_INNER):
        shapes.append((MMT_M[(2 * i + 1) % len(MMT_M)], MMT_N[(3 * i + 2) % len(MMT_N)], 3, inner))
    shapes = sorted(set(shapes))
    assert {s[0] for s in shapes} == set(MMT_M) and {s[1] for s in shapes} == set(MMT_N) and {s[3] for s in shapes} == set(MMT_INNER)
    assert {s[2] for s in shapes} == {1, 3}
    return shapes


def check_mmt_dispatch(B):
    """Even n and inner with 16-byte aligned arrays run on the tensor cores; an odd n, an odd inner or any array 8 bytes off the
    boundary runs the FMA-pipe kernel, and both give the product within the same bound."""
    check_mmt(B, 65, 18, 3, 66, "dmma")
    check_mmt(B, 65, 17, 3, 66, "fma")
    check_mmt(B, 65, 18, 3, 65, "fma")
    for which in ("mat", "in", "out"):
        check_mmt(B, 65, 18, 3, 66, "fma", offset=which)


def check_mmt_jacobi_matrices(B, Nr, Nrg, k=0):
    """The matrices of the radial Jacobi transform of a shell basis with Nr modes on Nrg grid points (JacobiMatrixTransform: forward
    Nr x Nrg, backward Nrg x Nr), applied along the middle axis as the shell transforms do (outer = angular components, inner = 1 for
    r-last data is not this path: here the radial axis is followed by a trailing axis of 18)."""
    from dedalus_b200.transforms import JacobiMatrixTransform
    T = JacobiMatrixTransform(Nrg, Nr, -0.5 + k, -0.5 + k, -0.5, -0.5)
    assert T.forward_matrix.shape == (Nr, Nrg) and T.backward_matrix.shape == (Nrg, Nr)
    rng = np.random.default_rng(Nr)
    for mat in (T.forward_matrix, T.backward_matrix):
        m, n = mat.shape
        x = rng.standard_normal((2, n, 18))
        got = mmt_apply(B, mat, x, "dmma" if n % 2 == 0 else "fma")
        ref = np.einsum('ij,ojr->oir', mat.astype(LD), x.astype(LD))
        mag = np.einsum('ij,ojr->oir', np.abs(mat).astype(LD), np.abs(x).astype(LD))
        assert np.all(np.abs(got - ref) <= (n + 1) * EPS * mag), (Nr, Nrg, mat.shape, float((np.abs(got - ref) / (mag + 1e-300)).max() / EPS))


# ------------------------------------------------------------------------------------------------------------------------------
# db_ragged_matvec
# ------------------------------------------------------------------------------------------------------------------------------
RG_ROW_CAP = 64 * 8        # csrc/pointwise.cu: rows one pass of the grid covers (64 y-blocks of RG_ROWS = 8 warps)


def ragged_reference(mats, entries, x, out_shape):
    """The header's formula in long double; returns (ref, magnitude, written mask)."""
    N0, N1o, N2o, N3 = out_shape
    ref, mag, written = np.zeros(out_shape, dtype=LD), np.zeros(out_shape, dtype=LD), np.zeros(out_shape, dtype=bool)
    xl = x.astype(LD)
    for e in entries:
        mat = mats[e.mat_off:e.mat_off + e.nrow * e.ncol].reshape(e.nrow, e.ncol).astype(LD)
        in_rows = e.in_row0 + np.arange(e.ncol) * e.in_step
        out_rows = e.out_row0 + np.arange(e.nrow) * e.out_step
        for i in range(e.nm):
            assert not written[:, e.out_i0 + i, out_rows].any(), "the case's entries overlap"
            written[:, e.out_i0 + i, out_rows] = True
            if e.zero:
                continue
            src = xl[:, e.in_i0 + i][:, in_rows]                                   # (N0, ncol, N3)
            ref[:, e.out_i0 + i, out_rows] = np.einsum('kj,ojr->okr', mat, src)
            mag[:, e.out_i0 + i, out_rows] = np.einsum('kj,ojr->okr', np.abs(mat), np.abs(src))
    return ref, mag, written


def check_ragged(B, entries_spec, N0, N3, seed=0):
    """entries_spec: list of dict(nrow, ncol, nm, in_step, out_step, zero).  The entries are laid out by hand: each writes its own
    rows of the output, next to the rows of its neighbours, with unwritten rows in between; N1 and N2 differ between input and output
    and the matrices start at offsets that are multiples of nothing."""
    rng = np.random.default_rng(seed)
    ents = (dlib.RaggedEntry * len(entries_spec))()
    mat_off, in_i, out_i = 3, 1, 0
    in_rows_needed = out_rows_needed = 0
    for e, sp in zip(ents, entries_spec):
        e.nrow, e.ncol, e.nm, e.in_step, e.out_step, e.zero = sp["nrow"], sp["ncol"], sp["nm"], sp["in_step"], sp["out_step"], sp.get("zero", 0)
        e.mat_off = mat_off; mat_off += e.nrow * e.ncol + 5
        e.in_i0, e.out_i0 = in_i, out_i
        in_i += e.nm; out_i += e.nm
        e.in_row0 = 2 if e.in_step > 0 else 2 + e.ncol - 1
        e.out_row0 = 1 if e.out_step > 0 else 1 + e.nrow - 1
        in_rows_needed, out_rows_needed = max(in_rows_needed, e.ncol + 3), max(out_rows_needed, e.nrow + 2)
    N1i, N1o, N2i = in_i + 1, out_i + 3, in_rows_needed
    N2o = out_rows_needed + (out_rows_needed == N2i)
    assert N1i != N1o and N2i != N2o and any(e.mat_off % 2 for e in ents)
    mats = rng.standard_normal(mat_off)
    x = rng.standard_normal((N0, N1i, N2i, N3))
    out = B.dev(_nan((N0, N1o, N2o, N3)))
    md, ed, xd = B.dev(mats), B.dev(_struct_bytes(ents)), B.dev(x)
    B.lib.call("db_ragged_matvec", B.ptr(md), B.ptr(ed), len(ents), max(e.nrow for e in ents), B.ptr(xd), B.ptr(out),
               N0, N1i, N2i, N1o, N2o, N3, B.stream)
    got = B.host(out)
    ref, mag, written = ragged_reference(mats, ents, x, got.shape)
    assert np.isnan(got[~written]).all(), "rows outside out_row0 + k * out_step were written"
    assert not np.isnan(got[written]).any(), "rows of an entry left unwritten"
    kmax = max(e.ncol for e in ents)
    bad = np.abs(got[written] - ref[written]) > (kmax + 6) * EPS * mag[written]       # + 5 additions of the shuffle tree
    assert not bad.any(), (entries_spec, N0, N3, int(bad.sum()))
    for e in ents:
        if e.zero:
            rows = e.out_row0 + np.arange(e.nrow) * e.out_step
            assert not got[:, e.out_i0:e.out_i0 + e.nm][:, :, rows].any()


def check_ragged_shapes(B, big=True):
    """Rows around the warp count of a CTA and the grid's row cap, contraction lengths around a warp, right-hand-side counts
    N0 * nm * N3 of 1, 7, 8, 9, 17 and 78 around the RG_C = 8 columns of a pass, both steps of both sides, zero entries."""
    counts = set()
    steps = [(1, 1), (-1, 1), (1, -1), (-1, -1)]
    nrows, ncols = (1, 8, 9, 512, 513, 600) if big else (1, 8, 9), (1, 31, 32, 33, 255)
    # (N0, N3, nm list): N0 * nm * N3 per entry
    geometries = [(1, 1, (1, 2, 3)), (1, 13, (1, 2, 3)), (3, 1, (3, 1)), (1, 6, (3, 1, 2)), (3, 13, (2,)), (1, 7, (1,)), (1, 4, (2,)), (1, 17, (1,))]
    case = 0
    for N0, N3, nms in geometries:
        spec = []
        for j, nm in enumerate(nms):
            k = case + j
            spec.append(dict(nrow=nrows[k % len(nrows)], ncol=ncols[(2 * k + 1) % len(ncols)], nm=nm,
                             in_step=steps[k % 4][0], out_step=steps[k % 4][1]))
            counts.add(N0 * nm * N3)
        spec.insert(1, dict(nrow=5, ncol=4, nm=2, in_step=1, out_step=-1, zero=1))       # a zero entry between live ones
        check_ragged(B, spec, N0, N3, seed=case)
        case += len(nms)
    assert {1, 7, 8, 9, 17, 78} <= counts, counts
    # every nrow with every step pair, and every ncol, in one launch per step pair
    for si, (a, b) in enumerate(steps):
        spec = [dict(nrow=nr, ncol=ncols[(i + si) % len(ncols)], nm=1 + (i % 2), in_step=a, out_step=b) for i, nr in enumerate(nrows)]
        if big:
            assert max(s["nrow"] for s in spec) > RG_ROW_CAP, "no entry past the grid's row cap"
        check_ragged(B, spec, 1, 3, seed=100 + si)


# ------------------------------------------------------------------------------------------------------------------------------
# db_pair_lincomb
# ------------------------------------------------------------------------------------------------------------------------------
def pair_lincomb(B, x, n_out, prog, syms, sym_div):
    """prog: per output a list of (re, im, sym_off or -1, src).  x (n_in, 2 * npair, ncol).  Returns the NaN-initialised output."""
    n_in, two_np, ncol = x.shape
    npair = two_np // 2
    term_ptr = np.zeros(n_out + 1, dtype=np.int32)
    flat = [t for o in prog for t in o]
    term_ptr[1:] = np.cumsum([len(o) for o in prog])
    terms = (dlib.PairLinTerm * max(len(flat), 1))()
    for T, (re, im, so, src) in zip(terms, flat):
        T.re, T.im, T.sym_off, T.src = re, im, so, src
    xd, od, tp, td, sd = B.dev(x), B.dev(_nan((n_out, two_np, ncol))), B.dev(term_ptr), B.dev(_struct_bytes(terms)), B.dev(syms)
    B.lib.call("db_pair_lincomb", B.ptr(xd), B.ptr(od), npair, ncol, n_out, B.ptr(tp), B.ptr(td), B.ptr(sd), sym_div, B.stream)
    return B.host(od).copy()


def pair_reference(x, prog, syms, sym_div):
    """The header's formula in complex long double; returns (ref, magnitude) as (n_out, npair, ncol) complex / real arrays."""
    n_in, two_np, ncol = x.shape
    npair = two_np // 2
    CLD = np.clongdouble
    z = x[:, 0::2].astype(LD) + 1j * x[:, 1::2].astype(LD)
    e = np.arange(npair * ncol).reshape(npair, ncol)
    ref, mag = np.zeros((len(prog), npair, ncol), dtype=CLD), np.zeros((len(prog), npair, ncol), dtype=LD)
    for o, terms in enumerate(prog):
        for re, im, so, src in terms:
            sym = syms[so + e // sym_div].astype(LD) if so >= 0 else LD(1)
            c = (LD(re) + 1j * LD(im)) * sym
            ref[o] += c * z[src]
            mag[o] += (np.abs(LD(re) * sym) + np.abs(LD(im) * sym)) * (np.abs(z[src].real) + np.abs(z[src].imag))
    return ref, mag


def check_pair_program(B, x, prog, syms, sym_div, what):
    got = pair_lincomb(B, x, len(prog), prog, syms, sym_div)
    ref, mag = pair_reference(x, prog, syms, sym_div)
    gz = got[:, 0::2].astype(LD) + 1j * got[:, 1::2].astype(LD)
    assert not np.isnan(got).any(), (what, "unwritten output")
    nterm = max(max(len(o) for o in prog), 1)
    tol = (2 * nterm + 3) * EPS * mag
    assert np.all(np.abs((gz - ref).real) <= tol) and np.all(np.abs((gz - ref).imag) <= tol), what
    for o, terms in enumerate(prog):
        if not terms:
            assert not got[o].any(), (what, "an output without terms must be written as zero")
    return got


def check_pair_lincomb_shapes(B):
    """sym_div 1 and 6 (ncol = 6 k), terms with and without symbols in one output, an output without terms, more and fewer outputs
    than inputs, a repeated source, npair * ncol of 1, 255, 257 and one total past the persistent grid's 8 * SMs * 256 elements."""
    cap = 8 * B.sms * 256
    shapes = [(1, 1, 1), (5, 51, 1), (1, 257, 1), (4, 12, 6), (7, 18, 6), (cap // 12 + 3, 12, 6)]
    totals = [a * b for a, b, _ in shapes]
    assert totals[:3] == [1, 255, 257] and totals[-1] > cap and all(nc % 6 == 0 for _, nc, d in shapes if d == 6)
    for npair, ncol, sym_div in shapes:
        rng = np.random.default_rng(npair + ncol)
        nsym = (npair * ncol + sym_div - 1) // sym_div
        syms = rng.standard_normal(2 * nsym + 5)
        for n_in, n_out in ((2, 4), (3, 2)):
            x = rng.standard_normal((n_in, 2 * npair, ncol))
            prog = [[(0.5, -2.0, 5, 0), (1.25, 0.0, -1, n_in - 1), (0.0, 3.0, nsym + 5, 0)],      # symbols, a constant, a repeated source
                    []]                                                                            # no terms: zero
            if n_out == 4:
                prog += [[(-1.0, 0.0, -1, 1)], [(0.0, 1.0, 5, 1), (0.0, -1.0, 5, 1), (2.0, 2.0, -1, 0)]]
            assert len(prog) == n_out
            check_pair_program(B, x, prog, syms, sym_div, dict(npair=npair, ncol=ncol, sym_div=sym_div, n_in=n_in))


def check_intertwiner_round_trip(B, Lmax=9, Nr=6):
    """The regularity recombination Q(l) of a rank-1 shell field and its transpose as pair programs with one symbol per (pair, l)
    constant along the radial index (sym_div = Nr): each against its definition, and Q(l)^T Q(l) = 1 for l >= 1 returns the input to
    a few eps."""
    from dedalus_b200.shell import Intertwiner
    npair, nl = 3, Lmax + 1
    ncol = nl * Nr
    Q = np.stack([Intertwiner(ell).matrix(1) for ell in range(nl)])             # (l, 3, 3)
    nsym = npair * nl
    # symbol table (a, b): Q[l, a, b] at sym_off(a, b) + pair * nl + l
    syms = np.concatenate([np.tile(Q[:, a, b], npair) for a in range(3) for b in range(3)])
    off = lambda a, b: (3 * a + b) * nsym
    fwd = [[(1.0, 0.0, off(a, b), b) for b in range(3)] for a in range(3)]
    bwd = [[(1.0, 0.0, off(b, a), b) for b in range(3)] for a in range(3)]
    rng = np.random.default_rng(31)
    x = rng.standard_normal((3, 2 * npair, ncol))
    y = check_pair_program(B, x, fwd, syms, Nr, "Q(l)")
    # the definition, in float64 numpy: y[a, row, l, r] = sum_b Q[l, a, b] x[b, row, l, r]
    x4 = x.reshape(3, 2 * npair, nl, Nr)
    assert np.allclose(y.reshape(x4.shape), np.einsum('lab,bjlr->ajlr', Q, x4), rtol=0, atol=8 * EPS * np.abs(x).max())
    z = check_pair_program(B, y, bwd, syms, Nr, "Q(l)^T").reshape(x4.shape)
    assert np.abs(z[:, :, 1:] - x4[:, :, 1:]).max() <= 16 * EPS * np.abs(x).max()


# ------------------------------------------------------------------------------------------------------------------------------
# db_index_move, db_index_move_runs
# ------------------------------------------------------------------------------------------------------------------------------
def check_index_move(B, count, run=None, seed=0):
    """Gather through an index table with negative entries (they gather zeros), then scatter into a NaN arena (they scatter nothing):
    the original on the indexed slots, NaN elsewhere; both exact.  run = None: db_index_move; else runs of `run` doubles."""
    rng = np.random.default_rng(seed)
    r = 1 if run is None else run
    nslots = 2 * count + 3
    slots = rng.permutation(nslots)[:count].astype(np.int64)
    idx = slots * r
    neg = rng.random(count) < 0.25
    neg[0], neg[-1] = count > 2, False
    idx[neg] = -1 - rng.integers(0, 5, size=int(neg.sum()))
    assert count < 3 or (neg.any() and not neg.all())
    arena = rng.standard_normal(nslots * r)
    idxd, ad, vd = B.dev(idx), B.dev(arena), B.dev(_nan(count * r))
    args = (count,) if run is None else (count, run)
    name = "db_index_move" if run is None else "db_index_move_runs"
    B.lib.call(name, B.ptr(idxd), *args, B.ptr(ad), B.ptr(vd), 1, B.stream)
    vec = B.host(vd).copy()
    expect = np.where(neg[:, None], 0.0, arena.reshape(nslots, r)[np.where(neg, 0, slots)])
    assert np.array_equal(vec.reshape(count, r), expect), (name, count, run, "gather")
    assert np.array_equal(B.host(ad), arena), "the gather wrote to the arena"
    a2 = B.dev(_nan(nslots * r))
    B.lib.call(name, B.ptr(idxd), *args, B.ptr(a2), B.ptr(vd), 0, B.stream)
    back = B.host(a2).reshape(nslots, r)
    hit = np.zeros(nslots, dtype=bool); hit[slots[~neg]] = True
    assert np.array_equal(back[hit], arena.reshape(nslots, r)[hit]), (name, count, run, "scatter")
    assert np.isnan(back[~hit]).all(), (name, count, run, "scatter wrote a slot that no index names")


def check_index_moves(B):
    cap = 8 * B.sms * 256
    for count in (1, 255, 257, cap + 77):
        check_index_move(B, count, seed=count)
    assert cap + 77 > cap
    for run in (1, 255, 256, 257, 64 * 256 + 3):
        assert run != 64 * 256 + 3 or run > 64 * 256
        check_index_move(B, 9, run=run, seed=run)


# ------------------------------------------------------------------------------------------------------------------------------
# db_absmax, db_cfl_max, db_cfl_max_spherical
# ------------------------------------------------------------------------------------------------------------------------------
def _reduce(B, name, out0, *args):
    out = B.dev(np.array([out0]))
    B.lib.call(name, *args, B.ptr(out), B.stream)
    return float(B.host(out)[0])


def cfl_frequency(u, inv_dx):
    """sum_c |u_c| * inv_dx_c[index along that component's axis], term by term in component order, in float64: u_c (g0, g1, g2), the
    components are the LAST ncomp axes."""
    ncomp = len(u)
    f = np.zeros(u[0].shape)
    for c in range(ncomp):
        axis = 3 - ncomp + c
        shape = [1, 1, 1]; shape[axis] = -1
        f = f + np.abs(u[c]) * inv_dx[c].reshape(shape)
    return f


def cfl_max(B, u, inv_dx, out0=0.0):
    ncomp = len(u)
    g0, g1, g2 = u[0].shape
    ud, dd = [B.dev(a) for a in u], [B.dev(a) for a in inv_dx]
    up, dp = (C.c_void_p * 3)(*[B.ptr(a).value for a in ud]), (C.c_void_p * 3)(*[B.ptr(a).value for a in dd])
    return _reduce(B, "db_cfl_max", out0, up, dp, ncomp, g0, g1, g2)


def check_cfl_axis_mapping(B):
    """ncomp = 3, 2, 1 on grids with three different extents: component c pairs with axis 3 - ncomp + c, and each axis' inverse
    spacings carry their own marker values, so that a wrong axis changes the maximum."""
    for shape, ncomp in (((5, 7, 11), 3), ((1, 7, 11), 2), ((1, 1, 11), 1), ((5, 7, 11), 2), ((5, 7, 11), 1)):
        rng = np.random.default_rng(ncomp + shape[0])
        assert len(set(shape[3 - ncomp:])) == ncomp
        u = [rng.standard_normal(shape) for _ in range(ncomp)]
        inv_dx = [10.0 ** (c + 1) * (1.0 + rng.random(shape[3 - ncomp + c])) for c in range(ncomp)]
        f = cfl_frequency(u, inv_dx)
        got = cfl_max(B, u, inv_dx)
        assert got == f.max(), (shape, ncomp, got, f.max())


def check_reduction_positions(B):
    """The maximum at the first element, at the last element and in the last partial block, for totals of 1, 255, 257 and one past the
    grid cap; `out` pre-set to a larger value stays (the accumulate contract that the multi-field CFL relies on); u_r = NULL."""
    cap = 8 * B.sms * 256
    for total in (1, 255, 257, cap + 300):
        assert total != cap + 300 or (total > cap and total % 256 != 0)
        for where in {0, total - 1, max(total - total % 256, 0) if total % 256 else total - 1}:
            rng = np.random.default_rng(total + where)
            v = rng.standard_normal(total)
            v[where] = -50.0
            vd = B.dev(v)
            assert _reduce(B, "db_absmax", 0.0, B.ptr(vd), total) == 50.0, ("absmax", total, where)
            assert _reduce(B, "db_absmax", 77.0, B.ptr(vd), total) == 77.0, ("absmax keeps a larger value", total)
            # Cartesian CFL on (1, 1, total) with one component
            inv = 1.0 + rng.random(total)
            got = cfl_max(B, [v.reshape(1, 1, total)], [inv])
            assert got == (np.abs(v) * inv).max() == 50.0 * inv[where], ("cfl", total, where)
            assert cfl_max(B, [v.reshape(1, 1, total)], [inv], out0=1e6) == 1e6
            # spherical CFL: (n_ang, n_r) with n_r = 1 or 3
            for n_r in (1, 3):
                if total % n_r:
                    continue
                n_ang = total // n_r
                up, ut, ur = v.copy(), rng.standard_normal(total), rng.standard_normal(total)
                ut[where] = 40.0
                inv_h, inv_dr = 1.0 + rng.random(n_r), 2.0 + rng.random(n_r)
                ir = np.arange(total) % n_r
                d = [B.dev(a) for a in (up, ut, ur, inv_h, inv_dr)]
                f2 = np.sqrt(up * up + ut * ut) * inv_h[ir]
                f3 = f2 + np.abs(ur) * inv_dr[ir]
                got3 = _reduce(B, "db_cfl_max_spherical", 0.0, *[B.ptr(a) for a in d], n_ang, n_r)
                got2 = _reduce(B, "db_cfl_max_spherical", 0.0, B.ptr(d[0]), B.ptr(d[1]), None, B.ptr(d[3]), None, n_ang, n_r)
                # the kernel may contract up * up + ut * ut into a fused multiply-add: 2 eps on the long-double maximum
                f2l = np.sqrt(up.astype(LD) ** 2 + ut.astype(LD) ** 2) * inv_h[ir]
                f3l = f2l + np.abs(ur) * inv_dr[ir].astype(LD)
                assert abs(got2 - f2l.max()) <= 2 * EPS * f2l.max(), ("spherical, u_r = NULL", total, where)
                assert abs(got3 - f3l.max()) <= 2 * EPS * f3l.max(), ("spherical", total, where)
                assert np.argmax(f2) == where
                assert _reduce(B, "db_cfl_max_spherical", 1e9, *[B.ptr(a) for a in d], n_ang, n_r) == 1e9


def check_reductions_propagate_nan(B):
    """A NaN anywhere in the input gives a NaN maximum, as np.max does: a velocity field that has blown up must not yield a finite
    CFL frequency.  An infinite value gives +inf.  A NaN already in `out` stays."""
    cap = 8 * B.sms * 256
    for total in (1, 257, cap + 300):
        for where in sorted({0, total // 2, total - 1}):
            rng = np.random.default_rng(total)
            v = rng.standard_normal(total)
            inv = 1.0 + rng.random(total)
            for bad, check in ((np.nan, np.isnan), (-np.inf, lambda r: r == np.inf)):
                w = v.copy(); w[where] = bad
                wd = B.dev(w)
                assert check(_reduce(B, "db_absmax", 0.0, B.ptr(wd), total)), ("absmax", total, where, bad)
                assert check(cfl_max(B, [w.reshape(1, 1, total)], [inv])), ("cfl", total, where, bad)
                d = [B.dev(a) for a in (v, w, w, inv[:1], inv[:1])]
                assert check(_reduce(B, "db_cfl_max_spherical", 0.0, *[B.ptr(a) for a in d], total, 1)), ("spherical", total, where, bad)
                assert check(_reduce(B, "db_cfl_max_spherical", 0.0, B.ptr(d[0]), B.ptr(d[1]), None, B.ptr(d[3]), None, total, 1))
    vd = B.dev(np.ones(5))
    assert np.isnan(_reduce(B, "db_absmax", np.nan, B.ptr(vd), 5))
