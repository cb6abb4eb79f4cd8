"""Initial value problems on a spherical shell (BASELINE config 5; SURVEY section 8f rank 2): per-l pencil matrices.

The reference builds one Subproblem per degree l (matrices independent of m; core/basis.py:4187-4192), every operator through
`SphericalEllOperator.subproblem_matrix` (core/operators.py:3159-3193).  Here the LHS expression tree is lowered, for one l at a
time, to blocks  (output component, variable, variable component) -> radial matrix  by restating each operator:
  gradient      xi(-+1, l + R) D-+(l + R)                      core/operators.py:3280-3310
  divergence    xi(-1, l + R + 1) D+ / xi(+1, l + R - 1) D-     core/operators.py:3577-3603
  trace         Q(l)^T (spin trace) Q(l)                        core/operators.py:1783-1827
  products with radial non-constant coefficients (er, rvec)     core/basis.py:284-330 (Gamma through the intertwiners,
                arithmetic.py:560-580) with the radial multiplication matrices of core/basis.py:3879-3915
  lift          e_n (x) Q(l)^T                                   core/basis.py:5155-5199
  interpolation Q(l) (x) row of (dR / r)^k P_n(z(r))             core/basis.py:5823-5889, 3798-3803
  integration   l = 0 row of radial quadrature weights          core/basis.py:5555-5575
  conversions   E^dk, constants -> l = 0 mode                    core/basis.py:4822-4842, 4782-4819
with the radial operators D+-, E of libraries/dedalus_sphere/shell.py:21-73 composed from the Jacobi operators of
dedalus_b200/jacobi.py.  R = regularity total of the component, Q(l) = dedalus_b200/shell.py Intertwiner.
"""
import numpy as np
from scipy import sparse
from . import jacobi
from . import operators as ops
from .field import Field
from .shell import ShellBasis, ShellRadialBasis, Intertwiner, shell_basis_of
from .sphere import SphereBasis

REG = (-1, +1, 0)


def xi(mu, l):
    """reference basis.py:3545-3546."""
    return np.sqrt((l + (mu + 1) // 2) / (2 * l + 1))


def regtotal(regindex):
    return sum(REG[i] for i in regindex)


def regularity_allowed(ell, regindex):
    if not regindex:
        return True
    return not Intertwiner(ell).forbidden_regularity(tuple(REG[i] for i in regindex))


class RadialOps:
    """Radial operators of a shell on N modes: D(p, l) and E map basis k -> k + 1 (libraries/dedalus_sphere/shell.py)."""

    def __init__(self, N, radii, alpha=(-0.5, -0.5)):
        self.N, self.radii, self.alpha = N, radii, alpha
        self.dR = radii[1] - radii[0]
        self.rho = (radii[1] + radii[0]) / self.dR
        self._cache = {}

    PAD = 8          # operators are composed on N + PAD modes and truncated ONCE (the reference composes infinite operators)

    def _parts(self, k):
        if k not in self._cache:
            a, b = k + self.alpha[0], k + self.alpha[1]
            P = self.N + self.PAD
            Z = (self.rho * sparse.identity(P) + jacobi.jacobi_matrix(P, a, b)).tocsr()
            AB = jacobi.conversion_matrix(P, a, b, a + 1, b + 1).tocsr()
            Dz = jacobi.differentiation_matrix(P, a, b).tocsr()
            cut = lambda M: sparse.csr_matrix(M.tocsr()[:self.N, :self.N])
            self._cache[k] = dict(DZ=cut(Dz @ Z), AB=cut(AB), E_pad=(0.5 * (AB @ Z)).tocsr(), Z=cut(Z))
        return self._cache[k]

    def D(self, p, l, k):
        """D = (d/dz Z - K AB) / dR with K = (k + 1) + p l + (p == -1) (2 - 3): the reference's K = A(0) - alpha_0 + ... is
        evaluated AFTER AB raised the Jacobi parameter, hence k + 1 (libraries/dedalus_sphere/shell.py:55-67)."""
        q = self._parts(k)
        K = k + 1 + p * l + (-1 if p == -1 else 0)
        return (q['DZ'] - K * q['AB']) / self.dR

    def E(self, k, dk=1):
        """(E^dk)[:N, :N]: E has one sub-diagonal, so the product is formed on padded matrices (dk <= PAD / 2)."""
        P = self.N + self.PAD
        M = sparse.identity(P, format='csr')
        for j in range(dk):
            M = self._parts(k + j)['E_pad'] @ M
        return sparse.csr_matrix(M.tocsr()[:self.N, :self.N])

    def basis_functions(self, k, r):
        """(dR / r)^k P_n^(alpha + k)(z(r)), n < N, at radii r: array (len(r), N)."""
        r = np.atleast_1d(np.asarray(r, dtype=float))
        z = 2 * r / self.dR - self.rho
        return ((self.dR / r) ** k)[:, None] * jacobi.polynomials(self.N, k + self.alpha[0], k + self.alpha[1], z).T

    def multiplication(self, f, k_in, k_out):
        """Matrix of g -> f(r) g from basis k_in to basis k_out by Gauss-Jacobi quadrature (exact for polynomial f times the
        (dR / r)^(k_out - k_in) mismatch being polynomial, which holds for the radial coefficients r and 1 met here)."""
        a, b = k_out + self.alpha[0], k_out + self.alpha[1]
        nq = 2 * self.N + 8
        z, w = jacobi.gauss_grid(nq, a, b)
        r = self.dR / 2 * (z + self.rho)
        Bin = self.basis_functions(k_in, r)                                   # (nq, N)
        Pout = jacobi.polynomials(self.N, a, b, z)                             # (N, nq)
        return (Pout * w[None, :]) @ (((r / self.dR) ** k_out * f(r))[:, None] * Bin)


class Node:
    """Lowered subexpression for one l: blocks[tder][(out comp, var index, var comp)] = radial matrix."""
    __slots__ = ("blocks", "kind", "k", "rank", "nrad")

    def __init__(self, blocks, kind, k, rank, nrad):
        self.blocks, self.kind, self.k, self.rank, self.nrad = blocks, kind, k, rank, nrad


def _map(node, fn, **kw):
    """Apply fn(out comp, matrix) -> list of (new out comp, new matrix) to every block."""
    out = {}
    for t, d in node.blocks.items():
        o = out.setdefault(t, {})
        for (co, iv, ci), B in d.items():
            for co2, B2 in fn(co, B):
                key = (co2, iv, ci)
                o[key] = o[key] + B2 if key in o else B2
    return Node(out, kw.get('kind', node.kind), kw.get('k', node.k), kw.get('rank', node.rank), kw.get('nrad', node.nrad))


class ShellLowering:
    def __init__(self, problem):
        self.problem = problem
        self.variables = problem.variables
        basis = None
        for v in self.variables:
            basis = basis or shell_basis_of(v)
        self.basis = basis
        self.Nr = basis.shape[2]
        self.rops = RadialOps(self.Nr, basis.radii, basis.alpha)
        self._Q = {}

    def Q(self, ell, rank):
        key = (ell, rank)
        if key not in self._Q:
            self._Q[key] = Intertwiner(ell).matrix(rank) if rank else np.ones((1, 1))
        return self._Q[key]

    def kind_of(self, e):
        b = e.bases
        if isinstance(b[-1], ShellBasis):
            return 'shell', b[-1].k
        if isinstance(b[0], (SphereBasis, ShellBasis)):
            return 'sphere', 0
        if isinstance(b[-1], ShellRadialBasis):
            return 'radial', b[-1].k
        return 'const', 0

    # ---- radial NCC: regularity components (at l = 0) of a field on the radial basis, as functions of r
    def ncc_functions(self, ncc):
        """[f_a(r)] over the regularity components a of a radial-basis field given by its coordinate components on the grid."""
        g = np.asarray(ncc['g']).reshape(max(ncc.ncomp, 1), -1)                       # (ncomp, Nr_g) coordinate components
        rank = len(ncc.tensorsig)
        rgrid = ncc.bases[-1].global_grid(ncc.scales[-1])
        if rank:
            cs = ncc.tensorsig[0]
            spin = cs.U_forward(rank) @ g
            if np.abs(spin.imag).max() > 1e-14 * max(np.abs(spin).max(), 1e-300):
                raise NotImplementedError("radial coefficients with angular components")
            reg = self.Q(0, rank).T @ spin.real
        else:
            reg = g
        # interpolating polynomials through the Chebyshev-grid values (the coefficients are low-degree polynomials in r)
        funcs = []
        for a in range(reg.shape[0]):
            coef = np.polynomial.chebyshev.chebfit(2 * rgrid / self.rops.dR - self.rops.rho, reg[a], len(rgrid) - 1)
            coef[np.abs(coef) < 1e-13 * max(np.abs(coef).max(), 1e-300)] = 0
            funcs.append((lambda c: (lambda r: np.polynomial.chebyshev.chebval(2 * r / self.rops.dR - self.rops.rho, c)))(coef)
                         if np.any(coef) else None)
        return funcs

    def gamma(self, ell, rank_a, ell_a, rank_b, ell_b, a_first=True):
        """Tensor-product coupling in regularity components: G[a, b, c] = sum Q_A[a', a] Q_B[b', b] Q_C[(a' b'), c]
        (reference arithmetic.py:560-580 with GammaCoord of the tensor product, 772-783)."""
        QA, QB, QC = self.Q(ell_a, rank_a), self.Q(ell_b, rank_b), self.Q(ell, rank_a + rank_b)
        na, nb = QA.shape[0], QB.shape[0]
        QC3 = QC.reshape(na, nb, -1)                                              # [a', b', c]
        return np.einsum('xa,yb,xyc->abc', QA, QB, QC3)

    # ---- recursive lowering
    def lower(self, e, ell):
        Nr, rops = self.Nr, self.rops
        for iv, v in enumerate(self.variables):
            if e is v:
                kind, k = self.kind_of(v)
                n = Nr if kind == 'shell' else 1
                I = sparse.identity(n, format='csr')
                return Node({0: {(c, iv, c): I for c in range(max(v.ncomp, 1))}}, kind, k, len(v.tensorsig), n)
        if isinstance(e, ops.Add):
            nodes = [self.lower(a, ell) for a in e.args]
            kind = 'shell' if any(n.kind == 'shell' for n in nodes) else nodes[0].kind
            k = max(n.k for n in nodes)
            out = {}
            for n in nodes:
                n = self.convert(n, kind, k, ell)
                for t, d in n.blocks.items():
                    o = out.setdefault(t, {})
                    for key, B in d.items():
                        o[key] = o[key] + B if key in o else B
            return Node(out, kind, k, nodes[0].rank, Nr if kind == 'shell' else 1)
        if isinstance(e, ops.ScalarMul):
            return _map(self.lower(e.args[0], ell), lambda co, B: [(co, B * e.c)])
        if isinstance(e, ops.TimeDerivative):
            n = self.lower(e.args[0], ell)
            return Node({t + 1: d for t, d in n.blocks.items()}, n.kind, n.k, n.rank, n.nrad)
        if isinstance(e, ops.Gradient):
            n = self.lower(e.args[0], ell)
            if n.kind != 'shell':
                raise NotImplementedError("gradient of a non-shell operand")
            ncomp = 3 ** n.rank
            def fn(co, B):
                rin = np.unravel_index(co, (3,) * n.rank) if n.rank else ()
                R = regtotal(rin)
                out = []
                for a, mu in ((0, -1), (1, +1)):
                    rout = (a,) + tuple(rin)
                    if regularity_allowed(ell, rin) and regularity_allowed(ell, rout):
                        out.append((a * ncomp + co, xi(mu, ell + R) * (rops.D(mu, ell + R, n.k) @ B)))
                return out
            return _map(n, fn, k=n.k + 1, rank=n.rank + 1)
        if isinstance(e, ops.Laplacian):
            # div(grad(.)) (reference SphericalLaplacian, core/operators.py:3958-4010: the same composition of D+ / D- blocks)
            return self.lower(ops.Divergence(ops.Gradient(e.args[0], e.args[0].dist.coordsys)), ell)
        if isinstance(e, ops.Divergence):
            n = self.lower(e.args[0], ell)
            nrest = 3 ** (n.rank - 1)
            def fn(co, B):
                rin = tuple(np.unravel_index(co, (3,) * n.rank))
                R = regtotal(rin)
                a, rest = rin[0], rin[1:]
                if a == 2 or not (regularity_allowed(ell, rin) and regularity_allowed(ell, rest)):
                    return []
                if a == 0:
                    M = xi(-1, ell + R + 1) * rops.D(+1, ell + R, n.k)
                else:
                    M = xi(+1, ell + R - 1) * rops.D(-1, ell + R, n.k)
                return [(co % nrest, M @ B)]
            return _map(n, fn, k=n.k + 1, rank=n.rank - 1)
        if isinstance(e, ops.TransposeComponents):
            # swap of the first two tensor indices: a permutation of the spin components, conjugated with the intertwiners
            # (reference SphericalTransposeComponents, core/operators.py:1950-2010)
            n = self.lower(e.args[0], ell)
            nrest = 3 ** (n.rank - 2)
            idx = np.arange(9 * nrest).reshape(3, 3, nrest).transpose(1, 0, 2).ravel()
            P = np.zeros((9 * nrest, 9 * nrest)); P[np.arange(idx.size), idx] = 1
            Q = self.Q(ell, n.rank)
            T = Q.T @ P @ Q
            def fn(co, B):
                return [(c, T[c, co] * B) for c in range(9 * nrest) if abs(T[c, co]) > 1e-14]
            return _map(n, fn)
        if isinstance(e, ops.Trace):
            n = self.lower(e.args[0], ell)
            nrest = 3 ** (n.rank - 2)
            tr = np.zeros(9); tr[[1, 3, 8]] = 1                                  # spin trace: (-+), (+-), (00)
            T = self.Q(ell, n.rank - 2).T @ np.kron(tr[None, :], np.eye(nrest)) @ self.Q(ell, n.rank)
            def fn(co, B):
                return [(c, T[c, co] * B) for c in range(nrest) if T[c, co] != 0]
            return _map(n, fn, rank=n.rank - 2)
        if isinstance(e, ops.Multiply):
            A, Bx = e.args
            a_ncc = not A.has(*self.variables)
            ncc, arg = (A, Bx) if a_ncc else (Bx, A)
            if ncc.has(*self.variables):
                raise ValueError("LHS must be linear in the problem variables.")
            if not isinstance(ncc, Field):
                raise NotImplementedError("only plain fields as LHS coefficients")
            n = self.lower(arg, ell)
            kind_n, k_ncc = self.kind_of(ncc)
            if kind_n == 'const':
                vals = np.asarray(ncc['c']).reshape(-1)
                if len(vals) != 1:
                    raise NotImplementedError("constant tensor coefficients on a shell")
                return _map(n, lambda co, B: [(co, B * vals[0])])
            if kind_n != 'radial' or n.kind != 'shell':
                raise NotImplementedError("LHS coefficients must be constants or fields on the shell's radial basis")
            funcs = self.ncc_functions(ncc)
            ra, rb = len(ncc.tensorsig), n.rank
            if a_ncc:
                G = self.gamma(ell, ra, 0, rb, ell)                             # [ncc comp, arg comp, out comp]
            else:
                G = self.gamma(ell, rb, ell, ra, 0).transpose(1, 0, 2)
            k_out = n.k + k_ncc
            mats = [None if f is None else sparse.csr_matrix(_clean(rops.multiplication(f, n.k, k_out))) for f in funcs]
            def fn(co, B):
                out = []
                for c in range(G.shape[2]):
                    M = None
                    for a, Ma in enumerate(mats):
                        if Ma is not None and abs(G[a, co, c]) > 1e-14:
                            M = G[a, co, c] * Ma if M is None else M + G[a, co, c] * Ma
                    if M is not None:
                        out.append((c, M @ B))
                return out
            return _map(n, fn, k=k_out, rank=ra + rb)
        if isinstance(e, ops.Lift):
            n = self.lower(e.args[0], ell)
            if n.kind != 'sphere' or not isinstance(e.basis, ShellBasis):
                raise NotImplementedError("Lift of a sphere field along a shell basis only")
            pos = e.n if e.n >= 0 else e.n + Nr
            col = sparse.csr_matrix(([1.0], ([pos], [0])), shape=(Nr, 1))
            Q = self.Q(ell, n.rank)
            def fn(co, B):
                return [(c, Q[co, c] * (col @ B)) for c in range(Q.shape[1]) if Q[co, c] != 0]
            return _map(n, fn, kind='shell', k=e.basis.k, nrad=Nr)
        if isinstance(e, ops.Interpolate):
            n = self.lower(e.args[0], ell)
            if n.kind != 'shell' or e.axis != e.dist.dim - 1:
                raise NotImplementedError("interpolation along the radius of a shell only")
            row = sparse.csr_matrix(rops.basis_functions(n.k, [float(e.position)]))   # (1, Nr)
            Q = self.Q(ell, n.rank)
            def fn(co, B):
                rin = tuple(np.unravel_index(co, (3,) * n.rank)) if n.rank else ()
                if not regularity_allowed(ell, rin):
                    return []
                return [(s, Q[s, co] * (row @ B)) for s in range(Q.shape[0]) if Q[s, co] != 0]
            return _map(n, fn, kind='sphere', k=0, nrad=1)
        if isinstance(e, ops.Component):
            # a selection of spin components (reference S2RadialComponent / S2AngularComponent.subproblem_matrix,
            # core/basis.py:5892-5970): the blocks move to the component they land on, unchanged
            n = self.lower(e.args[0], ell)
            if n.kind != 'sphere':
                raise NotImplementedError("radial / angular components on a shell: of fields on a sphere (interpolate first)")
            sel = component_selection(e)
            return _map(n, lambda co, B: [(sel[co], B)] if co in sel else [], rank=len(e.tensorsig))
        if isinstance(e, ops.Integrate):
            n = self.lower(e.args[0], ell)
            if n.kind != 'shell' or n.rank != 0 or e.average:
                raise NotImplementedError("integration of shell scalars only")
            if ell != 0:
                return Node({}, 'const', 0, 0, 1)
            z, w = np.polynomial.legendre.leggauss(2 * Nr)
            r = rops.dR / 2 * (z + rops.rho)
            Qk = jacobi.polynomials(Nr, n.k + rops.alpha[0], n.k + rops.alpha[1], z)
            row = ((r**2 * w * (r / rops.dR) ** (-n.k))[None, :] @ Qk.T) * (rops.dR / 2) * (4 * np.pi / np.sqrt(2))
            row = sparse.csr_matrix(row)
            return _map(n, lambda co, B: [(co, row @ B)], kind='const', k=0, nrad=1)
        raise NotImplementedError(f"{type(e).__name__} is not supported on the LHS of shell problems")

    def convert(self, n, kind, k, ell):
        Nr, rops = self.Nr, self.rops
        if n.kind == kind and n.k == k:
            return n
        if n.kind == 'shell' and kind == 'shell':
            E = rops.E(n.k, k - n.k)
            return _map(n, lambda co, B: [(co, E @ B)], k=k)
        if n.kind == 'const' and kind == 'shell':
            if n.rank:
                raise NotImplementedError("constant tensors on a shell")
            if ell != 0:
                return Node({}, 'shell', k, 0, Nr)
            cmv = (1 / np.sqrt(jacobi.mass(rops.alpha[0], rops.alpha[1]))) / np.sqrt(2)      # reference basis.py:4203-4207
            col = sparse.csr_matrix(([1 / cmv], ([0], [0])), shape=(Nr, 1))
            E = rops.E(0, k)
            return _map(n, lambda co, B: [(co, E @ col @ B)], kind='shell', k=k, nrad=Nr)
        raise NotImplementedError(f"conversion {n.kind} -> {kind}")


def _clean(M, tol=1e-13):
    M = np.array(M)
    M[np.abs(M) < tol * max(np.abs(M).max(), 1e-300)] = 0
    return M


def component_selection(e):
    """{operand component: result component} of a radial / angular component (C order over the tensor dims): the radial one keeps
    the components whose selected index is the spin-0 one (index 2) and drops that index; the angular one keeps those with spin
    -, + (indices 0, 1) at the same positions, the index now running over the 2 components of the S2 coordinates."""
    dims_in = tuple(cs.dim for cs in e.args[0].tensorsig)
    dims_out = tuple(cs.dim for cs in e.tensorsig)
    radial = isinstance(e, ops.RadialComponent)
    sel = {}
    for c, idx in enumerate(np.ndindex(*dims_in)):
        a = idx[e.index]
        if radial and a == 2:
            out = idx[:e.index] + idx[e.index + 1:]
        elif not radial and a < 2:
            out = idx
        else:
            continue
        sel[c] = int(np.ravel_multi_index(out, dims_out)) if dims_out else 0
    return sel


def component_layout(items, basis, ell):
    """Natural ordering of the unknowns (or equation rows) of degree l: for each item (kind, tensor signature), its components, each
    with its radial size, and their validity (reference: regularity_allowed / |total spin| <= l / l == 0).  Fields on a sphere
    may carry S2 indices (2 spin components -, +) next to spherical ones (3: -, +, 0)."""
    Nr = basis.shape[2]
    out = []
    for it, (kind, tensorsig) in enumerate(items):
        for c, idx in enumerate(np.ndindex(*(cs.dim for cs in tensorsig))):
            if kind == 'shell':
                if any(cs.dim != 3 for cs in tensorsig):
                    raise NotImplementedError("S2 tensor indices of shell fields")
                valid, n = regularity_allowed(ell, idx), Nr
            elif kind == 'sphere':
                valid, n = abs(sum(cs.spin_ordering[i] for cs, i in zip(tensorsig, idx))) <= ell, 1
            else:
                valid, n = (ell == 0), 1
            out.append(dict(item=it, comp=c, n=n, valid=valid))
    return out


def assemble(low, ell):
    """(M, L, row layout, column layout) of degree l in natural ordering: dense arrays over ALL components (invalid ones
    included, as zero rows / columns)."""
    problem = low.problem
    var_items = [(low.kind_of(v)[0], v.tensorsig) for v in low.variables]
    cols = component_layout(var_items, low.basis, ell)
    col_off = np.cumsum([0] + [c['n'] for c in cols])
    col_index = {(c['item'], c['comp']): i for i, c in enumerate(cols)}
    eq_nodes = [low.lower(eq['LHS'], ell) for eq in problem.equations]
    eq_items = [(low.kind_of(eq['LHS'])[0], eq['tensorsig']) for eq in problem.equations]
    rows = component_layout(eq_items, low.basis, ell)
    row_off = np.cumsum([0] + [r['n'] for r in rows])
    row_index = {(r['item'], r['comp']): i for i, r in enumerate(rows)}
    mats = {0: np.zeros((row_off[-1], col_off[-1])), 1: np.zeros((row_off[-1], col_off[-1]))}
    for ie, node in enumerate(eq_nodes):
        for t, d in node.blocks.items():
            if t > 1:
                raise NotImplementedError("Only first-order time derivatives are supported.")
            for (co, iv, ci), B in d.items():
                ri, cj = row_index[(ie, co)], col_index[(iv, ci)]
                B = B.toarray() if sparse.issparse(B) else np.asarray(B)
                mats[t][row_off[ri]:row_off[ri + 1], col_off[cj]:col_off[cj + 1]] += B
    return mats[1], mats[0], rows, cols


# ------------------------------------------------------------------------------------------------------------
# Device side: per-l dense systems with one right-hand-side column per (m <= l, cos | -sin)
# ------------------------------------------------------------------------------------------------------------
class ShellSystems:
    """Per-degree pencil systems of a shell IVP on the device, behind the interface of the IMEX loops in solvers.py
    (move / matvec / solve / factor_verified), served by csrc/dense.cu.

    System l: the valid unknowns of degree l in natural order (variable, component, radial mode), padded to the common size
    n with identity rows; its right-hand-side columns are r = 2 m + part for m <= l (reference: one Subproblem per l with one
    subsystem per m, core/subsystems.py:272-274; real dtype: the cos and -sin parts see the same real matrix)."""

    VERIFY_TOL = 1e-9

    def __init__(self, solver, nslots, nlu):
        import torch
        from .lib import DenseSys
        self.solver = solver
        dev = solver.device
        problem = solver.problem
        low = self.low = ShellLowering(problem)
        basis = low.basis
        sb = basis.sphere_basis
        Lmax, Nphi = basis.Lmax, basis.shape[0]
        dist = solver.dist
        j0, j1 = sb.local_pairs(dist)
        Nc0, Nc1, Nr = 2 * (j1 - j0), basis.coeff_shape[1], basis.coeff_shape[2]
        local_ms = sorted(m for m, _ in sb.local_wavenumbers(dist))
        per_l = []
        for ell in range(Lmax + 1):
            M, L, rows, cols = assemble(low, ell)
            vr = np.array([r['valid'] for r in rows for _ in range(r['n'])], dtype=bool)
            vc = np.array([c['valid'] for c in cols for _ in range(c['n'])], dtype=bool)
            if vr.sum() != vc.sum():
                raise ValueError(f"shell problem: {int(vr.sum())} equations for {int(vc.sum())} unknowns at l = {ell}")
            per_l.append(dict(M=M[np.ix_(vr, vc)], L=L[np.ix_(vr, vc)], rows=rows, cols=cols, vr=vr, vc=vc))
        n = max(p['M'].shape[0] for p in per_l)
        self.n, self.nsys = n, Lmax + 1
        Mall, Lall = np.zeros((self.nsys, n, n)), np.zeros((self.nsys, n, n))
        for ell, p in enumerate(per_l):
            k = p['M'].shape[0]
            Mall[ell, :k, :k], Lall[ell, :k, :k] = p['M'], p['L']
            Lall[ell, np.arange(k, n), np.arange(k, n)] = 1.0                   # padding unknowns: identity
        Mall[np.abs(Mall) < solver.entry_cutoff] = 0
        Lall[np.abs(Lall) < solver.entry_cutoff] = 0
        # ---- right-hand-side columns and index tables
        arr = (DenseSys * self.nsys)()
        vec_off, xi_all, fi_all = 0, [], []
        mode = {m: sb.mode_columns(m) for m in range(Nphi // 2)}
        var_items = [(low.kind_of(v)[0], v.tensorsig) for v in low.variables]
        eq_items = [(low.kind_of(eq['LHS'])[0], eq['tensorsig']) for eq in problem.equations]
        self.total_modes = 0
        for ell, p in enumerate(per_l):
            ms_l = [m for m in local_ms if m <= ell and mode[m][0] is not None]       # this rank's columns of degree l
            ncols = 2 * len(ms_l)
            arr[ell].ncols, arr[ell].vec_off = ncols, vec_off
            for side, layout, valid, arena, items in ((0, p['cols'], p['vc'], solver.var_arena, var_items),
                                                      (1, p['rows'], p['vr'], solver.eq_arena, eq_items)):
                idx = np.full((n, ncols), -1, dtype=np.int64)
                i = 0
                ms = np.array(ms_l, dtype=np.int64)
                cpos = np.arange(len(ms_l), dtype=np.int64)                               # column pair of each local m
                js = np.array([mode[m][0] - j0 for m in ms_l], dtype=np.int64)
                slots = np.array([mode[m][1][ell - m] for m in ms_l], dtype=np.int64)
                for comp in layout:
                    if not comp['valid']:
                        continue
                    kind = items[comp['item']][0]
                    nrad = comp['n']
                    base = arena.offsets[comp['item']]
                    if kind == 'const':
                        if ncols and ms_l[0] == 0:
                            idx[i, 0] = base
                        i += 1
                        continue
                    plane = Nc0 * Nc1 * nrad
                    nr = np.arange(nrad)[:, None]
                    for part in (0, 1):
                        if ncols:
                            idx[i:i + nrad, 2 * cpos + part] = (base + comp['comp'] * plane + ((2 * js + part) * Nc1 + slots)[None, :] * nrad + nr)
                    i += nrad
                (xi_all if side == 0 else fi_all).append(idx.ravel())
            self.total_modes += int(p['vc'].sum()) * ncols
            vec_off += n * ncols
        self.nvec = max(vec_off, 1)
        self.max_ncols = max(max(a.ncols for a in arr), 1)
        t64 = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
        self.M_t, self.L_t = t64(Mall), t64(Lall)                       # dense: the LHS a0 M + b0 L is factorised in this form
        self.csr = {}
        for name, A in (('M', Mall), ('L', Lall)):                       # CSR: the operators are a few percent dense (mat-vecs)
            nz = A != 0
            counts = nz.sum(axis=2)                                       # (nsys, n)
            ptr = np.zeros((self.nsys, n + 1), dtype=np.int64)
            ptr[:, 1:] = np.cumsum(counts, axis=1)
            ptr += np.concatenate([[0], np.cumsum(counts.sum(axis=1))[:-1]])[:, None]
            s_, r_, c_ = np.nonzero(nz)
            self.csr[name] = (t64(ptr), t64(c_.astype(np.int32)), t64(A[s_, r_, c_]))
        self.desc = torch.from_numpy(np.frombuffer(bytes(arr), dtype=np.uint8).copy()).to(dev)
        self.idx = [t64(np.concatenate(xi_all)), t64(np.concatenate(fi_all))]
        self.vecs = [torch.zeros(self.nvec, dtype=torch.float64, device=dev) for _ in range(nslots)]
        self.lu = [torch.zeros((self.nsys, n, n), dtype=torch.float64, device=dev) for _ in range(nlu)]
        self.ipiv = [torch.zeros((self.nsys, n), dtype=torch.int32, device=dev) for _ in range(nlu)]
        self.info = torch.zeros(self.nsys, dtype=torch.int32, device=dev)
        self.reorders, self.last_verify = 0, None

    def _call(self, name, *args):
        self.solver.lib.call(name, *args, self.solver.stream())

    def move(self, side, gather, slot, arena_t):
        from .solvers import Timed
        with Timed(self.solver.prof, "pencil_gather" if gather else "pencil_scatter", 24 * self.nvec):
            self._call("db_index_move", self.idx[side].data_ptr(), self.nvec, arena_t.data_ptr(), self.vecs[slot].data_ptr(), 1 if gather else 0)

    def matvec(self, x_slot, ym_slot=-1, yl_slot=-1):
        from .solvers import Timed
        ym = self.vecs[ym_slot].data_ptr() if ym_slot >= 0 else None
        yl = self.vecs[yl_slot].data_ptr() if yl_slot >= 0 else None
        nout = (ym_slot >= 0) + (yl_slot >= 0)
        (mp, mc, mv), (lp, lc, lv) = self.csr['M'], self.csr['L']
        with Timed(self.solver.prof, "pencil_matvec", 12 * (mv.numel() * (ym_slot >= 0) + lv.numel() * (yl_slot >= 0)) + 8 * (1 + nout) * self.nvec):
            self._call("db_csr_matvec", self.desc.data_ptr(), self.nsys, self.n, mp.data_ptr(), mc.data_ptr(), mv.data_ptr(),
                       lp.data_ptr(), lc.data_ptr(), lv.data_ptr(), self.vecs[x_slot].data_ptr(), ym, yl)

    def solve(self, lu_slot, x_slot, terms):
        import ctypes as C
        from .lib import VecComb
        from .solvers import Timed
        vc = VecComb()
        vc.nvec = len(terms)
        for k, (slot, coef) in enumerate(terms):
            if slot == x_slot:
                raise ValueError("the solution slot must not be one of the right-hand-side slots")
            vc.vec[k] = self.vecs[slot].data_ptr(); vc.coef[k] = coef
        with Timed(self.solver.prof, "pencil_solve", 8 * (self.nsys * self.n * self.n + self.nvec * (len(terms) + 1))):
            self._call("db_dense_solve", self.desc.data_ptr(), self.nsys, self.n, self.max_ncols, self.lu[lu_slot].data_ptr(),
                       self.ipiv[lu_slot].data_ptr(), C.byref(vc), self.vecs[x_slot].data_ptr())

    def factor(self, lu_slot, a0, b0):
        self._call("db_dense_combine", self.nsys, self.n, float(a0), self.M_t.data_ptr(), float(b0), self.L_t.data_ptr(), self.lu[lu_slot].data_ptr())
        self._call("db_dense_factor", self.nsys, self.n, self.lu[lu_slot].data_ptr(), self.ipiv[lu_slot].data_ptr(), self.info.data_ptr())

    def check_info(self):
        from .lib import DedalusB200Error
        bad = int((self.info != 0).sum().item())
        if bad:
            raise DedalusB200Error(f"{bad} shell pencil systems hit a zero / non-finite pivot during factorisation.")

    def factor_verified(self, lhs, slots):
        """Factorise a0 M + b0 L into each slot and check the backward error of a probe solve."""
        import torch
        from .lib import DedalusB200Error
        s_b, s_x, s_m, s_l = slots
        worst = 0.0
        for lu_slot, a0, b0 in lhs:
            self.factor(lu_slot, a0, b0)
            self.check_info()
            gen = torch.Generator(device=self.solver.device); gen.manual_seed(1234)
            self.vecs[s_b].normal_(generator=gen)
            self.solve(lu_slot, s_x, [(s_b, 1.0)])
            self.matvec(s_x, s_m, s_l)
            b, mx, lx = self.vecs[s_b], self.vecs[s_m], self.vecs[s_l]
            r = float((a0 * mx + b0 * lx - b).abs().max() / (b.abs().max() + (a0 * mx).abs().max() + (b0 * lx).abs().max()))
            worst = max(worst, r)
        self.last_verify = worst
        if not worst <= self.VERIFY_TOL:
            raise DedalusB200Error(f"shell pencil factorisation failed verification: backward error {worst:.2e}")
        return worst


# ------------------------------------------------------------------------------------------------------------
# Right-hand sides:  sum coef * (state field | grad(state field)) products, evaluated on the dealiased grid
# ------------------------------------------------------------------------------------------------------------
class ShellGradient:
    """Gradient of a shell field of tensor rank `rank` (radial basis k = 0) in coefficient space, regularity components
    (reference SphericalGradient, core/operators.py:3280-3310): two l-independent radial matrices per sign and the
    multiplication AB / dR (db_mmt_apply along r), then ONE db_pair_lincomb with the per-(m, l) symbols xi(mu, l + R) and
    xi(mu, l + R) (l + R).  Output: (3 * 3^rank, pairs, l, r) in the basis k = 1, gradient index first."""

    _cache = {}

    @classmethod
    def cached(cls, basis, rops, rank, dist, dev):
        key = (basis, rank, dist.rank, dist.size, str(dev))
        if key not in cls._cache:
            cls._cache[key] = cls(basis, rops, rank, dist, dev)
        return cls._cache[key]

    def __init__(self, basis, rops, rank, dist, dev):
        import torch
        from .sphere import PairProgram
        if basis.k != 0:
            raise NotImplementedError("gradients of shell fields in a k > 0 radial basis")
        sb = basis.sphere_basis
        j0, j1 = sb.local_pairs(dist)
        self.cshape = (2 * (j1 - j0), basis.coeff_shape[1], basis.coeff_shape[2])
        self.device = dev
        _, ell_map = sb.elements_to_groups()
        ell_pairs = ell_map[0::2][j0:j1]
        in_range = ell_pairs <= sb.Lmax
        lidx = np.minimum(ell_pairs, sb.Lmax)
        q = rops._parts(0)
        dense = lambda M: torch.from_numpy(np.ascontiguousarray(M.toarray())).to(dev)
        self.D0 = {mu: dense((q['DZ'] - (1 - (1 if mu == -1 else 0)) * q['AB']) / rops.dR) for mu in (-1, +1)}
        self.ABm = dense(q['AB'] / rops.dR)
        nin = self.nin = 3 ** rank
        syms, rows = [], []
        for a, mu in ((0, -1), (1, +1), (2, 0)):
            for ci in range(nin):
                rin = tuple(np.unravel_index(ci, (3,) * rank)) if rank else ()
                R = regtotal(rin)
                if mu == 0:
                    rows.append([])
                    continue
                rout = (a,) + rin
                tab = np.zeros(sb.Lmax + 1); tab2 = np.zeros(sb.Lmax + 1)
                for ell in range(sb.Lmax + 1):
                    if regularity_allowed(ell, rin) and regularity_allowed(ell, rout):
                        tab[ell] = xi(mu, ell + R)
                        tab2[ell] = xi(mu, ell + R) * (ell + R)
                off1 = len(syms) * ell_pairs.size; syms.append(np.where(in_range, tab[lidx], 0.0).ravel())
                off2 = len(syms) * ell_pairs.size; syms.append(np.where(in_range, tab2[lidx], 0.0).ravel())
                src_D = (0 if mu == -1 else 1) * nin + ci
                rows.append([(src_D, 1.0, off1), (2 * nin + ci, -float(mu), off2)])
        self.prog = PairProgram(rows, dev, torch.from_numpy(np.concatenate(syms)).to(dev))

    def _mmt(self, mat, inp, out):
        from .lib import get_lib, current_stream
        n_out, n_in = mat.shape
        get_lib().call("db_mmt_apply", mat.data_ptr(), n_out, n_in, inp.data_ptr(), out.data_ptr(), inp.numel() // n_in, 1, current_stream())

    def apply(self, c):
        """c: (3^rank, pairs, l, r) contiguous regularity components."""
        import torch
        Nc0, Nc1, Nr = self.cshape
        nin = self.nin
        stack = torch.empty((3 * nin, Nc0, Nc1, Nr), dtype=torch.float64, device=self.device)
        self._mmt(self.D0[-1], c, stack[0:nin]); self._mmt(self.D0[+1], c, stack[nin:2 * nin]); self._mmt(self.ABm, c, stack[2 * nin:])
        out = torch.empty((3 * nin, Nc0, Nc1, Nr), dtype=torch.float64, device=self.device)
        self.prog.apply(stack, out, Nc0 // 2, Nc1 * Nr, sym_div=Nr)
        return out


class ShellRHSPlan:
    """Explicit terms of a shell IVP (reference: Evaluator walking the RHS trees, core/evaluator.py:95-146).
      1. gradients of state fields in coefficient space: two l-independent radial matrices per sign (db_mmt_apply along r) and
         ONE db_pair_lincomb with the per-(m, l) symbols xi(mu, l + R), xi(mu, l + R) (l + R) (core/operators.py:3280-3310)
      2. every operand to the grid (dedalus_b200/shell.py shell_components_to_grid), one pointwise launch for all products
      3. products back to coefficients in the product basis k = k_A + k_B, converted to the equation's basis with E^dk and
         written into the equation arena (db_mmt_apply with -E^dk folded in).
    Supported: sums of numeric multiples of dot / tensor products whose factors are state fields or gradients of state fields; the
    equations on a sphere (boundary conditions) take field data, written every stage by analysis.BoundaryData."""

    def __init__(self, solver):
        import torch
        from .analysis import BoundaryData, CurvilinearEvaluation, is_shell_boundary
        self.solver = solver
        problem = solver.problem
        dev = self.device = solver.device
        low = ShellLowering(problem)
        basis = self.basis = low.basis
        self.rops = low.rops
        sb = basis.sphere_basis
        dist = self.dist = solver.dist
        j0, j1 = sb.local_pairs(dist)
        Nc0, Nc1, Nr = 2 * (j1 - j0), basis.coeff_shape[1], basis.coeff_shape[2]
        self.cshape = (Nc0, Nc1, Nr)
        self.scales = tuple(basis.dealias)
        gfull = basis.grid_shape(self.scales)
        self.gshape = (gfull[0], gfull[1] // dist.size, gfull[2])
        self.npoints = int(np.prod(self.gshape))
        variables = problem.variables
        plane = Nc0 * Nc1 * Nr
        self.static = []
        operands, op_ids = [], {}

        def operand(e):
            """Grid operand: a state field on the shell or the gradient of one."""
            if id(e) in op_ids:
                return operands[op_ids[id(e)]]
            if isinstance(e, Field) and any(e is v for v in variables) and low.kind_of(e)[0] == 'shell':
                rec = dict(kind='field', field=e, rank=len(e.tensorsig), k=0, g0=sum(3 ** o['rank'] for o in operands))
            elif isinstance(e, ops.Gradient) and isinstance(e.args[0], Field) and any(e.args[0] is v for v in variables):
                f = e.args[0]
                rec = dict(kind='grad', field=f, rank=len(f.tensorsig) + 1, k=1, g0=sum(3 ** o['rank'] for o in operands))
            else:
                raise NotImplementedError(f"RHS factor {type(e).__name__} of a shell problem (state fields and their gradients only)")
            op_ids[id(e)] = len(operands)
            operands.append(rec)
            return rec

        def poly(e):
            if isinstance(e, ops.DotProduct):
                A, B = e.args
                ra, ka, na = poly(A); rb, kb, nb = poly(B)
                d = 3
                nA, nB = na // d, nb // d
                out = {ia * nB + ib: [(x * y, fx + fy) for i in range(d) for x, fx in ra[ia * d + i] for y, fy in rb[i * nB + ib]]
                       for ia in range(nA) for ib in range(nB)}
                return out, ka + kb, nA * nB
            if isinstance(e, ops.Multiply):
                A, B = e.args
                ra, ka, na = poly(A); rb, kb, nb = poly(B)
                return ({ca * nb + cb: [(x * y, fx + fy) for x, fx in ra[ca] for y, fy in rb[cb]] for ca in range(na) for cb in range(nb)},
                        ka + kb, na * nb)
            if isinstance(e, ops.ScalarMul):
                r, k, n = poly(e.args[0])
                return {c: [(x * e.c, f) for x, f in t] for c, t in r.items()}, k, n
            o = operand(e)
            n = 3 ** o['rank']
            return {c: [(1.0, (o['g0'] + c,))] for c in range(n)}, o['k'], n

        self.products = []            # (eq index, rank, k of the product basis, terms per component)
        self.boundary = []            # data of the equations on a sphere (analysis.BoundaryData)
        for ie, eq in enumerate(problem.equations):
            rhs = eq['RHS']
            if not isinstance(rhs, ops.Operand):
                if rhs != 0:
                    self._add_constant(ie, eq, float(rhs), low)
                continue
            if is_shell_boundary(eq):
                self.boundary.append(BoundaryData(solver, ie, rhs, CurvilinearEvaluation(dist)))
                continue
            terms = rhs.args if isinstance(rhs, ops.Add) else [rhs]
            acc, kprod, ncomp = None, None, None
            for t in terms:
                r, k, n = poly(t)
                if acc is None:
                    acc, kprod, ncomp = r, k, n
                else:
                    if k != kprod:
                        raise NotImplementedError("RHS terms in different radial bases")
                    for c, tl in r.items():
                        acc[c] = acc.get(c, []) + tl
            self.products.append(dict(eq=ie, rank=len(eq['tensorsig']), k=kprod, poly=acc, ncomp=ncomp, k_eq=low.kind_of(eq['LHS'])[1]))
        self.operands = operands
        self.n_g = sum(3 ** o['rank'] for o in operands)
        self.n_p = sum(p['ncomp'] for p in self.products)
        if self.n_p == 0:
            return
        # ---- gradient programs, one per tensor rank of the differentiated fields
        self.grads = {}
        for o in operands:
            if o['kind'] == 'grad' and id(o['field']) not in self.grads:
                self.grads[id(o['field'])] = ShellGradient.cached(basis, self.rops, len(o['field'].tensorsig), dist, dev)
        # ---- pointwise program (general kernel)
        coef, fac_ptr, fac, term_ptr = [], [0], [], [0]
        for p in self.products:
            for c in range(p['ncomp']):
                for x, f in p['poly'].get(c, []):
                    if x != 0:
                        coef.append(float(x)); fac.extend(f); fac_ptr.append(len(fac))
                term_ptr.append(len(coef))
        i32 = lambda a: torch.from_numpy(np.asarray(a, dtype=np.int32)).to(dev)
        self.term_ptr, self.fac_ptr, self.fac = i32(term_ptr), i32(fac_ptr), i32(fac if fac else [0])
        self.coef = torch.from_numpy(np.asarray(coef if coef else [0.0])).to(dev)
        self.nfac = len(fac)
        self.g_in = torch.zeros((self.n_g,) + self.gshape, dtype=torch.float64, device=dev)
        self.g_out = torch.zeros((self.n_p,) + self.gshape, dtype=torch.float64, device=dev)
        # the products are transformed straight into their equation's radial basis (evaluate): k_eq must not be below the product's
        for p in self.products:
            if p['k_eq'] < p['k']:
                raise NotImplementedError("RHS in a higher radial basis than its equation")
        self.bases_k = {}

    def _basis_k(self, k):
        if k not in self.bases_k:
            self.bases_k[k] = self.basis.clone_with(k=k)
        return self.bases_k[k]

    def _add_constant(self, ie, eq, value, low):
        """Constant right-hand side of a scalar equation: its l = 0, m = 0 cosine mode (sphere: value / (1 / sqrt 2))."""
        kind, _ = low.kind_of(eq['LHS'])
        if eq['tensorsig']:
            raise NotImplementedError("nonzero constant right-hand side of a tensor equation")
        off = self.solver.eq_arena.offsets[ie]
        if low.basis.sphere_basis.local_pairs(self.solver.dist)[0] != 0:
            return                                             # the l = 0, m = 0 mode lives on the rank that owns pair 0
        if kind == 'sphere':
            self.static.append((off, value * np.sqrt(2)))
        elif kind == 'const':
            self.static.append((off, value))
        else:
            raise NotImplementedError("nonzero constant right-hand side of a shell-interior equation")

    def set_static(self, eq_t):
        eq_t.zero_()
        for off, val in self.static:
            eq_t[off] = val

    def _mmt(self, mat, inp, out):
        from .lib import get_lib, current_stream
        n_out, n_in = mat.shape
        outer = inp.numel() // n_in
        get_lib().call("db_mmt_apply", mat.data_ptr(), n_out, n_in, inp.data_ptr(), out.data_ptr(), outer, 1, current_stream())

    def evaluate(self, eq_t):
        import torch
        from .lib import get_lib, current_stream
        from .shell import shell_components_to_grid, shell_grid_to_components
        from .solvers import Timed
        for bd in self.boundary:
            bd.write(eq_t)
        if self.n_p == 0:
            return
        solver, basis = self.solver, self.basis
        prof = solver.prof
        Nc0, Nc1, Nr = self.cshape
        views = {id(v): view for v, view in zip(solver.state, solver.state_views)}
        grads = {}
        for o in self.operands:
            f = o['field']
            c = views[id(f)].reshape((-1, Nc0, Nc1, Nr))
            if o['kind'] == 'grad':
                if id(f) not in grads:
                    with Timed(prof, "shell_gradient", 8 * 4 * c.numel()):
                        grads[id(f)] = self.grads[id(f)].apply(c)
                c = grads[id(f)]
            with Timed(prof, "shell_backward", 8 * (c.numel() + 3 ** o['rank'] * self.npoints)):
                g = shell_components_to_grid(self._basis_k(o['k']), c.contiguous(), o['rank'], self.scales, self.dist)
            self.g_in[o['g0']:o['g0'] + 3 ** o['rank']].copy_(g)
        with Timed(prof, "pointwise", 8 * self.npoints * (self.n_g + self.n_p)):
            get_lib().call("db_pointwise", self.g_in.data_ptr(), self.g_out.data_ptr(), self.npoints, self.n_g, self.n_p,
                           self.term_ptr.data_ptr(), self.coef.data_ptr(), self.fac_ptr.data_ptr(), self.fac.data_ptr(), self.nfac, current_stream())
        p0 = 0
        for p in self.products:
            # straight into the EQUATION's radial basis: the reference converts F to the equation's bases while it is still on the
            # grid (a copy, core/operators.py:1628-1638), so the one forward transform is the one of basis k_eq -- transforming in the
            # product's basis first and converting with E afterwards truncates differently (visible once |u| is not tiny)
            with Timed(prof, "shell_forward", 8 * p['ncomp'] * (self.npoints + Nc0 * Nc1 * Nr)):
                c = shell_grid_to_components(self._basis_k(p['k_eq']), self.g_out[p0:p0 + p['ncomp']].contiguous(), p['rank'], self.dist)
            off = solver.eq_arena.offsets[p['eq']]
            eq_t[off:off + c.numel()].view(c.shape).copy_(c)
            p0 += p['ncomp']
