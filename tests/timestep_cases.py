"""Shared bodies of the timestepping tests: the IMEX step loops of solvers.py (`_step_multistep`, `_step_rk`) on the Cartesian
(BatchSet, real and complex), sphere (SphereSystems) and shell (ShellSystems) system sets, replayed step by step in long double.
They run through the CPU emulation of the kernels (tests/test_emu_timesteps.py) and on the GPU (tests/test_gpu_1g_timesteps.py).

1. Coefficients, exactly.  The multistep coefficients are derived here from Lagrange weights over the step history in
   `fractions.Fraction` arithmetic, independently of timesteppers.py; the Runge-Kutta tableaux are written down from their
   published definitions in exact (sympy) arithmetic and checked for row sums, order conditions and the diagonal structure the
   loop assumes.  These exact values, not the product's, feed the replay.

2. Replay.  A solver is stepped through a `dt` sequence with every right-hand-side evaluation (sim_time, state arena before, equation
   arena after), every scatter of a new state, every factorisation and solve, and the work vectors after every step copied to the host.
   Work vectors and LU slots start as NaN, so a slot read before it is written poisons the step.  Per step (multistep) or stage (RK)
   the replay gathers X and F from the recorded arenas with the reference gathers (line maps with member signs on the Cartesian path,
   `arena[idx]` on the curvilinear ones), builds the right-hand side from the recorded history and the exact coefficients, and asserts
   the normwise backward error of the new state against the set's own host matrices, the history slots the loop keeps, sim_time at
   every evaluation, which LU slot each stage solved with and when the LHS was refactorised.

Backward error of x against  A x = rhs,  A = a0 M + b0 L,  rhs = sum_t coef_t v_t, per system and right-hand-side column:
    |A x - rhs|_inf / (|A|_inf |x|_inf + sum_t |coef_t| |v_t|_inf)  <=  1e-12,
the level of check_solution in pencil_batch_cases.py."""
import types
from decimal import Decimal, getcontext
from fractions import Fraction as Fr
from math import prod
import numpy as np
import scipy.sparse as sps
import sympy as sp
from dedalus_b200 import examples
from dedalus_b200 import timesteppers as ts
from dedalus_b200.pencils import line_maps
import pencil_batch_cases as PB
import program_interp as pi

LD = np.longdouble
EPS = np.finfo(np.float64).eps
BE_TOL = 1e-12
# first step; a repeated dt (LU reused where the LHS does not change); ratios 1.75 and 0.357 (above and below 1); a return to 4e-3
DTS = (4e-3, 4e-3, 7e-3, 2.5e-3, 2.5e-3, 4e-3)
# a Runge-Kutta step depends on the history only through whether dt changed: first step, a repeat, up by 1.75, down by 4 / 7 to an
# earlier dt
RK_DTS = (4e-3, 4e-3, 7e-3, 4e-3)
MULTISTEP = ("CNAB1", "SBDF1", "CNAB2", "MCNAB2", "SBDF2", "CNLF2", "SBDF3", "SBDF4")
RUNGE_KUTTA = ("RK111", "RK222", "RK443", "RKSMR", "RKGFY")
ALL_SCHEMES = MULTISTEP + RUNGE_KUTTA


def scheme_class(name):
    return ts.schemes.get(name, getattr(ts, name))


def to_ld(x):
    """Exact rational or sympy number -> long double, correctly rounded to well below long-double precision."""
    getcontext().prec = 40
    if isinstance(x, Fr):
        return LD(str(Decimal(x.numerator) / Decimal(x.denominator)))
    return LD(str(sp.N(x, 40)))


# ---------------------------------------------------------------------------------------------------------------------------------
# 1. exact coefficients
# ---------------------------------------------------------------------------------------------------------------------------------
def lagrange(nodes, p, deriv=False):
    """Weights w_j with  f(p) = sum_j w_j f(nodes_j)  (or f'(p) with deriv=True) for every polynomial of degree < len(nodes)."""
    w = []
    for j, tj in enumerate(nodes):
        others = [t for i, t in enumerate(nodes) if i != j]
        den = prod((tj - t for t in others), start=Fr(1))
        if deriv:
            num = sum((prod((p - t for i, t in enumerate(others) if i != m), start=Fr(1)) for m in range(len(others))), start=Fr(0))
        else:
            num = prod((p - t for t in others), start=Fr(1))
        w.append(num / den)
    return w


def second_order_weights(nodes, p, fixed):
    """Weights on nodes[0], nodes[1] that, with the given weights on the remaining nodes, sum to 1 and have no first moment about p
    (second-order approximation of the value at p)."""
    rest = sum(fixed, start=Fr(0))
    moment = sum((w * (t - p) for w, t in zip(fixed, nodes[2:])), start=Fr(0))
    d0, d1 = nodes[0] - p, nodes[1] - p
    # w0 + w1 = 1 - rest;  w0 d0 + w1 d1 = -moment
    w0 = (-moment - (1 - rest) * d1) / (d0 - d1)
    return [w0, 1 - rest - w0] + list(fixed)


def startup_scheme(name, iteration):
    """The scheme run at `iteration` (0-based) while the history fills: SBDFk runs SBDF(min(k, iteration + 1)); the Crank-Nicolson
    schemes start with one CNAB1 step."""
    if name.startswith("SBDF"):
        return f"SBDF{min(int(name[4]), iteration + 1)}"
    return name if iteration >= 1 else "CNAB1"


def exact_multistep(name, dts, iteration):
    """(a, b, c) as lists of Fractions: a_j M.X(t_{n-j}) + b_j L.X(t_{n-j}) = c_j F(t_{n-j}) for the step of size dts[0] from t_{n-1} to
    t_n; dts = (k_0, k_1, ...) newest first."""
    name = startup_scheme(name, iteration)
    k = [Fr(x) for x in dts]
    t = [Fr(0)]
    for kk in k:
        t.append(t[-1] - kk)
    if name.startswith("SBDF"):
        s = int(name[4])
        a = lagrange(t[:s + 1], t[0], deriv=True)               # BDFs: derivative at t_n of the interpolant through s + 1 points
        b = [Fr(1)] + [Fr(0)] * s                                # L X implicit at t_n
        c = [Fr(0)] + lagrange(t[1:s + 1], t[0])                  # F extrapolated to t_n from t_{n-1} .. t_{n-s}
    elif name in ("CNAB1", "CNAB2", "MCNAB2"):
        s = int(name[-1])
        mid = (t[0] + t[1]) / 2
        a = lagrange(t[:2], mid, deriv=True)                      # BDF1 (the derivative of a line is the same everywhere)
        b = lagrange(t[:2], mid) if name != "MCNAB2" else second_order_weights(t[:3], mid, [Fr(1, 16)])
        c = [Fr(0)] + lagrange(t[1:s + 1], mid)                   # F extrapolated to the midpoint t_{n-1/2}
    elif name == "CNLF2":
        a = lagrange(t[:3], t[1], deriv=True)                     # centred derivative at t_{n-1}
        b = second_order_weights(t[:3], t[1], [Fr(1, 2)])         # L X at t_{n-1}, half the weight on t_{n-2}
        c = [Fr(0), Fr(1)]                                       # F at t_{n-1}
    else:
        raise KeyError(name)
    return a, b, c


def _padded(x, n):
    return list(x) + [0] * (n - len(x))


def check_multistep_coefficients(name, seed):
    """compute_coefficients against the exact values at every startup iteration and past it, for random rational step ratios in
    [1/5, 5] and for a constant step: |a - a_exact| <= 1e-13 sum |a_exact|, the same for b and c."""
    cls = scheme_class(name)
    rng = np.random.default_rng(seed)
    histories = [[1e-2] * cls.steps]
    for _ in range(6):
        ks = [Fr(1, 100)]
        for _ in range(cls.steps - 1):
            ks.append(ks[-1] * Fr(int(rng.integers(5, 26)), int(rng.integers(5, 26))))      # ratio p / q in [1/5, 5]
        histories.append([float(x) for x in ks])
    for dts in histories:
        for it in range(cls.steps + 1):
            got = cls.compute_coefficients(list(dts), it)
            want = exact_multistep(name, dts, it)
            for label, g, w in zip("abc", got, want):
                n = max(len(g), len(w))
                g, w = _padded(g, n), _padded(w, n)
                scale = float(sum(abs(x) for x in w))
                err = max(abs(Fr(float(gj)) - wj) for gj, wj in zip(g, w))
                assert float(err) <= 1e-13 * scale, (name, it, dts, label, [float(x) for x in w], list(g))


# Runge-Kutta tableaux from their published definitions: (c, A, H) of  (M + k H_ii L) X_i = M X_0 + k sum_j<i A_ij F_j - k sum_j<i H_ij L X_j
def exact_tableau(name):
    R = sp.Rational
    if name == "RK111":                                          # forward / backward Euler
        c, A, H = [0, 1], [[0, 0], [1, 0]], [[0, 0], [0, 1]]
    elif name == "RK222":                                        # Ascher, Ruuth & Spiteri 1997, (2, 2, 2)
        g = (2 - sp.sqrt(2)) / 2
        d = 1 - 1 / (2 * g)
        c, A, H = [0, g, 1], [[0, 0, 0], [g, 0, 0], [d, 1 - d, 0]], [[0, 0, 0], [0, g, 0], [0, 1 - g, g]]
    elif name == "RK443":                                        # Ascher, Ruuth & Spiteri 1997, (4, 4, 3)
        c = [0, R(1, 2), R(2, 3), R(1, 2), 1]
        A = [[0] * 5, [R(1, 2), 0, 0, 0, 0], [R(11, 18), R(1, 18), 0, 0, 0], [R(5, 6), R(-5, 6), R(1, 2), 0, 0],
             [R(1, 4), R(7, 4), R(3, 4), R(-7, 4), 0]]
        H = [[0] * 5, [0, R(1, 2), 0, 0, 0], [0, R(1, 6), R(1, 2), 0, 0], [0, R(-1, 2), R(1, 2), R(1, 2), 0],
             [0, R(3, 2), R(-3, 2), R(1, 2), R(1, 2)]]
    elif name == "RKSMR":                                        # Spalart, Moser & Rogers 1991, as cumulative stages
        a1, a2, a3 = R(29, 96), R(-3, 40), R(1, 6)
        b1, b2, b3 = R(37, 160), R(5, 24), R(1, 6)
        g1, g2, g3 = R(8, 15), R(5, 12), R(3, 4)
        z2, z3 = R(-17, 60), R(-5, 12)
        c = [0, R(8, 15), R(2, 3), 1]
        A = [[0] * 4, [g1, 0, 0, 0], [g1 + z2, g2, 0, 0], [g1 + z2, g2 + z3, g3, 0]]
        H = [[0] * 4, [a1, b1, 0, 0], [a1, b1 + a2, b2, 0], [a1, b1 + a2, b2 + a3, b3]]
    elif name == "RKGFY":                                        # Heun with Crank-Nicolson
        c = [0, 1, 1]
        A = [[0, 0, 0], [1, 0, 0], [R(1, 2), R(1, 2), 0]]
        H = [[0, 0, 0], [R(1, 2), R(1, 2), 0], [R(1, 2), 0, R(1, 2)]]
    else:
        raise KeyError(name)
    return sp.Matrix(c), sp.Matrix(A), sp.Matrix(H)


RK_ORDER = dict(RK111=1, RK222=2, RK443=3, RKSMR=2, RKGFY=2)


def order_conditions(c, A, H, p):
    """Residuals of the order-p conditions (p <= 4) of the additive pair (A, H) with shared abscissae c and the last rows as weights: one
    per rooted tree of order p and colouring of its internal vertices by A or H (the leaves are c, since the row sums agree)."""
    s = A.shape[0]
    q = sp.Rational
    cp = lambda k: sp.Matrix([x**k for x in c])
    res = []
    for b in (A[s - 1, :], H[s - 1, :]):
        if p == 1:
            res.append((b * sp.ones(s, 1))[0] - 1)
        if p == 2:
            res.append((b * c)[0] - q(1, 2))
        if p == 3:
            res.append((b * cp(2))[0] - q(1, 3))
            for X in (A, H):
                res.append((b * X * c)[0] - q(1, 6))
        if p == 4:
            res.append((b * cp(3))[0] - q(1, 4))
            for X in (A, H):
                res.append((b * sp.matrix_multiply_elementwise(c, X * c))[0] - q(1, 8))
                res.append((b * X * cp(2))[0] - q(1, 12))
                for Y in (A, H):
                    res.append((b * X * Y * c)[0] - q(1, 24))
    return [sp.nsimplify(sp.simplify(r)) for r in res]


def check_rk_tableau(name):
    """Exact: c = row sums of A and of H; A strictly and H weakly lower triangular with zero first rows (the loop reads only j < i and
    puts H_ii on the left); the last rows satisfy every condition of the scheme's order and not all of the next; the number of distinct
    H_ii is the number of LU slots _prepare_batches allocates.  The product's floats are within 4 ulps of the exact values (RK222 computes
    its delta = 1 - 1 / (2 gamma) = -sqrt(2) / 2 with a cancellation: 2 ulps)."""
    cls = scheme_class(name)
    c, A, H = exact_tableau(name)
    s = cls.stages
    assert A.shape == H.shape == (s + 1, s + 1) and c.shape == (s + 1, 1)
    for X in (A, H):
        assert all(sp.simplify(sum(X[i, :]) - c[i]) == 0 for i in range(s + 1)), (name, "row sums")
    assert all(A[i, j] == 0 for i in range(s + 1) for j in range(i, s + 1)), (name, "A not strictly lower triangular")
    assert all(H[i, j] == 0 for i in range(s + 1) for j in range(i + 1, s + 1)) and all(H[0, j] == 0 for j in range(s + 1))
    assert c[s] == 1, (name, "the last stage is the new state")
    p = RK_ORDER[name]
    for q in range(1, p + 1):
        assert all(r == 0 for r in order_conditions(c, A, H, q)), (name, "order", q)
    assert any(r != 0 for r in order_conditions(c, A, H, p + 1)), (name, "satisfies order", p + 1)
    distinct = {sp.nsimplify(sp.simplify(H[i, i])) for i in range(1, s + 1)}
    assert len(distinct) == len({float(cls.H[i, i]) for i in range(1, s + 1)}), (name, "distinct H_ii")
    for got, want in ((cls.c, c), (cls.A, A), (cls.H, H)):
        got = np.asarray(got, dtype=np.float64).reshape(want.shape)
        for idx in np.ndindex(*want.shape):
            w = to_ld(want[idx])
            assert abs(LD(got[idx]) - w) <= 4 * EPS * abs(w), (name, idx, got[idx], w)
    return len(distinct)


# ---------------------------------------------------------------------------------------------------------------------------------
# problems
# ---------------------------------------------------------------------------------------------------------------------------------
def rayleigh_benard(dim=2, Nh=16, Nz=16):
    """Rayleigh-Benard with the O(1) random velocity of tall_pencils.py, resolved in z: F carries signal in every variable."""
    pb = examples.rayleigh_benard(dim=dim, Nh=Nh, Nz=Nz)
    examples.rayleigh_benard_initial_condition(pb['b'], pb['bases'], pb['Lz'])
    u = pb['u']
    u.fill_random('g', seed=7, distribution='normal', scale=1.0)
    uc = np.array(u['c']); uc[..., Nz // 2:] = 0; u['c'] = uc
    return pb, 1.0


def ginzburg_landau(Nx=16, Nz=12):
    pb = examples.complex_ginzburg_landau(Nx, Nz)
    examples.complex_ginzburg_landau_initial_condition(pb['u'], pb['bases'])
    return pb, 1.0


def shallow_water(Nphi=16, Ntheta=8):
    pb = examples.shallow_water(Nphi, Ntheta)
    examples.shallow_water_initial_condition(pb['u'], pb['h'], pb['basis'], pb['units'])
    return pb, pb['timestep'] / DTS[0]


def shell_convection(Nphi=16, Ntheta=8, Nr=6):
    """Shell convection with a random O(1e-2) velocity on top of the conductive profile, so that both products carry signal."""
    pb = examples.shell_convection(Nphi, Ntheta, Nr)
    examples.shell_convection_initial_condition(pb['b'], pb['shell'], pb['Ri'], pb['Ro'])
    pb['u'].fill_random('g', seed=5, distribution='normal', scale=1e-2)
    return pb, 1.0


# ---------------------------------------------------------------------------------------------------------------------------------
# the system sets seen from the host: blocks of (C columns sharing one matrix) x (n rows) x (S matrices)
# ---------------------------------------------------------------------------------------------------------------------------------
def _host(t):
    return t.detach().cpu().numpy().copy()


class _HostVecs:
    """Case.vec of pencil_batch_cases on host copies of a batch's work vectors."""
    host = staticmethod(lambda a: a)
    vec = PB.Case.vec


class CartesianView:
    """BatchSet: block = batch, columns = members (line signs applied by the gathers), one matrix per member pencil.  The matrices and
    line maps are taken in the batch's current column order; M X, L X and F are row-space vectors, which a new column order leaves
    alone, so the replay of steps taken before a re-order is valid in the final order.  The X slot is column-space: it is read only
    where it was written in the final order."""
    kind = "cartesian"

    def __init__(self, solver):
        self.solver = solver
        self.blocks = []
        for db in solver.bset.items:
            b = db.batch
            self.blocks.append(dict(db=db, n=db.n, S=db.S, C=db.R, cols=line_maps(b, solver.var_arena, 'cols'),
                                    rows=line_maps(b, solver.eq_arena, 'rows'),
                                    mats=[(b.matrix('M', g), b.matrix('L', g)) for g in b.groups]))

    @staticmethod
    def snapshot(bset):
        return [[_host(v) for v in db.vecs] for db in bset.items]

    def gather(self, i, side, arena):
        blk = self.blocks[i]
        maps = blk['cols' if side == 0 else 'rows']
        return np.stack([pi.gather(maps, arena, blk['n'], blk['S'], member=m) for m in range(blk['C'])])

    def slot(self, snap, i, slot):
        db = self.blocks[i]['db']
        v = _HostVecs().vec(types.SimpleNamespace(vecs=snap[i], n=db.n, ld=db.ld, R_alloc=db.R_alloc), slot)
        return v[:db.R, :, :db.S]

    def valid(self, i):
        blk = self.blocks[i]
        return np.ones((blk['C'], blk['n'], blk['S']), dtype=bool)


class _IndexView:
    """Curvilinear sets: the vectors are  vec[e] = arena[idx[e]]  (0 where idx < 0)."""

    @staticmethod
    def snapshot(bset):
        return [_host(v) for v in bset.vecs]

    def gather(self, i, side, arena):
        blk = self.blocks[i]
        idx = blk['xi' if side == 0 else 'fi']
        v = np.where(idx >= 0, arena[np.maximum(idx, 0)], 0.0)
        return self._shape(blk, v)

    def slot(self, snap, i, slot):
        blk = self.blocks[i]
        return self._shape(blk, snap[slot][blk['off']:blk['off'] + blk['n'] * blk['C']])

    def valid(self, i):
        """Unknowns with a place in the state arena; the others (padding, constants outside their column) are dropped by the
        scatter."""
        blk = self.blocks[i]
        return self._shape(blk, blk['xi'] >= 0)


class SphereView(_IndexView):
    """SphereSystems: one banded system per m, one right-hand-side column."""
    kind = "sphere"

    def __init__(self, solver):
        self.blocks = [dict(n=s['n'], C=1, S=1, xi=np.asarray(s['xi']), fi=np.asarray(s['fi']), off=s['vec_off'],
                            mats=[(s['M'].tocsr(), s['L'].tocsr())]) for s in solver.bset.systems]

    @staticmethod
    def _shape(blk, v):
        return v.reshape(1, blk['n'], 1)


class ShellView(_IndexView):
    """ShellSystems: one dense system per l (its M and L as kept on the device), columns (m, cos / -sin) stored row-major (n, ncols)."""
    kind = "shell"

    def __init__(self, solver):
        from dedalus_b200.lib import DenseSys
        bs = solver.bset
        desc = (DenseSys * bs.nsys).from_buffer_copy(_host(bs.desc).tobytes())
        M, L = _host(bs.M_t), _host(bs.L_t)
        xi, fi = _host(bs.idx[0]), _host(bs.idx[1])
        self.blocks = []
        for l in range(bs.nsys):
            nc, off, n = int(desc[l].ncols), int(desc[l].vec_off), bs.n
            if nc == 0:
                continue
            self.blocks.append(dict(n=n, C=nc, S=1, off=off, xi=xi[off:off + n * nc], fi=fi[off:off + n * nc],
                                    mats=[(sps.csr_matrix(M[l]), sps.csr_matrix(L[l]))]))

    @staticmethod
    def _shape(blk, v):
        return np.ascontiguousarray(v.reshape(blk['n'], blk['C']).T)[:, :, None]


def view_of(solver):
    return ShellView(solver) if solver.shell else SphereView(solver) if solver.curvilinear else CartesianView(solver)


def fill_nan(bset):
    """Every work vector and LU slot of a system set to NaN."""
    nan = float('nan')
    if hasattr(bset, 'items'):
        for db in bset.items:
            for v in list(db.vecs) + list(db.lu.values()):
                v.fill_(nan)
    else:
        for v in list(bset.vecs) + list(bset.lu):
            v.fill_(nan)


# ---------------------------------------------------------------------------------------------------------------------------------
# 2. recording
# ---------------------------------------------------------------------------------------------------------------------------------
class Run:
    """One solver stepped through `dts`, every device event of interest copied to the host.

    edit: {step index: callable(run)} applied between steps (host edits of the state); reorder_at: step index at which a test double
    around BatchSet.probe reports one member above VERIFY_TOL once, so that factor_verified re-orders that batch."""

    def __init__(self, solver, scheme, dts, pb=None, edit=None, reorder_at=None):
        self.solver, self.name, self.cls, self.dts, self.pb = solver, scheme, scheme_class(scheme), [float(x) for x in dts], pb
        self.steps = []
        solver._init_device()
        cls = self.cls
        if cls.kind == "rk":
            solver._prepare_batches(1.0, self.dts[0] * float(cls.H[1, 1]))      # as the first step would create it
        else:
            a, b, _ = cls.compute_coefficients([self.dts[0]] + [0.0] * (cls.steps - 1), 0)
            solver._prepare_batches(a[0], b[0])
        bs = self.bset = solver.bset
        fill_nan(bs)
        snapshot = (ShellView if solver.shell else SphereView if solver.curvilinear else CartesianView).snapshot
        plan = solver.rhs_plan
        evaluate, mark, factor, solve, verify = plan.evaluate, solver._mark_state_on_device, bs.factor, bs.solve, bs.factor_verified
        self.verifying = False
        enforce = solver.enforce_hermitian_symmetry

        def rec_evaluate(eq_t):
            before = _host(solver.state_t)
            out = evaluate(eq_t)
            self.cur['evals'].append((solver.sim_time, before, _host(eq_t)))
            return out

        def rec_mark():
            self.cur['scatters'].append(_host(solver.state_t))
            self.cur['solved'].append(snapshot(bs))
            self.cur['order'].append(bs.reorders)
            return mark()

        def rec_factor(lu_slot, a0, b0):
            self.cur['factors'].append((lu_slot, float(a0), float(b0)))
            return factor(lu_slot, a0, b0)

        def rec_solve(lu_slot, x_slot, terms):
            if not self.verifying:                    # the probe solves of factor_verified are not steps
                self.cur['solves'].append((lu_slot, x_slot, list(terms)))
            return solve(lu_slot, x_slot, terms)

        def rec_verify(lhs, slots):
            self.verifying = True
            try:
                return verify(lhs, slots)
            finally:
                self.verifying = False

        def rec_enforce(fields):
            self.cur['enforced'] += 1
            return enforce(fields)

        plan.evaluate, solver._mark_state_on_device, bs.factor, bs.solve = rec_evaluate, rec_mark, rec_factor, rec_solve
        bs.factor_verified = rec_verify
        solver.enforce_hermitian_symmetry = rec_enforce
        self.armed = reorder_at is not None
        if self.armed:
            probe = bs.probe

            def forced_probe(lu_slot, a0, b0, slots, seed=1234):
                res = probe(lu_slot, a0, b0, slots, seed)
                if self.armed and len(self.steps) == reorder_at:
                    res[0] = res[0].copy(); res[0][0] = 10 * bs.VERIFY_TOL
                    self.armed = False
                return res
            bs.probe = forced_probe
        edit = edit or {}
        for s, dt in enumerate(self.dts):
            if s in edit:
                self.edited = edit[s](self)
            self.cur = dict(dt=dt, evals=[], scatters=[], solved=[], order=[], factors=[], solves=[], enforced=0)
            solver.step(dt)
            self.cur['after'] = _host(solver.state_t)
            self.cur['vecs'] = snapshot(bs)
            self.cur['reorders'] = bs.reorders
            if cls.kind == "rk":
                self.cur['slots'] = dict(MX0=solver.slot_MX0, LX=list(solver.slot_LX), F=list(solver.slot_F))
            else:
                self.cur['slots'] = dict(MX=list(solver.slot_MX), LX=list(solver.slot_LX), F=list(solver.slot_F))
            self.steps.append(self.cur)


# ---------------------------------------------------------------------------------------------------------------------------------
# replay
# ---------------------------------------------------------------------------------------------------------------------------------
class Replay:
    """Long-double products of the recorded states with each block's host matrices (cached per recorded array)."""

    def __init__(self, run):
        self.run, self.view = run, view_of(run.solver)
        self._x, self._p, self._f = {}, {}, {}

    def x(self, key, arena):
        if key not in self._x:
            self._x[key] = [self.view.gather(i, 0, arena) for i in range(len(self.view.blocks))]
        return self._x[key]

    def f(self, key, arena):
        if key not in self._f:
            self._f[key] = [self.view.gather(i, 1, arena).astype(LD) for i in range(len(self.view.blocks))]
        return self._f[key]

    def products(self, key, arena=None, xs=None):
        """Per block: (M X, L X, |M||X|, |L||X|), each (C, n, S) in long double, of X gathered from `arena` or given per block (xs)."""
        if key not in self._p:
            out = []
            for blk, x in zip(self.view.blocks, self.x(key, arena) if xs is None else xs):
                res = [np.zeros(x.shape, dtype=LD) for _ in range(4)]
                for s, (M, L) in enumerate(blk['mats']):
                    xs = x[:, :, s].T
                    for k, A in enumerate((M, L)):
                        res[k][:, :, s] = PB._ld_matvec(A, xs).T
                        res[k + 2][:, :, s] = PB._ld_matvec(abs(A), np.abs(xs)).T
                out.append(res)
            self._p[key] = out
        return self._p[key]

    def backward_error(self, a0, b0, xkey, xarena, terms):
        """Worst backward error over blocks, matrices and columns of x (gathered from xarena) for  (a0 M + b0 L) x = sum coef v;
        terms: list of (coef, per-block (C, n, S) arrays)."""
        worst = 0.0
        prods = self.products(xkey, xarena)
        for i, blk in enumerate(self.view.blocks):
            mx, lx = prods[i][0], prods[i][1]
            x = self.x(xkey, xarena)[i].astype(LD)
            ax = a0 * mx + b0 * lx
            rhs = np.zeros(x.shape, dtype=LD)
            den = np.zeros(x.shape[::2], dtype=LD)                                       # (C, S)
            for coef, v in terms:
                rhs += coef * v[i]
                den += abs(coef) * np.abs(v[i]).max(axis=1)
            anorm = np.array([abs(float(a0) * M + float(b0) * L).sum(axis=1).max() for M, L in blk['mats']], dtype=LD)
            den += anorm[None, :] * np.abs(x).max(axis=1)
            num = np.abs(ax - rhs).max(axis=1)
            with np.errstate(invalid='ignore', divide='ignore'):
                be = np.where(den > 0, num / den, np.where(num > 0, np.inf, 0))
            be = float(np.nan_to_num(be.astype(np.float64), nan=np.inf).max())
            assert be <= BE_TOL, (self.view.kind, "block", i, dict(n=blk['n'], C=blk['C'], S=blk['S']), "backward error", be)
            worst = max(worst, be)
        return worst

    def check_product_slot(self, snap, slot, which, key, arena, tag, xs=None):
        """A work vector against M X or L X of a recorded state, componentwise within (nnz_row + 2) eps (|A| |x|)."""
        prods = self.products(key, arena, xs)
        k = 0 if which == 'M' else 1
        for i, blk in enumerate(self.view.blocks):
            got = self.view.slot(snap, i, slot)
            ref, mag = prods[i][k], prods[i][k + 2]
            nnz = np.stack([np.diff(mats[k].indptr) for mats in blk['mats']], axis=1)            # (n, S)
            bound = (nnz[None] + 2) * EPS * mag
            err = np.abs(got - ref)
            assert np.all(err <= bound), (tag, which, "block", i, float(np.nan_to_num((err - bound).astype(np.float64), nan=np.inf).max()))

    def check_scatter(self, snap, slot, arena, tag):
        """The state arena after a scatter holds the solved work vector bitwise (member signs undone) wherever an unknown has a place."""
        for i in range(len(self.view.blocks)):
            got, ref, valid = self.view.gather(i, 0, arena), self.view.slot(snap, i, slot), self.view.valid(i)
            assert got[valid].tobytes() == ref[valid].tobytes(), (tag, "scatter", "block", i)

    def check_move_slot(self, snap, slot, key, arena, tag):
        """A gathered right-hand side bitwise equal to the reference gather of the recorded equation arena."""
        for i in range(len(self.view.blocks)):
            got = self.view.slot(snap, i, slot)
            ref = self.view.gather(i, 1, arena)
            assert got.tobytes() == ref.tobytes(), (tag, "F slot", "block", i)


def _time_check(got, want, nulp, tag):
    """got (double) within nulp ulps of want (long double)."""
    assert abs(LD(got) - want) <= nulp * LD(np.spacing(abs(float(want)))), (tag, float(got), float(want), float(LD(got) - want))


def check_step_start(sim, s, t_exact, t_loop, tag):
    """The time at the start of step s: what the loop's additions of the step sizes give, bitwise, and within the one rounding per
    addition (s / 2 ulps, at least one) of the long-double sum of the previous steps."""
    assert sim == t_loop, (tag, "start of step", sim, t_loop)
    _time_check(sim, t_exact, max(1.0, s / 2), tag)


def replay_multistep(run):
    rp = Replay(run)
    steps, name, cls = run.steps, run.name, run.cls
    worst, refactors, prev_key, t, t_loop = 0.0, [], None, LD(0), 0.0
    Xk = lambda s: ("X", s)
    for s, st in enumerate(steps):
        assert len(st['evals']) == len(st['scatters']) == len(st['solves']) == 1, (name, s)
        hist = [steps[r]['dt'] for r in range(s, -1, -1)]
        a, b, c = exact_multistep(name, hist, s)
        # sim_time at the evaluation: the sum of the previous steps
        check_step_start(st['evals'][0][0], s, t, t_loop, (name, s, "sim_time"))
        t += LD(st['dt']); t_loop += st['dt']
        # the right-hand side of step s (new time t_{s+1}) from the recorded history: F^r and X^r at the start of step r
        assert not any(x != 0 for x in a[s + 2:] + b[s + 2:] + c[s + 2:]), (name, s, "the startup reads past the history")
        terms = []
        for j in range(1, len(c)):
            if c[j] != 0:
                r = s + 1 - j
                terms.append((to_ld(c[j]), rp.f(("F", r), steps[r]['evals'][0][2])))
        for j in range(1, len(a)):
            if a[j] != 0:
                r = s + 1 - j
                terms.append((-to_ld(a[j]), [p[0] for p in rp.products(Xk(r), steps[r]['evals'][0][1])]))
        for j in range(1, len(b)):
            if b[j] != 0:
                r = s + 1 - j
                terms.append((-to_ld(b[j]), [p[1] for p in rp.products(Xk(r), steps[r]['evals'][0][1])]))
        a0, b0 = to_ld(a[0]), to_ld(b[0])
        worst = max(worst, rp.backward_error(a0, b0, ("new", s), st['scatters'][0], terms))
        if st['order'][0] == run.bset.reorders:          # the solved X slot is column-space: readable in the final column order only
            rp.check_scatter(st['solved'][0], st['solves'][0][1], st['scatters'][0], (name, s))
        # LHS refactorised exactly when (a0, b0) changed, with the exact values rounded
        key = (a[0], b[0])
        refactors.append(key != prev_key)
        prev_key = key
        if refactors[-1]:
            assert st['factors'] and all(f[0] == 0 for f in st['factors']), (name, s, st['factors'])
            for _, fa, fb in st['factors']:
                assert abs(LD(fa) - a0) <= 2 * EPS * abs(a0) and abs(LD(fb) - b0) <= 2 * EPS * abs(b0), (name, s, fa, fb)
        else:
            assert not st['factors'], (name, s, "refactorised with an unchanged LHS")
        assert st['solves'][0][0] == 0
        # the history the loop keeps: slot_MX[j], slot_LX[j], slot_F[j] hold M X^{s-j}, L X^{s-j}, F^{s-j}
        sl = st['slots']
        for j in range(cls.amax):
            if s - j >= 0:
                rp.check_product_slot(st['vecs'], sl['MX'][j], 'M', Xk(s - j), steps[s - j]['evals'][0][1], (name, s, "MX", j))
        for j in range(cls.bmax):
            if s - j >= 0:
                rp.check_product_slot(st['vecs'], sl['LX'][j], 'L', Xk(s - j), steps[s - j]['evals'][0][1], (name, s, "LX", j))
        for j in range(cls.cmax):
            if s - j >= 0:
                rp.check_move_slot(st['vecs'], sl['F'][j], ("F", s - j), steps[s - j]['evals'][0][2], (name, s, "F", j))
    return summary(run, worst, refactors, expected_terms=max_terms_multistep(run))


def max_terms_multistep(run):
    out = 0
    for s in range(len(run.steps)):
        a, b, c = exact_multistep(run.name, [run.steps[r]['dt'] for r in range(s, -1, -1)], s)
        out = max(out, sum(x != 0 for x in a[1:]) + sum(x != 0 for x in b[1:]) + sum(x != 0 for x in c[1:]))
    return out


def replay_rk(run):
    rp = Replay(run)
    steps, name, cls = run.steps, run.name, run.cls
    c, A, H = exact_tableau(name)
    S = cls.stages
    cl, Al, Hl = ([[to_ld(X[i, j]) for j in range(X.shape[1])] for i in range(X.shape[0])] for X in (c, A, H))
    hii = [sp.nsimplify(sp.simplify(H[i, i])) for i in range(S + 1)]
    worst, refactors, t, t_loop, prev = 0.0, [], LD(0), 0.0, None
    max_terms = 0
    for s, st in enumerate(steps):
        assert len(st['evals']) == len(st['scatters']) == len(st['solves']) == S, (name, s)
        k = LD(st['dt'])
        refactors.append(st['dt'] != prev)
        prev = st['dt']
        # which LU slot holds which H_ii: from the factorisations of this step (or the last one that had any)
        if refactors[-1]:
            slot_b0 = {}
            for lu, fa, fb in st['factors']:
                assert fa == 1.0
                slot_b0[lu] = LD(fb)
            assert len(slot_b0) == len(set(hii[1:])) == len(st['factors']), (name, s, st['factors'])
        else:
            assert not st['factors'], (name, s, "refactorised with an unchanged dt")
        X = lambda i: steps[s]['evals'][i][1]
        for i in range(1, S + 1):
            sim, _, _ = st['evals'][i - 1]
            if i == 1:
                check_step_start(sim, s, t, t_loop, (name, s, "sim_time"))
                t_start = LD(sim)
            _time_check(sim, t_start + k * cl[i - 1][0], 1, (name, s, i, "sim_time"))      # t0 + k c_{i-1}
            terms = [(LD(1), [p[0] for p in rp.products(("X", s, 0), X(0))])]
            for j in range(i):
                if A[i, j] != 0:
                    terms.append((k * Al[i][j], rp.f(("F", s, j), st['evals'][j][2])))
                if H[i, j] != 0:
                    terms.append((-k * Hl[i][j], [p[1] for p in rp.products(("X", s, j), X(j))]))
            max_terms = max(max_terms, len(terms))
            b0 = k * Hl[i][i]
            lu = st['solves'][i - 1][0]
            assert abs(slot_b0[lu] - b0) <= 2 * EPS * abs(b0), (name, s, i, "solved with the LU of another stage", lu)
            xkey = ("X", s, i) if i < S else ("new", s)
            xarena = X(i) if i < S else st['scatters'][S - 1]
            assert st['scatters'][i - 1].tobytes() == xarena.tobytes(), (name, s, i, "the next stage did not start from the scatter")
            worst = max(worst, rp.backward_error(LD(1), b0, xkey, xarena, terms))
            rp.check_scatter(st['solved'][i - 1], st['solves'][i - 1][1], st['scatters'][i - 1], (name, s, i))
        t += k; t_loop += st['dt']
        # the vectors the loop keeps: MX0 = M X_0 and LX[0] = L X_0 of the gathered state; LX[j] (j >= 1) = L X_j of the solved X
        # slot, which also holds the unknowns the scatter drops (rounding-level values in rows without a right-hand side)
        sl = st['slots']
        rp.check_product_slot(st['vecs'], sl['MX0'], 'M', ("X", s, 0), X(0), (name, s, "MX0"))
        for j in range(S):
            if any(H[i, j] != 0 for i in range(j + 1, S + 1)):
                xs = None if j == 0 else [rp.view.slot(st['solved'][j - 1], b, st['solves'][j - 1][1]) for b in range(len(rp.view.blocks))]
                rp.check_product_slot(st['vecs'], sl['LX'][j], 'L', ("solved", s, j) if j else ("X", s, 0), X(j), (name, s, "LX", j), xs)
            rp.check_move_slot(st['vecs'], sl['F'][j], ("F", s, j), st['evals'][j][2], (name, s, "F", j))
    return summary(run, worst, refactors, expected_terms=max_terms, expected_lu=len(set(hii[1:])))


def summary(run, worst, refactors, expected_terms, expected_lu=1):
    """The edges a run reached, from host data, checked against what the exact coefficients ask for."""
    lu_used = {sv[0] for st in run.steps for sv in st['solves']}
    terms = max(len(sv[2]) for st in run.steps for sv in st['solves'])
    seen = [bool(st['factors']) for st in run.steps]
    assert seen == refactors, (run.name, "refactorisations", seen, refactors)
    assert len(lu_used) == expected_lu, (run.name, "LU slots used", lu_used)
    assert terms == expected_terms, (run.name, "solve terms", terms, expected_terms)
    return dict(worst=worst, lu_slots=len(lu_used), max_terms=terms, refactors=refactors, reorders=run.bset.reorders,
                kind=view_of(run.solver).kind)


def replay(run):
    return replay_rk(run) if run.cls.kind == "rk" else replay_multistep(run)


# ---------------------------------------------------------------------------------------------------------------------------------
# cases
# ---------------------------------------------------------------------------------------------------------------------------------
def run_case(make, scheme, dts=None, solver_kw=None, **run_kw):
    """Build the problem, step it through dts (default DTS or RK_DTS, scaled by the problem's time unit) and replay; returns
    (summary, run)."""
    if dts is None:
        dts = RK_DTS if scheme in RUNGE_KUTTA else DTS
    pb, unit = make()
    solver = pb['problem'].build_solver(scheme_class(scheme), **(solver_kw or {}))
    run = Run(solver, scheme, [unit * d for d in dts], pb=pb, **run_kw)
    return replay(run), run


def check_scheme(make, scheme, report=None, **kw):
    """Every step of `scheme` on one problem against the replay; the edges it has to reach."""
    out, run = run_case(make, scheme, **kw)
    assert out['reorders'] == 0
    # the dt sequence reaches both a refactorisation after the first step and, where the LHS allows it, a reuse of the LU
    assert any(out['refactors'][1:]), (scheme, out['refactors'])
    if scheme in RUNGE_KUTTA or scheme in ("CNAB1", "SBDF1", "CNAB2"):
        assert not all(out['refactors']), (scheme, "no step reused its LU", out['refactors'])
    if report is not None:
        report[out['kind']] = max(report.get(out['kind'], 0.0), out['worst'])
    return out


def check_reorder_keeps_history(make, report=None):
    """SBDF3 with the re-order forced at step 3, once the history is full: bset.reorders goes from 0 to 1 at that step, and the replay
    (history slots included) holds for that step and the next two."""
    out, run = run_case(make, "SBDF3", reorder_at=3)
    assert [st['reorders'] for st in run.steps] == [0, 0, 0, 1, 1, 1], [st['reorders'] for st in run.steps]
    assert len(run.steps[3]['factors']) == 2 and len(run.steps) >= 6          # the rejected factorisation and the new order's
    if report is not None:
        report[out['kind']] = max(report.get(out['kind'], 0.0), out['worst'])
    return out


def check_host_edit(make, field="u", at=3):
    """SBDF2 with u['g'] assigned between steps at-1 and at: step `at` starts from the edited state (uploaded by _sync_state_to_device),
    every other variable as the previous step left it, and the replay -- whose history comes from the steps before -- still holds.
    (Past iteration 1 the default cadence enforces no Hermitian symmetry, so the previous step's state arena is what it left.)"""
    def edit(run):
        f = run.pb[field]
        f['g'] = 0.5 * np.asarray(f['g'])
        return np.array(f['c'])
    out, run = run_case(make, "SBDF2", edit={at: edit})
    assert not run.steps[at - 1]['enforced']
    solver = run.solver
    iv = next(i for i, v in enumerate(solver.problem.variables) if v is run.pb[field])
    start, prev = run.steps[at]['evals'][0][1], run.steps[at - 1]['after']
    mask = np.zeros(start.size, dtype=bool)
    off = solver.var_arena.offsets[iv]
    size = solver.state_views[iv].numel()
    mask[off:off + size] = True
    assert start[mask].tobytes() == run.edited.reshape(-1).tobytes(), "the step did not start from the edited field"
    assert not np.array_equal(start[mask], prev[mask]), "the edit did not change the state"
    assert start[~mask].tobytes() == prev[~mask].tobytes(), "an unedited variable changed between the steps"
    return out


def check_hermitian_cadence(make, scheme="SBDF3", cadence=2):
    """enforce_real_cadence=2: the grid round trip runs after every step, inside the multistep history (also past the first
    `steps` iterations, where the default cadence would skip it); the replay reads the recorded states, so it still holds."""
    out, run = run_case(make, scheme, solver_kw=dict(enforce_real_cadence=cadence))
    assert [st['enforced'] for st in run.steps] == [1 if s % cadence < run.cls.steps else 0 for s in range(len(run.steps))]
    assert any(st['enforced'] for st in run.steps[run.cls.steps:])
    return out
