"""Symbolic operand tree for the IVP hot path (Cartesian Fourier^n x Jacobi problems).

Plays the role of the reference's core/field.py Operand API (40-342), core/arithmetic.py (Add, Multiply,
DotProduct) and core/operators.py (Differentiate, Gradient, Divergence, Laplacian, Trace, Interpolate,
Integrate, Lift, Convert, TimeDerivative).  Instead of one class per (operator, basis) pair with
`subproblem_matrix`, every linear node can emit *Kronecker terms*
        coef * comp (x) sym_axis0(k0) (x) ... (x) Z_last
whose separable-axis factors are polynomials in the wavenumber.  dedalus_b200/pencils.py turns those into
per-class matrix templates, so pencil matrices for all (kx, ky) are expanded on the device instead of being
assembled one pencil at a time on the host (reference subsystems.py:497-602).
"""
import numbers
import numpy as np
from scipy import sparse
from .basis import Jacobi, RealFourier, ComplexFourier


# --------------------------------------------------------------------------------------------------------
# helpers for separable-axis symbols: dict {power: small dense matrix}
# --------------------------------------------------------------------------------------------------------
def sym_mul(A, B):
    """(sum_m k^m A_m) @ (sum_n k^n B_n)."""
    out = {}
    for m, Am in A.items():
        for n, Bn in B.items():
            P = Am @ Bn
            if np.any(P != 0):
                out[m + n] = out.get(m + n, 0) + P
    return out


class Operand:
    """Base class with the arithmetic overloads of the reference Operand (field.py:40-200)."""
    __array_priority__ = 100.

    def __add__(self, other):
        return Add(self, other)
    __radd__ = __add__

    def __sub__(self, other):
        return Add(self, -1 * other if not isinstance(other, numbers.Number) else -other)

    def __rsub__(self, other):
        return Add(other, ScalarMul(-1, self))

    def __neg__(self):
        return ScalarMul(-1, self)

    def __mul__(self, other):
        if isinstance(other, numbers.Number):
            return ScalarMul(other, self)
        return Multiply(self, other)

    def __rmul__(self, other):
        if isinstance(other, numbers.Number):
            return ScalarMul(other, self)
        return Multiply(other, self)

    def __truediv__(self, other):
        if isinstance(other, numbers.Number):
            return ScalarMul(1 / other, self)
        raise NotImplementedError("Division by fields is not supported on the GPU hot path.")

    def __matmul__(self, other):
        return DotProduct(self, other)

    def __pow__(self, n):
        return Power(self, n)

    def __array_ufunc__(self, ufunc, method, *inputs, **kw):
        """numpy ufuncs on operands (reference field.py:60-88): unary ufuncs become grid functions, np.sqrt(u@u); the binary
        arithmetic ufuncs numpy dispatches for `np.float64(2) * field` go back to the Python overloads."""
        import operator
        if method != '__call__' or kw:
            return NotImplemented
        inputs = tuple(x.item() if isinstance(x, np.generic) else x for x in inputs)
        if len(inputs) == 1:
            if ufunc is np.negative:
                return -inputs[0]
            return UnaryGridFunction(ufunc, inputs[0])
        binary = {np.add: operator.add, np.subtract: operator.sub, np.multiply: operator.mul, np.true_divide: operator.truediv,
                  np.power: operator.pow, np.matmul: operator.matmul}
        if ufunc in binary and len(inputs) == 2:
            return binary[ufunc](*inputs)
        return NotImplemented

    def __call__(self, **positions):
        out = self
        for name, pos in positions.items():
            coord = self.dist.get_coord(name)
            out = Interpolate(out, coord, pos)
        return out

    # domain helpers ---------------------------------------------------------------------------------
    @property
    def ncomp(self):
        return int(np.prod([cs.dim for cs in self.tensorsig], dtype=int))

    @property
    def tshape(self):
        return tuple(cs.dim for cs in self.tensorsig)

    def atoms(self):
        out = []
        for a in getattr(self, 'args', ()):
            if isinstance(a, Operand):
                out.extend(a.atoms())
        return out

    def has(self, *fields):
        ids = {id(f) for f in fields}
        return any(id(a) in ids for a in self.atoms())

    def evaluate(self):
        """Evaluate the expression on the device into a new Field (reference future.py:149-206)."""
        from .evaluator import evaluate_expression
        return evaluate_expression(self)


def _merge_bases(op, bases_list):
    """Combine per-axis bases with '+' (Add) or '*' (products)."""
    out = []
    for per_axis in zip(*bases_list):
        cur = None
        for b in per_axis:
            if b is None:
                continue
            if cur is None:
                cur = b
            else:
                cur = (cur + b) if op == 'add' else (cur * b)
                if cur is NotImplemented:
                    raise ValueError("Incompatible bases in expression.")
        out.append(cur)
    return tuple(out)


class Future(Operand):
    def __getitem__(self, key):
        """op['g'] / op['c']: evaluate, then index the result (reference core/future.py Future / FutureField)."""
        return self.evaluate()[key]


class UnaryGridFunction(Future):
    """func(arg) pointwise on the dealiased grid (reference operators.py:505-640).  Evaluated by evaluator.ExpressionProgram;
    not available inside equations (the hot path's right-hand sides are polynomial)."""
    def __init__(self, func, arg):
        if not isinstance(arg, Operand):
            raise ValueError("UnaryGridFunction needs an operand argument.")
        self.func = func
        self.args = [arg]
        self.dist, self.dtype, self.tensorsig, self.bases = arg.dist, arg.dtype, arg.tensorsig, arg.bases


class Add(Future):
    def __init__(self, *args):
        flat = []
        for a in args:
            if isinstance(a, Add):
                flat.extend(a.args)
            elif isinstance(a, numbers.Number):
                if a != 0:
                    flat.append(a)
            else:
                flat.append(a)
        ops = [a for a in flat if isinstance(a, Operand)]
        if not ops:
            raise ValueError("Add needs at least one operand.")
        self.args = flat
        self.dist = ops[0].dist
        self.dtype = ops[0].dtype
        ts = ops[0].tensorsig
        for o in ops:
            if o.tensorsig != ts:
                raise ValueError("Cannot add operands with different tensor signatures.")
        self.tensorsig = ts
        self.bases = _merge_bases('add', [o.bases for o in ops])
        if any(isinstance(a, numbers.Number) for a in flat) and ts:
            raise ValueError("Cannot add a number to a tensor field.")


class ScalarMul(Future):
    def __init__(self, c, A):
        self.c = c
        self.args = [A]
        self.dist, self.dtype, self.tensorsig, self.bases = A.dist, A.dtype, A.tensorsig, A.bases


class Multiply(Future):
    """Tensor (outer) product of two fields (reference arithmetic.py:560-620, 800-866)."""
    def __init__(self, A, B):
        self.args = [A, B]
        self.dist, self.dtype = A.dist, A.dtype
        self.tensorsig = A.tensorsig + B.tensorsig
        self.bases = _merge_bases('mul', [A.bases, B.bases])


class DotProduct(Future):
    """Contract last index of A with first index of B (reference arithmetic.py:625-674)."""
    def __init__(self, A, B):
        if not A.tensorsig or not B.tensorsig:
            raise ValueError("Dot product requires tensor operands.")
        if A.tensorsig[-1] is not B.tensorsig[0]:
            raise ValueError("Dot product requires matching contracted coordinate systems.")
        self.args = [A, B]
        self.dist, self.dtype = A.dist, A.dtype
        self.tensorsig = A.tensorsig[:-1] + B.tensorsig[1:]
        self.bases = _merge_bases('mul', [A.bases, B.bases])


class Power(Future):
    def __init__(self, A, n):
        if A.tensorsig or not (isinstance(n, numbers.Integral) and n >= 1):
            raise NotImplementedError("Only positive integer powers of scalar fields are supported.")
        self.args = [A]
        self.n = int(n)
        self.dist, self.dtype, self.tensorsig = A.dist, A.dtype, ()
        self.bases = _merge_bases('mul', [A.bases] * max(self.n, 1)) if n > 1 else A.bases


class LinearOperator(Future):
    """Linear in its single operand."""
    @property
    def operand(self):
        return self.args[0]


class TimeDerivative(LinearOperator):
    def __init__(self, A):
        self.args = [A]
        self.dist, self.dtype, self.tensorsig, self.bases = A.dist, A.dtype, A.tensorsig, A.bases


def _diff_bases(bases, axis):
    b = bases[axis]
    out = list(bases)
    if b is not None:
        out[axis] = b.derivative_basis(1)
    return tuple(out)


class Differentiate(LinearOperator):
    def __init__(self, A, coord):
        if isinstance(A, numbers.Number):
            raise ValueError("Cannot differentiate a number.")
        self.args = [A]
        self.coord = coord
        self.axis = A.dist.get_axis(coord)
        self.dist, self.dtype, self.tensorsig = A.dist, A.dtype, A.tensorsig
        self.bases = _diff_bases(A.bases, self.axis)
        self.vanishes = A.bases[self.axis] is None


class Gradient(LinearOperator):
    """Cartesian gradient: new leading tensor index (reference operators.py:2340-2411)."""
    def __init__(self, A, cs=None):
        self.args = [A]
        self.cs = cs if cs is not None else A.dist.coordsys
        self.dist, self.dtype = A.dist, A.dtype
        self.tensorsig = (self.cs,) + A.tensorsig
        bases = A.bases
        for c in self.cs.coords:
            bases = _diff_bases(bases, A.dist.get_axis(c))
        self.bases = bases


class Divergence(LinearOperator):
    """Cartesian divergence contracting the first index (reference operators.py:3438-3495)."""
    def __init__(self, A, index=0):
        if not A.tensorsig:
            raise ValueError("Divergence requires a tensor operand.")
        if index != 0:
            raise NotImplementedError("Divergence is implemented for index=0.")
        self.args = [A]
        self.cs = A.tensorsig[0]
        self.dist, self.dtype = A.dist, A.dtype
        self.tensorsig = A.tensorsig[1:]
        bases = A.bases
        for c in self.cs.coords:
            bases = _diff_bases(bases, A.dist.get_axis(c))
        self.bases = bases


class Laplacian(LinearOperator):
    """Cartesian Laplacian = sum_i d_i d_i (reference operators.py:3700-3760)."""
    def __init__(self, A, cs=None):
        self.args = [A]
        self.cs = cs if cs is not None else A.dist.coordsys
        self.dist, self.dtype, self.tensorsig = A.dist, A.dtype, A.tensorsig
        bases = A.bases
        for c in self.cs.coords:
            ax = A.dist.get_axis(c)
            bases = _diff_bases(_diff_bases(bases, ax), ax)
        self.bases = bases


class Trace(LinearOperator):
    def __init__(self, A):
        if len(A.tensorsig) < 2 or A.tensorsig[0] is not A.tensorsig[1]:
            raise ValueError("Trace requires a tensor with two matching leading indices.")
        self.args = [A]
        self.dist, self.dtype, self.tensorsig, self.bases = A.dist, A.dtype, A.tensorsig[2:], A.bases


class TransposeComponents(LinearOperator):
    def __init__(self, A):
        if len(A.tensorsig) < 2:
            raise ValueError("TransposeComponents requires rank >= 2.")
        self.args = [A]
        ts = A.tensorsig
        self.dist, self.dtype, self.bases = A.dist, A.dtype, A.bases
        self.tensorsig = (ts[1], ts[0]) + ts[2:]


class Skew(LinearOperator):
    """90-degree positive rotation of a 2-D vector index (reference operators.py:2049-2160; on S2 the spin components are
    multiplied by -+1j, SpinSkew)."""
    def __init__(self, A, index=0):
        if not A.tensorsig:
            raise ValueError("Skew requires a tensor operand.")
        if A.tensorsig[index].dim != 2:
            raise ValueError("Skew is only defined for 2-D vector indices.")
        self.args = [A]
        self.index = index
        self.cs = A.tensorsig[index]
        self.dist, self.dtype, self.tensorsig, self.bases = A.dist, A.dtype, A.tensorsig, A.bases


class Curl(LinearOperator):
    """Curl of a 3-D Cartesian vector field (reference CartesianCurl, core/operators.py:3640-3720): (curl u)_i = eps_ijk d_j u_k."""
    def __init__(self, A, index=0):
        if not A.tensorsig or A.tensorsig[index].dim != 3 or getattr(A.tensorsig[index], 'curvilinear', False) or index != 0:
            raise NotImplementedError("Curl: first index of 3-D Cartesian vector fields")
        self.args = [A]
        self.index = index
        self.cs = A.tensorsig[index]
        self.dist, self.dtype, self.tensorsig = A.dist, A.dtype, A.tensorsig
        b = tuple(A.bases)
        for coord in self.cs.coords:
            b = _diff_bases(b, A.dist.get_axis(coord))
        self.bases = b


class MulCosine(LinearOperator):
    """Multiplication by cos(colatitude) on S2 (reference operators.py:2995-3050)."""
    def __init__(self, A, coordsys=None):
        self.args = [A]
        self.cs = coordsys if coordsys is not None else A.dist.coordsys
        if not getattr(self.cs, 'curvilinear', False):
            raise ValueError("MulCosine needs an S2 coordinate system.")
        self.dist, self.dtype, self.tensorsig, self.bases = A.dist, A.dtype, A.tensorsig, A.bases


class Interpolate(LinearOperator):
    def __init__(self, A, coord, position):
        self.args = [A]
        self.coord, self.position = coord, position
        self.axis = A.dist.get_axis(coord)
        self.dist, self.dtype, self.tensorsig = A.dist, A.dtype, A.tensorsig
        b = list(A.bases)
        self.trivial = b[self.axis] is None
        b[self.axis] = None
        self.bases = tuple(b)


class Integrate(LinearOperator):
    def __init__(self, A, coords=None, average=False):
        self.args = [A]
        if coords is None:
            coords = A.dist.coords
        elif hasattr(coords, 'coords') and not isinstance(coords, (tuple, list)):
            coords = coords.coords
        elif not isinstance(coords, (tuple, list)):
            coords = (coords,)
        self.coords = tuple(coords)
        self.average = average
        self.axes = tuple(A.dist.get_axis(c) for c in self.coords)
        self.dist, self.dtype, self.tensorsig = A.dist, A.dtype, A.tensorsig
        b = list(A.bases)
        for ax in self.axes:
            b[ax] = None
        self.bases = tuple(b)


class Lift(LinearOperator):
    """Tau lift: operand * P_n of `basis` (reference LiftJacobi basis.py:790-814; LiftShell basis.py:5155-5199: the operand
    lives on the sphere and is lifted along the radius of a shell basis)."""
    def __init__(self, A, basis, n):
        self.args = [A]
        self.basis, self.n = basis, n
        self.axis = A.dist.get_axis(basis.coord) + (basis.dim - 1)          # the last axis of a multi-dimensional (shell) basis
        if A.bases[self.axis] is not None:
            raise ValueError("Lift operand must be constant along the lift basis axis.")
        self.dist, self.dtype, self.tensorsig = A.dist, A.dtype, A.tensorsig
        b = list(A.bases)
        for sub in range(basis.dim):
            b[self.axis - (basis.dim - 1) + sub] = basis
        self.bases = tuple(b)


class Component(LinearOperator):
    """Selection along one tensor index over SphericalCoordinates (reference Component, core/operators.py:2190-2226): on a sphere
    basis the spin components (-, +, 0) of that index; radial = spin 0, angular = spins (-, +) (core/basis.py:5892-5970)."""
    def __init__(self, A, index=0):
        if not isinstance(A, Operand):
            raise ValueError("Component selection needs an operand.")
        rank = len(A.tensorsig)
        if index < 0:
            index += rank
        if not 0 <= index < rank:
            raise ValueError("index greater than rank")
        self.args = [A]
        self.index = index
        self.coordsys = A.tensorsig[index]
        if getattr(self.coordsys, 'S2coordsys', None) is None:
            raise NotImplementedError("radial / angular components of indices over SphericalCoordinates only")
        self.dist, self.dtype, self.bases = A.dist, A.dtype, A.bases


class RadialComponent(Component):
    def __init__(self, A, index=0):
        super().__init__(A, index)
        ts = A.tensorsig
        self.tensorsig = ts[:self.index] + ts[self.index + 1:]


class AngularComponent(Component):
    def __init__(self, A, index=0):
        super().__init__(A, index)
        ts = A.tensorsig
        self.tensorsig = ts[:self.index] + (self.coordsys.S2coordsys,) + ts[self.index + 1:]


class Convert(LinearOperator):
    """Convert(A, bases): per-axis tuple of output bases, or -- the reference's form (core/operators.py:1533-1560) -- ONE output
    basis, which replaces the operand's basis along that basis' axis."""
    def __init__(self, A, bases):
        self.args = [A]
        self.dist, self.dtype, self.tensorsig = A.dist, A.dtype, A.tensorsig
        if not isinstance(bases, (tuple, list)):
            out = list(A.bases)
            ax = A.dist.get_basis_axis(bases)
            for sub in range(getattr(bases, 'dim', 1)):
                out[ax + sub] = bases
            bases = out
        self.bases = tuple(bases)


# user-facing aliases (reference public.py / operators.py aliases)
def grad(A, cs=None): return Gradient(A, cs)
def div(A, index=0): return Divergence(A, index)
def lap(A, cs=None): return Laplacian(A, cs)
def skew(A, index=0): return Skew(A, index)
def curl(A, index=0): return Curl(A, index)
def trace(A): return Trace(A)
def transpose(A): return TransposeComponents(A)
def dt(A): return TimeDerivative(A)
def integ(A, coords=None): return Integrate(A, coords)
def ave(A, coords=None): return Integrate(A, coords, average=True)
def Average(A, coords=None): return Integrate(A, coords, average=True)
def dot(A, B): return DotProduct(A, B)
def interp(A, **positions): return A(**positions)
def radial(A, index=0): return RadialComponent(A, index)
def angular(A, index=0): return AngularComponent(A, index)


# --------------------------------------------------------------------------------------------------------
# Linear-map extraction:  expression  ->  {variable: [LinTerm, ...]}
# --------------------------------------------------------------------------------------------------------
class LinTerm:
    __slots__ = ("coef", "comp", "ops", "bases", "tder")

    def __init__(self, coef, comp, ops, bases, tder=0):
        self.coef, self.comp, self.ops, self.bases, self.tder = coef, comp, ops, tuple(bases), tder

    def copy(self):
        return LinTerm(self.coef, self.comp.copy(), [o.copy() if isinstance(o, dict) else o for o in self.ops], self.bases, self.tder)


def _axis_identity(basis, coupled):
    if coupled:
        n = basis.size if basis is not None else 1
        return sparse.identity(n, format='csr')
    if basis is None:
        return {0: np.eye(1)}
    return basis.sym_identity()


def _apply_axis(term, axis, coupled, kind, **kw):
    """Left-multiply the axis factor of `term` by a 1-D operator; returns None if the result vanishes."""
    basis = term.bases[axis]
    t = term.copy()
    bases = list(t.bases)
    if kind == 'diff':
        if basis is None:
            return None
        if coupled:
            t.ops[axis] = basis.derivative_matrix() @ t.ops[axis]
            bases[axis] = basis.derivative_basis(1)
        else:
            t.ops[axis] = sym_mul(basis.sym_derivative(), t.ops[axis])
    elif kind == 'convert':
        out = kw['out']
        if out == basis:
            return t
        if basis is None:
            if coupled:
                t.ops[axis] = out.embed_constant_vector() @ t.ops[axis]
            else:
                t.ops[axis] = sym_mul(out.sym_embed_constant(), t.ops[axis])
        elif isinstance(basis, Jacobi) and isinstance(out, Jacobi) and basis.grid_params == out.grid_params and basis.size == out.size:
            if not coupled:
                raise NotImplementedError("Jacobi bases are only supported on the last (coupled) axis.")
            t.ops[axis] = basis.conversion_matrix(out) @ t.ops[axis]
        else:
            raise NotImplementedError(f"Conversion {basis} -> {out} is not supported.")
        bases[axis] = out
    elif kind == 'interp':
        if basis is None:
            return t
        if not coupled:
            raise NotImplementedError("Interpolation along a separable (Fourier) axis is not supported on the hot path.")
        t.ops[axis] = basis.interpolation_vector(kw['position']) @ t.ops[axis]
        bases[axis] = None
    elif kind == 'integ':
        average = kw.get('average', False)
        if basis is None:
            if not average:
                raise NotImplementedError("Integrating a constant along an axis without basis needs a length; not supported.")
            return t
        if coupled:
            vec = basis.average_vector() if (average and hasattr(basis, 'average_vector')) else basis.integration_vector()
            if average and not hasattr(basis, 'average_vector'):
                vec = vec / basis.COV.problem_length
            t.ops[axis] = vec @ t.ops[axis]
        else:
            t.ops[axis] = sym_mul(basis.sym_average() if average else basis.sym_integrate(), t.ops[axis])
        bases[axis] = None
    elif kind == 'lift':
        lb, n = kw['basis'], kw['n']
        if not coupled:
            raise NotImplementedError("Lift is only supported along the last (coupled) axis.")
        if n < 0:
            n += lb.size
        col = sparse.csr_matrix(([1.0], ([n], [0])), shape=(lb.size, 1))
        t.ops[axis] = col @ t.ops[axis]
        bases[axis] = lb
    else:
        raise ValueError(kind)
    t.bases = tuple(bases)
    return t


def _convert_terms(terms, bases, coupled_axis):
    out = []
    for t in terms:
        for ax, b in enumerate(bases):
            if t is None:
                break
            if t.bases[ax] != b:
                t = _apply_axis(t, ax, ax == coupled_axis, 'convert', out=b)
        if t is not None:
            out.append(t)
    return out


def _comp_select(dim, i, nrest, row=True):
    """kron(e_i, I_nrest) as (dim*nrest x nrest) if row else its transpose."""
    e = sparse.csr_matrix(([1.0], ([i], [0])), shape=(dim, 1))
    K = sparse.kron(e, sparse.identity(nrest), format='csr')
    return K if row else K.T.tocsr()


def _const_values(field):
    """Tensor components of a constant (basis-free) field as a flat array."""
    if any(b is not None for b in field.bases):
        raise NotImplementedError("Non-constant coefficients (NCCs with bases) on the LHS are not supported yet.")
    data = np.asarray(field['c'])
    return data.reshape(field.ncomp)


def _product_selector(e, ncc, arg, ncc_left, vals):
    """Component matrix of  ncc * arg / ncc @ arg / arg * ncc / arg @ ncc  for constant tensor components `vals` of the coefficient."""
    nn, na = ncc.ncomp, arg.ncomp
    if isinstance(e, Multiply):
        col = sparse.csr_matrix(vals.reshape(nn, 1))
        K = sparse.kron(col, sparse.identity(na)) if ncc_left else sparse.kron(sparse.identity(na), col)
    elif ncc_left:       # ncc_(..., i) arg_(i, ...)
        d = ncc.tensorsig[-1].dim
        K = sparse.kron(sparse.csr_matrix(vals.reshape(nn // d, d)), sparse.identity(na // d))
    else:                # arg_(..., i) ncc_(i, ...)
        d = ncc.tensorsig[0].dim
        K = sparse.kron(sparse.identity(na // d), sparse.csr_matrix(vals.reshape(d, nn // d).T))
    return sparse.csr_matrix(K)


def _ncc_product(e, ncc, arg, ncc_left, sub, coupled_axis):
    """LHS product with a coefficient that varies along the coupled (Jacobi) axis only -- background profiles N^2(z), dzB(z).
    Reference: Jacobi.ncc_matrix via Clenshaw on the N x N Jacobi matrix J of the operand's basis (core/basis.py:560-628,
    tools/clenshaw.py:24-41), padded to Nmat = 3 ceil(N / 2) and truncated to N x N: f(J) = V diag(f(z_q)) V^T with the Gauss nodes
    z_q of that basis, i.e. the Nmat-point Gauss quadrature of <P_i, f P_j>, i, j < N; the product stays in the operand's basis
    (basis.py:546-557)."""
    from . import jacobi
    from .basis import Jacobi
    nb = ncc.bases[coupled_axis]
    if not isinstance(nb, Jacobi) or any(b is not None for ax, b in enumerate(ncc.bases) if ax != coupled_axis):
        raise NotImplementedError("Non-constant LHS coefficients may only vary along the coupled (last, Jacobi) axis.")
    coeffs = np.asarray(ncc['c']).reshape(max(ncc.ncomp, 1), -1)                     # (components, Nz) in the coefficient's own basis
    active = [c for c in range(coeffs.shape[0]) if np.abs(coeffs[c]).max() > 0]
    cache = {}

    def matrix(c, tb):
        key = (c, tb)
        if key not in cache:
            if tb is None:                                                          # operand constant along z: f itself, in f's basis
                cache[key] = (sparse.csr_matrix(coeffs[c][:, None]), nb)
            else:
                if not (isinstance(tb, Jacobi) and tb.grid_params == nb.grid_params):
                    raise NotImplementedError("coefficient and operand live on different axes / grids")
                N = tb.size
                Nmat = 3 * ((N + 1) // 2)                                            # the reference's padded size (basis.py:620-628)
                z, w = jacobi.gauss_grid(Nmat, tb.a, tb.b)
                P = jacobi.polynomials(N, tb.a, tb.b, z)                             # (N modes, Nmat nodes), orthonormal
                f = coeffs[c] @ jacobi.polynomials(nb.size, nb.a, nb.b, z)
                M = (P * (w * f)[None, :]) @ P.T
                M[np.abs(M) < 1e-14 * np.abs(M).max()] = 0
                cache[key] = (sparse.csr_matrix(M), tb)
        return cache[key]

    out = {}
    for k, terms in sub.items():
        new = []
        for c in active:
            unit = np.zeros(coeffs.shape[0]); unit[c] = 1.0
            K = _product_selector(e, ncc, arg, ncc_left, unit)
            for t in terms:
                u = t.copy()
                u.comp = sparse.csr_matrix(K @ u.comp)
                if u.comp.nnz == 0:
                    continue
                M, ob = matrix(c, u.bases[coupled_axis])
                u.ops[coupled_axis] = M @ u.ops[coupled_axis]
                bases = list(u.bases); bases[coupled_axis] = ob
                u.bases = tuple(bases)
                new.append(u)
        # up to the expression's bases where that is a conversion upwards; terms already above them stay (the parent sum converts)
        conv = []
        for u in new:
            tb, eb = u.bases[coupled_axis], e.bases[coupled_axis]
            if isinstance(tb, Jacobi) and isinstance(eb, Jacobi) and (eb.a < tb.a or eb.b < tb.b):
                conv.append(u)
            else:
                conv.extend(_convert_terms([u], e.bases, coupled_axis))
        out[k] = conv
    return out


def linear_map(expr, variables, coupled_axis):
    """Return {var: [LinTerm]} for an expression that is linear in `variables` (all terms in expr.bases)."""
    varids = {id(v): v for v in variables}
    dist = expr.dist if isinstance(expr, Operand) else None

    def rec(e):
        from .field import Field
        if isinstance(e, Field):
            if id(e) not in varids:
                raise ValueError(f"LHS contains field '{e.name}' that is not a problem variable (only constant NCC factors are allowed).")
            ops = [_axis_identity(b, ax == coupled_axis) for ax, b in enumerate(e.bases)]
            return {id(e): [LinTerm(1.0, sparse.identity(e.ncomp, format='csr'), ops, e.bases)]}
        if isinstance(e, Add):
            out = {}
            for a in e.args:
                if isinstance(a, numbers.Number):
                    raise ValueError("LHS must be linear and homogeneous in the variables (found a number).")
                for k, terms in rec(a).items():
                    out.setdefault(k, []).extend(_convert_terms(terms, e.bases, coupled_axis))
            return out
        if isinstance(e, ScalarMul):
            out = rec(e.args[0])
            for terms in out.values():
                for t in terms:
                    t.coef = t.coef * e.c
            return out
        if isinstance(e, (Multiply, DotProduct)):
            A, B = e.args
            a_var, b_var = A.has(*variables), B.has(*variables)
            if a_var and b_var:
                raise ValueError("LHS must be linear in the problem variables.")
            if not a_var and not b_var:
                raise ValueError("LHS term does not involve any problem variable.")
            ncc, arg, ncc_left = (A, B, True) if b_var else (B, A, False)
            from .field import Field as _F
            if not isinstance(ncc, _F):
                raise NotImplementedError("Only plain fields are supported as LHS coefficients.")
            if any(b is not None for b in ncc.bases):
                return _ncc_product(e, ncc, arg, ncc_left, rec(arg), coupled_axis)
            vals = _const_values(ncc)
            sub = rec(arg)
            nn, na = ncc.ncomp, arg.ncomp
            if isinstance(e, Multiply):
                col = sparse.csr_matrix(vals.reshape(nn, 1))
                K = sparse.kron(col, sparse.identity(na)) if ncc_left else sparse.kron(sparse.identity(na), col)
            else:
                if ncc_left:     # ncc_(..., i) arg_(i, ...)
                    d = ncc.tensorsig[-1].dim
                    W = vals.reshape(nn // d, d)
                    K = sparse.kron(sparse.csr_matrix(W), sparse.identity(na // d))
                else:            # arg_(..., i) ncc_(i, ...)
                    d = ncc.tensorsig[0].dim
                    W = vals.reshape(d, nn // d)
                    K = sparse.kron(sparse.identity(na // d), sparse.csr_matrix(W.T))
            K = sparse.csr_matrix(K)
            for k, terms in sub.items():
                new = []
                for t in terms:
                    t.comp = sparse.csr_matrix(K @ t.comp)
                    new.append(t)
                sub[k] = _convert_terms(new, e.bases, coupled_axis)
            return sub
        if isinstance(e, TimeDerivative):
            out = rec(e.args[0])
            for terms in out.values():
                for t in terms:
                    t.tder += 1
            return out
        if isinstance(e, Differentiate):
            out = rec(e.args[0])
            for k in out:
                out[k] = [u for u in (_apply_axis(t, e.axis, e.axis == coupled_axis, 'diff') for t in out[k]) if u is not None]
            return out
        if isinstance(e, Gradient):
            sub = rec(e.args[0])
            out = {}
            nin = e.args[0].ncomp
            for k, terms in sub.items():
                new = []
                for i, c in enumerate(e.cs.coords):
                    ax = e.dist.get_axis(c)
                    sel = _comp_select(e.cs.dim, i, nin, row=True)
                    for t in terms:
                        u = _apply_axis(t, ax, ax == coupled_axis, 'diff')
                        if u is not None:
                            u.comp = sparse.csr_matrix(sel @ u.comp)
                            new.append(u)
                out[k] = _convert_terms(new, e.bases, coupled_axis)
            return out
        if isinstance(e, Divergence):
            sub = rec(e.args[0])
            out = {}
            nrest = e.ncomp
            for k, terms in sub.items():
                new = []
                for i, c in enumerate(e.cs.coords):
                    ax = e.dist.get_axis(c)
                    sel = _comp_select(e.cs.dim, i, nrest, row=False)
                    for t in terms:
                        u = t.copy()
                        u.comp = sparse.csr_matrix(sel @ u.comp)
                        if u.comp.nnz == 0:
                            continue
                        u = _apply_axis(u, ax, ax == coupled_axis, 'diff')
                        if u is not None:
                            new.append(u)
                out[k] = _convert_terms(new, e.bases, coupled_axis)
            return out
        if isinstance(e, Laplacian):
            sub = rec(e.args[0])
            out = {}
            for k, terms in sub.items():
                new = []
                for c in e.cs.coords:
                    ax = e.dist.get_axis(c)
                    for t in terms:
                        u = _apply_axis(t, ax, ax == coupled_axis, 'diff')
                        if u is not None:
                            u = _apply_axis(u, ax, ax == coupled_axis, 'diff')
                        if u is not None:
                            new.append(u)
                out[k] = _convert_terms(new, e.bases, coupled_axis)
            return out
        if isinstance(e, Trace):
            sub = rec(e.args[0])
            d = e.args[0].tensorsig[0].dim
            nrest = e.ncomp
            rows, cols = [], []
            for i in range(d):
                for r in range(nrest):
                    rows.append(r); cols.append((i * d + i) * nrest + r)
            T = sparse.csr_matrix((np.ones(len(rows)), (rows, cols)), shape=(nrest, d * d * nrest))
            for k, terms in sub.items():
                for t in terms:
                    t.comp = sparse.csr_matrix(T @ t.comp)
                sub[k] = [t for t in terms if t.comp.nnz]
            return sub
        if isinstance(e, Curl):
            sub = rec(e.args[0])
            nrest = e.ncomp // 3
            out = {}
            for k, terms in sub.items():
                new = []
                for i in range(3):
                    for j, kk, sign in (((i + 1) % 3, (i + 2) % 3, 1.0), ((i + 2) % 3, (i + 1) % 3, -1.0)):      # eps_ijk d_j u_k
                        ax = e.dist.get_axis(e.cs.coords[j])
                        pick = _comp_select(3, kk, nrest, row=False)           # component kk of the operand
                        place = _comp_select(3, i, nrest, row=True)            # into component i of the result
                        for t in terms:
                            u = t.copy()
                            u.comp = sparse.csr_matrix(place @ (pick @ u.comp)) * sign
                            if u.comp.nnz == 0:
                                continue
                            u = _apply_axis(u, ax, ax == coupled_axis, 'diff')
                            if u is not None:
                                new.append(u)
                out[k] = _convert_terms(new, e.bases, coupled_axis)
            return out
        if isinstance(e, Skew):
            # Cartesian skew of the first index: kron([[0, -1], [1, 0]], I) on the components (reference CartesianSkew.subproblem_matrix,
            # core/operators.py:2102-2110)
            if e.index != 0 or getattr(e.cs, 'curvilinear', False):
                raise NotImplementedError("Skew on the LHS: Cartesian vectors, index 0")
            sub = rec(e.args[0])
            nrest = e.ncomp // 2
            S = sparse.kron(sparse.csr_matrix(np.array([[0.0, -1.0], [1.0, 0.0]])), sparse.identity(nrest), format='csr')
            for k, terms in sub.items():
                for t in terms:
                    t.comp = sparse.csr_matrix(S @ t.comp)
            return sub
        if isinstance(e, TransposeComponents):
            sub = rec(e.args[0])
            d0, d1 = e.args[0].tensorsig[0].dim, e.args[0].tensorsig[1].dim
            nrest = e.ncomp // (d0 * d1)
            idx = np.arange(d0 * d1 * nrest).reshape(d0, d1, nrest).transpose(1, 0, 2).ravel()
            P = sparse.csr_matrix((np.ones(idx.size), (np.arange(idx.size), idx)), shape=(idx.size, idx.size))
            for k, terms in sub.items():
                for t in terms:
                    t.comp = sparse.csr_matrix(P @ t.comp)
            return sub
        if isinstance(e, Interpolate):
            out = rec(e.args[0])
            for k in out:
                out[k] = [_apply_axis(t, e.axis, e.axis == coupled_axis, 'interp', position=e.position) for t in out[k]]
            return out
        if isinstance(e, Integrate):
            out = rec(e.args[0])
            for k in out:
                terms = out[k]
                for ax in e.axes:
                    terms = [_apply_axis(t, ax, ax == coupled_axis, 'integ', average=e.average) for t in terms]
                out[k] = terms
            return out
        if isinstance(e, Lift):
            out = rec(e.args[0])
            for k in out:
                out[k] = [_apply_axis(t, e.axis, e.axis == coupled_axis, 'lift', basis=e.basis, n=e.n) for t in out[k]]
            return out
        if isinstance(e, Convert):
            out = rec(e.args[0])
            for k in out:
                out[k] = _convert_terms(out[k], e.bases, coupled_axis)
            return out
        raise NotImplementedError(f"Operator {type(e).__name__} is not supported on the LHS.")

    res = rec(expr)
    return {varids[k]: v for k, v in res.items()}
