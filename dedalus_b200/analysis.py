"""Stand-alone evaluation of output expressions on curvilinear domains (sphere, spherical shell): the analysis tasks and flow
properties of the stock scripts -- `b(r=(Ri+Ro)/2)`, `flux(r=Ro)`, `flux(phi=0)` with `flux = er @ (-kappa*grad(b) + u*b)`,
`np.sqrt(u@u)/nu` (examples/ivp_shell_convection/shell_convection.py:82-109) -- evaluated when a handler fires, not inside a step.

Reference: Future.evaluate (core/future.py:149-206) walking the tree with the layout rules of each node:
  * products, powers and grid functions act on the dealiased grid values of their operands (arithmetic.py:560-580, 666-674,
    855-866; operators.py:505-640), with lower-dimensional operands (the radial unit vector) broadcast;
  * sums that contain such a term meet their operands on the grid: the conversions the reference inserts between different
    radial bases (arithmetic.py:94-98) are plain copies in grid space (operators.py:1628-1638), so nothing is truncated;
  * linear operators act on coefficients: shell gradient (dedalus_b200/shell_ivp.py ShellGradient), the separable sphere
    operators (dedalus_b200/sphere.py evaluate_linear_expression), radial interpolation of scalars and tensors
    (ShellRadialInterpolate, core/basis.py:5823-5889), radial / angular components as slices (core/basis.py:5892-5970);
  * azimuthal interpolation acts on grid values and returns a field locked to the grid (InterpolateAzimuth, basis.py:5578-5635).
Transforms are the library's own kernels (field layout changes); the elementwise arithmetic between whole grids is done with
torch tensor expressions on the device -- cadence-scheduled output, never part of the time step."""
import numpy as np
from . import operators as ops
from .field import Field

_TORCH_NAMES = {'absolute': 'abs', 'arcsin': 'asin', 'arccos': 'acos', 'arctan': 'atan', 'arcsinh': 'asinh', 'arccosh': 'acosh',
                'arctanh': 'atanh', 'conjugate': 'conj'}
_NONLINEAR = (ops.Multiply, ops.DotProduct, ops.Power, ops.UnaryGridFunction, ops.MulCosine)


class LockedField:
    """Result of an azimuthal interpolation: grid data only (reference LockedField, core/field.py:1046-1075)."""

    def __init__(self, tensor, scales, tensorsig):
        self._dev, self.scales, self.tensorsig, self.layout = tensor, tuple(scales), tensorsig, 'g'

    def change_scales(self, scales):
        if isinstance(scales, (int, float)):
            scales = (scales,) * len(self.scales)
        if tuple(scales) != self.scales:
            raise ValueError("Cannot change the scales of a field locked to the grid.")

    def change_layout(self, layout):
        if layout not in ('g', 'grid'):
            raise ValueError("Cannot change locked axis to coeff space.")

    def device_data(self):
        return self._dev

    @property
    def data(self):
        return self._dev.detach().cpu().numpy()

    def __getitem__(self, key):
        layout = key[0] if isinstance(key, tuple) else key
        if isinstance(key, tuple):
            self.change_scales(key[1])
        self.change_layout(layout)
        return self.data


def _const(x):
    return all(b is None for b in x.bases)


def _full_basis(e):
    from .sphere import sphere_basis_of
    from .shell import shell_basis_of
    return shell_basis_of(e) or sphere_basis_of(e)


def _temp_field(e, bases):
    f = Field(e.dist, bases=bases, tensorsig=e.tensorsig, dtype=e.dtype)
    e.dist._fields.pop()
    return f


class CurvilinearEvaluation:
    def __init__(self, dist):
        self.dist = dist

    # ---- grid side ---------------------------------------------------------------------------------------------------
    def grid(self, e):
        """Coordinate components of e on the dealiased grid: tensor of shape tshape + grid (size-1 axes where e is constant)."""
        import torch
        if not isinstance(e, ops.Operand):
            return float(e)
        if isinstance(e, Field):
            return e.copy_device_to_grid()
        if isinstance(e, ops.ScalarMul):
            return e.c * self.grid(e.args[0])
        if isinstance(e, ops.Add):
            total = None
            for a in e.args:
                g = self.grid(a)
                total = g if total is None else total + g
            return total
        if isinstance(e, ops.Multiply):
            A, B = e.args
            ga, gb = self.grid(A), self.grid(B)
            if torch.is_tensor(ga) and torch.is_tensor(gb):       # tensor product: A's indices first
                ra, rb = len(A.tensorsig), len(B.tensorsig)
                ga = ga.reshape(tuple(ga.shape[:ra]) + (1,) * rb + tuple(ga.shape[ra:]))
                gb = gb.reshape((1,) * ra + tuple(gb.shape))
            return ga * gb
        if isinstance(e, ops.DotProduct):
            A, B = e.args
            ga, gb = self.grid(A), self.grid(B)
            ra, rb = len(A.tensorsig), len(B.tensorsig)
            ga = ga.reshape(tuple(ga.shape[:ra]) + (1,) * (rb - 1) + tuple(ga.shape[ra:]))
            gb = gb.reshape((1,) * (ra - 1) + tuple(gb.shape))
            return (ga * gb).sum(dim=ra - 1)
        if isinstance(e, ops.Power):
            return self.grid(e.args[0]) ** e.n
        if isinstance(e, ops.UnaryGridFunction):
            name = getattr(e.func, '__name__', str(e.func))
            fn = getattr(torch, _TORCH_NAMES.get(name, name), None)
            if fn is None:
                raise NotImplementedError(f"grid function {name!r} has no device implementation")
            return fn(self.grid(e.args[0]))
        if isinstance(e, ops.MulCosine):
            # cos(colatitude) times the operand, formed on the dealiased grid (the product raises the degree by one and the forward
            # transform truncates it, as the reference's truncated operator matrix does, core/operators.py:2995-3050)
            g = self.grid(e.args[0])
            basis = _full_basis(e.args[0])
            ax = self.dist.get_basis_axis(basis)
            scale = basis.dealias[1]
            sb = getattr(basis, 'sphere_basis', basis)
            theta = sb.global_grid_colatitude(scale)[self.dist.grid_local_slice(ax + 1, basis, scale)]
            shape = [1] * self.dist.dim; shape[ax + 1] = theta.size
            return g * torch.from_numpy(np.cos(theta).reshape(shape)).to(g.device)
        if isinstance(e, ops.Interpolate) and self._azimuthal(e):
            g = self.grid(e.args[0])
            basis = _full_basis(e.args[0])
            nt = len(e.tensorsig)
            w = torch.from_numpy(self._azimuth_weights(basis, g.shape[nt], e.position)).to(g.device)
            shape = [1] * g.dim(); shape[nt] = -1
            return (g * w.reshape(shape)).sum(dim=nt, keepdim=True)
        return self.field(e).copy_device_to_grid()

    def _azimuthal(self, e):
        basis = _full_basis(e.args[0])
        return basis is not None and e.axis == self.dist.get_basis_axis(basis)

    @staticmethod
    def _azimuth_weights(basis, Ng, position):
        """Interpolation to azimuth `position` from Ng equispaced grid values of a function band-limited to |m| < Nphi / 2:
        interpolation row of the real Fourier basis times its forward transform matrix (reference basis.py:5615-5624)."""
        K = basis.shape[0] // 2 - 1
        phi_j = 2 * np.pi * np.arange(Ng) / Ng
        w = np.ones(Ng)
        for k in range(1, K + 1):
            w += 2 * np.cos(k * (position - phi_j))
        return w / Ng

    # ---- coefficient side --------------------------------------------------------------------------------------------
    def field(self, e):
        """e as a Field (coefficient data available through the usual layout changes)."""
        from .sphere import sphere_basis_of, evaluate_linear_expression
        from .shell import shell_basis_of
        if isinstance(e, Field):
            return e
        if isinstance(e, ops.Convert):
            return self.field(e.args[0])
        nonlinear_top = isinstance(e, _NONLINEAR) or (isinstance(e, (ops.Add, ops.ScalarMul)) and self._has_nonlinear(e))
        if nonlinear_top:
            return self._materialize(e, self.grid(e))
        if isinstance(e, ops.Component):
            return self._component(self.field(e.args[0]), e)
        shell = shell_basis_of(e.args[0]) if getattr(e, 'args', None) else None
        if isinstance(e, ops.Interpolate) and self._azimuthal(e):
            raise NotImplementedError("azimuthal interpolation returns grid data only; use it as the outermost operator of a task")
        if shell is not None:
            if isinstance(e, ops.Gradient) and shell.k == 0 and isinstance(e.args[0], Field):
                return self._shell_gradient(self.field(e.args[0]), e)          # the kernel path (also used inside time steps)
            if isinstance(e, ops.Interpolate) and e.axis == self.dist.get_basis_axis(shell) + 2:
                return self._shell_radial_interpolation(self.field(e.args[0]), e)
            if isinstance(e, (ops.Gradient, ops.Divergence, ops.Laplacian, ops.Trace, ops.TransposeComponents, ops.Add, ops.ScalarMul)):
                return self._shell_linear(e)
            raise NotImplementedError(f"{type(e).__name__} of shell fields in output expressions")
        if isinstance(e, ops.Integrate) and sphere_basis_of(e.args[0]) is not None and shell is None:
            return self._sphere_integral(self.field(e.args[0]), e)
        if sphere_basis_of(e) is not None:
            return evaluate_linear_expression(self._with_field_leaves(e))
        raise NotImplementedError(f"{type(e).__name__} in curvilinear output expressions")

    def _has_nonlinear(self, e):
        if isinstance(e, _NONLINEAR):
            return True
        if isinstance(e, ops.Interpolate) and self._azimuthal(e):
            return True
        return any(self._has_nonlinear(a) for a in getattr(e, 'args', []) if isinstance(a, ops.Operand))

    def _with_field_leaves(self, e):
        """Replace the nonlinear subtrees of a separable-operator expression by fields."""
        import copy
        if isinstance(e, Field) or not isinstance(e, ops.Operand):
            return e
        if isinstance(e, _NONLINEAR):
            return self.field(e)
        new = copy.copy(e)
        new.args = [self._with_field_leaves(a) for a in e.args]
        return new

    def _materialize(self, e, g, basis=None):
        """Grid values (dealias scales) -> a temporary field on e's bases (or on `basis`: the same grid, another radial basis k)."""
        basis = basis if basis is not None else _full_basis(e)
        if basis is None or any(b is None for b in e.bases):
            raise NotImplementedError("lower-dimensional results of grid expressions")
        f = _temp_field(e, (basis,))
        ax = self.dist.get_basis_axis(basis)
        scales = tuple(basis.dealias)
        full = f.tshape + tuple(self.dist.grid_local_slice(ax + i, basis, scales[i]).stop - self.dist.grid_local_slice(ax + i, basis, scales[i]).start
                                for i in range(basis.dim))
        f.set_device_data(g.expand(full).contiguous(), 'g', scales=self.dist.remedy_scales(scales))
        return f

    def _shell_gradient(self, f, e):
        from .shell import shell_basis_of
        from .shell_ivp import ShellGradient, RadialOps
        basis = shell_basis_of(f)
        if any(b is not None and b is not basis for b in f.bases):
            raise NotImplementedError("gradients of fields that are not on the full shell basis")
        rops = RadialOps(basis.shape[2], basis.radii, basis.alpha)
        f.change_layout('c')
        dev = f.device_data()
        rank = len(f.tensorsig)
        prog = ShellGradient.cached(basis, rops, rank, self.dist, dev.device)
        c = dev.reshape((3 ** rank,) + tuple(dev.shape[rank:])).contiguous()
        out = prog.apply(c)
        res = _temp_field(e, (basis.derivative_basis(1),))
        res.set_device_data(out.reshape(res.tshape + tuple(out.shape[1:])), 'c')
        return res

    def _shell_radial_interpolation(self, f, e):
        """Field at radius r0: sum_n c[a, m, l, n] (dR / r0)^k P_n^(alpha + k)(z(r0)) for every regularity component a, then --
        tensors -- the regularity -> spin recombination Q(l) of the shell chain, which leaves the spin components a field on the
        sphere holds (reference basis.py:5823-5889)."""
        import torch
        from .shell import shell_basis_of
        from .shell_ivp import RadialOps
        basis = shell_basis_of(f)
        rank = len(f.tensorsig)
        rops = RadialOps(basis.shape[2], basis.radii, basis.alpha)
        f.change_layout('c')
        c = f.device_data()
        vec = torch.from_numpy(np.ascontiguousarray(rops.basis_functions(basis.k, e.position)[0])).to(c.device)
        out = (c * vec).sum(dim=-1, keepdim=True).contiguous()
        if rank:
            Nc0, Nc1 = out.shape[rank:rank + 2]
            spin = torch.empty_like(out)
            basis.regularity_table(rank, False, c.device, self.dist).apply(out, spin, Nc0 // 2, Nc1, sym_div=1)
            out = spin
        res = _temp_field(e, (basis.S2_basis(radius=e.position),))
        res.set_device_data(out, 'c', scales=self.dist.remedy_scales(tuple(basis.dealias)))      # reference: outputs at the dealias scales
        return res

    def _component(self, f, e):
        """Radial / angular component of a field on a sphere: a slice along the selected tensor axis of its data in either layout
        -- index 2 (spin 0, or the r coordinate) and indices 0:2 (spins -, +, or the phi, theta coordinates) -- on the device
        (reference S2RadialComponent / S2AngularComponent.operate, core/basis.py:5920-5970)."""
        from .sphere import sphere_basis_of
        from .shell import shell_basis_of
        basis = sphere_basis_of(f)
        if basis is None or shell_basis_of(f) is not None:
            raise NotImplementedError("radial / angular components of fields on a sphere (interpolate shell fields first)")
        d = f.device_data()
        d = d.select(e.index, 2) if isinstance(e, ops.RadialComponent) else d.narrow(e.index, 0, 2)
        res = _temp_field(e, (basis,))
        res.set_device_data(d.contiguous(), f.layout, scales=f.scales)
        return res

    def _shell_linear(self, e):
        """Any expression of gradients / divergences / Laplacians / traces / sums of shell fields: for every degree l, the radial
        block matrices of the per-l lowering that also builds the pencil systems (shell_ivp.ShellLowering: reference
        SphericalEllOperator subproblem matrices, core/operators.py:3108-3310, 3546-3603) applied to the (m, l) lines of the
        operands' regularity components.  Nonlinear subtrees are evaluated first and enter as fields."""
        import torch
        from types import SimpleNamespace
        from .shell import shell_basis_of
        from .shell_ivp import ShellLowering, regularity_allowed
        e = self._with_field_leaves(e)
        leaves = []
        for f in e.atoms():
            if not any(f is g for g in leaves):
                leaves.append(f)
        if any(shell_basis_of(f) is None or any(b is not shell_basis_of(f) for b in f.bases) for f in leaves):
            raise NotImplementedError("linear shell expressions: operands on the full shell basis only")
        low = ShellLowering(SimpleNamespace(variables=leaves))
        basis, sb = low.basis, low.basis.sphere_basis
        kind, k_out = low.kind_of(e)
        if kind != 'shell':
            raise NotImplementedError("linear shell expressions with lower-dimensional results")
        rank_out = len(e.tensorsig)
        j0, j1 = sb.local_pairs(self.dist)
        _, ell_map = sb.elements_to_groups()
        ell_pairs = ell_map[0::2][j0:j1]                                   # (local pairs, Nl): degree of every (pair, column)
        data = []
        for f in leaves:
            f.change_layout('c')
            d = f.device_data()
            data.append(d.reshape((3 ** len(f.tensorsig),) + tuple(d.shape[len(f.tshape):])))
        dev = data[0].device
        Nc0, Nc1, Nr = data[0].shape[1:]
        out = torch.zeros((3 ** rank_out, Nc0, Nc1, Nr), dtype=torch.float64, device=dev)
        idx_of = lambda c, rank: tuple(np.unravel_index(c, (3,) * rank)) if rank else ()
        for ell in range(sb.Lmax + 1):
            pj, pc = np.nonzero(ell_pairs == ell)
            if pj.size == 0:
                continue
            rows = torch.from_numpy(np.concatenate([2 * pj, 2 * pj + 1])).to(dev)
            cols = torch.from_numpy(np.concatenate([pc, pc])).to(dev)
            node = low.lower(e, ell)
            for (co, iv, ci), B in node.blocks.get(0, {}).items():
                if not (regularity_allowed(ell, idx_of(co, rank_out)) and regularity_allowed(ell, idx_of(ci, len(leaves[iv].tensorsig)))):
                    continue
                Bm = torch.from_numpy(np.ascontiguousarray(B.toarray() if hasattr(B, 'toarray') else np.asarray(B))).to(dev)
                out[co, rows, cols, :] += data[iv][ci, rows, cols, :] @ Bm.T
        res = _temp_field(e, (basis.clone_with(k=k_out),))
        res.set_device_data(out.reshape(res.tshape + (Nc0, Nc1, Nr)), 'c')
        return res

    def _sphere_integral(self, f, e):
        """Average / integral of a scalar over the sphere: the (m = 0, l = 0) coefficient times the constant mode value 1 / sqrt 2
        (reference SphereAverage, core/basis.py:5296-5317; the integral is the average times 4 pi R^2)."""
        import torch
        from .sphere import sphere_basis_of
        if f.tensorsig:
            raise NotImplementedError("sphere averages of tensor fields")
        basis = sphere_basis_of(f)
        f.change_layout('c')
        c = f.device_data()
        j, cols = basis.mode_columns(0)
        j0, j1 = basis.local_pairs(self.dist)
        val = torch.zeros(1, dtype=c.dtype, device=c.device)
        if j0 <= j < j1:
            val = c.reshape(c.shape[0], c.shape[1], -1)[2 * (j - j0), int(cols[0]), :1].clone() / np.sqrt(2.0)
        if self.dist.size > 1:
            import torch.distributed as td
            td.all_reduce(val)
        if not e.average:
            val = val * (4 * np.pi * basis.radius ** 2)
        res = _temp_field(e, ())
        res.set_device_data(val.reshape(res.local_shape('c', res.scales)), 'c')
        return res

    # ---- entry -------------------------------------------------------------------------------------------------------
    def evaluate(self, e):
        if isinstance(e, ops.Interpolate) and self._azimuthal(e):
            basis = _full_basis(e.args[0])
            return LockedField(self.grid(e), self.dist.remedy_scales(tuple(basis.dealias)), e.tensorsig)
        return self.field(e)


def evaluate_curvilinear(expr):
    return CurvilinearEvaluation(expr.dist).evaluate(expr)


def is_shell_boundary(eq):
    """An equation of a shell problem that lives on a sphere: angular bases, none along the radius."""
    return eq['bases'][-1] is None and eq['bases'][0] is not None


class BoundaryData:
    """Field right-hand side of an equation on a sphere of a shell problem (boundary data such as `angular(u(r=Ri)) = uw`,
    `b(r=Ro) = bt`; reference: F evaluated with the other right-hand sides every stage, core/problems.py:84-100).  Each write
    reads the expression's fields afresh, so data the user changes between steps takes effect.  The equation rows hold the spin
    components of the sphere's coefficient packing, which is what a sphere field holds in coefficient space: a plain field is
    copied as it is, any other expression (products, grid functions) is formed on the grid and transformed once."""

    def __init__(self, solver, ie, rhs, evaluation):
        from .shell import shell_basis_of
        from .sphere import sphere_basis_of
        eq = solver.problem.equations[ie]
        ts = eq['tensorsig']
        if len({type(cs) for cs in ts}) > 1 and not isinstance(rhs, Field):
            raise NotImplementedError("grid expressions as data of equations with mixed spherical / S2 indices")
        basis = sphere_basis_of(rhs)
        shell = shell_basis_of(eq['LHS'])
        if basis is None or any(b is not None and b is not basis for b in rhs.bases) or basis.shape != shell.shape[:2]:
            raise NotImplementedError("boundary data must live on a sphere of the shell's angular resolution")
        self.solver, self.rhs, self.eval, self.basis = solver, rhs, evaluation, basis
        self.off = solver.eq_arena.offsets[ie]
        tsh, shp = solver.eq_arena.shapes[ie]
        self.shape = (max(int(np.prod(tsh, dtype=int)), 1),) + tuple(shp)
        self.rank = len(ts)
        self.spins = [int(s) for s in basis.spin_weights(ts).reshape(-1)] or [0]
        self.cs = type(ts[0]) if ts else None

    def write(self, eq_t):
        from .sphere import grid_to_components
        from .coords import S2Coordinates
        n = int(np.prod(self.shape))
        dst = eq_t[self.off:self.off + n].view(self.shape)
        if isinstance(self.rhs, Field):
            self.rhs.change_layout('c')
            dst.copy_(self.rhs.device_data().reshape(self.shape))
            return
        g = self.eval.grid(self.rhs)
        sl = [self.solver.dist.grid_local_slice(ax, self.basis, self.basis.dealias[ax]) for ax in range(2)]
        full = (self.shape[0], sl[0].stop - sl[0].start, sl[1].stop - sl[1].start)
        tsh = tuple(g.shape[:self.rank])
        g = g.reshape(tsh + tuple(g.shape[self.rank:self.rank + 2])).expand(tsh + full[1:]).reshape(full).contiguous()
        c = grid_to_components(self.basis, g, self.spins, self.rank, cs=self.cs or S2Coordinates, dist=self.solver.dist)
        dst.copy_(c.reshape(self.shape))


class GenericCurvilinearRHS:
    """Right-hand sides of sphere / shell problems that the fused plans (sphere.SphereRHSPlan, shell_ivp.ShellRHSPlan) do not cover --
    grid functions, forcings, fields that are not problem variables, products with radial profiles, operators applied to products:
    every equation's F is evaluated with the expression evaluator above (one field per equation), converted to the equation's
    radial basis (shell: E^dk along r, reference ConvertShell, core/basis.py:3868-3872) and copied into the equation arena.  Same
    interface as the fused plans; slower (one transform chain per node), used only when they decline an equation."""

    def __init__(self, solver):
        from .shell import shell_basis_of
        self.solver = solver
        self.dist = solver.dist
        self.eval = CurvilinearEvaluation(solver.dist)
        self.entries = []                 # (equation index, expression, conversion matrix on the device or None)
        self.boundary = []                # BoundaryData of the equations on a sphere of a shell
        self.static = []
        problem = solver.problem
        for ie, eq in enumerate(problem.equations):
            rhs = eq['RHS']
            if not isinstance(rhs, ops.Operand):
                if rhs != 0:
                    self._constant(ie, eq, float(rhs))
                continue
            if any(b is None for b in eq['bases']):
                if not (solver.shell and is_shell_boundary(eq)):
                    raise NotImplementedError("field right-hand sides of lower-dimensional equations on curvilinear domains")
                self.boundary.append(BoundaryData(solver, ie, rhs, self.eval))
                continue
            self.entries.append([ie, rhs, None, shell_basis_of(eq['LHS'])])

    def _constant(self, ie, eq, value):
        from .sphere import sphere_basis_of
        from .shell import shell_basis_of
        if eq['tensorsig']:
            raise NotImplementedError("nonzero constant right-hand side of a tensor equation")
        off = self.solver.eq_arena.offsets[ie]
        shell, sphere = shell_basis_of(eq['LHS']), sphere_basis_of(eq['LHS'])
        basis = shell.sphere_basis if shell is not None else sphere
        if basis is not None and basis.local_pairs(self.dist)[0] != 0:
            return
        from .shell import ShellBasis
        if all(b is None for b in eq['bases']):
            self.static.append((off, value))
        elif not isinstance(eq['bases'][-1], ShellBasis) or len(eq['bases']) == 2:
            self.static.append((off, value * np.sqrt(2)))                # a field on a sphere: the l = 0 mode, 1 / constant_mode_value
        else:
            raise NotImplementedError("nonzero constant right-hand side of a shell-interior equation")

    def set_static(self, eq_t):
        eq_t.zero_()
        for off, val in self.static:
            eq_t[off] = val

    def evaluate(self, eq_t):
        import torch
        from .sphere import sphere_basis_of
        arena = self.solver.eq_arena
        for bd in self.boundary:
            bd.write(eq_t)
        for ie, rhs, _, eq_shell in self.entries:
            # F on the dealiased grid, then ONE forward transform in the equation's own basis: the reference converts F to the
            # equation's bases while it is on the grid (a copy), so no intermediate truncation in the expression's basis happens
            g = self.eval.grid(rhs)
            eq = self.solver.problem.equations[ie]
            basis = eq_shell if eq_shell is not None else sphere_basis_of(eq['LHS'])
            if not torch.is_tensor(g):
                raise NotImplementedError("numeric right-hand side expressions")
            F = self.eval._materialize(rhs, g, basis=basis)
            F.change_layout('c')
            c = F.device_data().contiguous()
            eq_t[arena.offsets[ie]:arena.offsets[ie] + c.numel()].view(c.shape).copy_(c)
