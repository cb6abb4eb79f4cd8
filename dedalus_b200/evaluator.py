"""Right-hand-side evaluation plan (D3 + P1 + the transform chain of T1/T2).

Reference: Evaluator.evaluate_handlers (core/evaluator.py:95-146) walks every field of every F expression up
and down the layout chain, one transform call per field per axis and one numpy call per operator node
(probe: 18 backward + 4 forward scalar 3-D transforms per RB3D stage, SURVEY.md section 8a row D3).
Here each equation's RHS is lowered ONCE at build time to
        F_out = sum_terms coef * prod_factors  d^alpha(field component)
and evaluated as three fused phases on the device:
  1. backward transforms of the unique grid inputs, sharing partial transforms along a prefix tree
     (z-stage results are reused by every x/y derivative of the same field; derivatives are applied inside the
     transform kernels' load stage, not as separate coefficient-space passes),
  2. one pointwise kernel for all products of all equations (csrc/pointwise.cu),
  3. forward transforms of the outputs; the last (coupled-axis) pass applies the conversion to the equation's
     basis and writes straight into the equation arena that the pencil gather reads.
"""
import numbers
import numpy as np
from . import operators as ops
from .operators import Operand
from .field import Field
from .basis import RealFourier, ComplexFourier, Jacobi


class NonPolynomialError(NotImplementedError):
    pass


def lower(expr):
    """Lower an expression to {flat component index: [(coef, ((field, comp, derivs), ...)), ...]}."""
    dim = expr.dist.dim if isinstance(expr, Operand) else 0

    def rec(e):
        if isinstance(e, numbers.Number):
            return {0: [(e, ())]} if e != 0 else {0: []}
        if isinstance(e, Field):
            out = {}
            if all(b is None for b in e.bases):
                vals = np.asarray(e['c']).reshape(-1)
                for c in range(e.ncomp):
                    out[c] = [(vals[c], ())] if vals[c] != 0 else []
                return out
            for c in range(e.ncomp):
                out[c] = [(1.0, ((e, c, (0,) * dim),))]
            return out
        if isinstance(e, ops.Add):
            out = {}
            for a in e.args:
                for c, terms in rec(a).items():
                    out.setdefault(c, []).extend(terms)
            return out
        if isinstance(e, ops.ScalarMul):
            return {c: [(coef * e.c, f) for coef, f in terms] for c, terms in rec(e.args[0]).items()}
        if isinstance(e, ops.Convert):
            return rec(e.args[0])
        if isinstance(e, ops.Multiply):
            A, B = e.args
            ra, rb = rec(A), rec(B)
            nb = B.ncomp
            out = {}
            for ca, ta in ra.items():
                for cb, tb in rb.items():
                    out[ca * nb + cb] = [(x * y, fx + fy) for x, fx in ta for y, fy in tb]
            return out
        if isinstance(e, ops.DotProduct):
            A, B = e.args
            ra, rb = rec(A), rec(B)
            d = A.tensorsig[-1].dim
            na, nb = A.ncomp // d, B.ncomp // d
            out = {}
            for ia in range(na):
                for ib in range(nb):
                    terms = []
                    for i in range(d):
                        for x, fx in ra.get(ia * d + i, []):
                            for y, fy in rb.get(i * nb + ib, []):
                                terms.append((x * y, fx + fy))
                    out[ia * nb + ib] = terms
            return out
        if isinstance(e, ops.Power):
            base = rec(e.args[0])[0]
            cur = base
            for _ in range(e.n - 1):
                cur = [(x * y, fx + fy) for x, fx in cur for y, fy in base]
            return {0: cur}

        def diff_terms(terms, axis):
            new = []
            for coef, facs in terms:
                if len(facs) != 1:
                    raise NonPolynomialError(
                        "Differentiating a product on the RHS is not supported: expand it or introduce an auxiliary field.")
                f, c, dv = facs[0]
                if f.bases[axis] is None:
                    continue
                dv = list(dv); dv[axis] += 1
                new.append((coef, ((f, c, tuple(dv)),)))
            return new

        if isinstance(e, ops.Differentiate):
            return {c: diff_terms(t, e.axis) for c, t in rec(e.args[0]).items()}
        if isinstance(e, ops.Gradient):
            sub = rec(e.args[0]); nin = e.args[0].ncomp
            out = {}
            for i, coord in enumerate(e.cs.coords):
                ax = e.dist.get_axis(coord)
                for c, t in sub.items():
                    out[i * nin + c] = diff_terms(t, ax)
            return out
        if isinstance(e, ops.Divergence):
            sub = rec(e.args[0]); nrest = e.ncomp
            out = {r: [] for r in range(nrest)}
            for i, coord in enumerate(e.cs.coords):
                ax = e.dist.get_axis(coord)
                for r in range(nrest):
                    out[r].extend(diff_terms(sub.get(i * nrest + r, []), ax))
            return out
        if isinstance(e, ops.Laplacian):
            sub = rec(e.args[0])
            out = {c: [] for c in sub}
            for coord in e.cs.coords:
                ax = e.dist.get_axis(coord)
                for c, t in sub.items():
                    out[c].extend(diff_terms(diff_terms(t, ax), ax))
            return out
        if isinstance(e, ops.Trace):
            sub = rec(e.args[0]); d = e.args[0].tensorsig[0].dim; nrest = e.ncomp
            return {r: [t for i in range(d) for t in sub.get((i * d + i) * nrest + r, [])] for r in range(nrest)}
        if isinstance(e, ops.Curl):
            sub = rec(e.args[0]); nrest = e.ncomp // 3
            out = {}
            for i in range(3):
                j, k = (i + 1) % 3, (i + 2) % 3                      # (curl u)_i = d_j u_k - d_k u_j
                axj, axk = e.dist.get_axis(e.cs.coords[j]), e.dist.get_axis(e.cs.coords[k])
                for r in range(nrest):
                    out[i * nrest + r] = diff_terms(sub.get(k * nrest + r, []), axj) + \
                        [(-c, f) for c, f in diff_terms(sub.get(j * nrest + r, []), axk)]
            return out
        if isinstance(e, ops.Skew):
            # Cartesian skew (reference CartesianSkew.operate, operators.py:2112-2122): out_x = -arg_y, out_y = arg_x
            if e.index != 0 or getattr(e.cs, 'curvilinear', False):
                raise NonPolynomialError("Skew: Cartesian vectors, index 0 only")
            sub = rec(e.args[0]); nrest = e.ncomp // 2
            out = {}
            for r in range(nrest):
                out[r] = [(-c, f) for c, f in sub.get(nrest + r, [])]
                out[nrest + r] = list(sub.get(r, []))
            return out
        if isinstance(e, ops.TransposeComponents):
            sub = rec(e.args[0]); d0, d1 = e.args[0].tensorsig[0].dim, e.args[0].tensorsig[1].dim
            nrest = e.ncomp // (d0 * d1)
            return {(j * d0 + i) * nrest + r: sub.get((i * d1 + j) * nrest + r, []) for i in range(d0) for j in range(d1) for r in range(nrest)}
        raise NonPolynomialError(f"{type(e).__name__} is not supported on the right-hand side of the GPU hot path.")

    return rec(expr)


class RHSPlan:
    """Compiled evaluation of all equation right-hand sides into the equation arena."""

    def __init__(self, solver):
        import torch
        self.solver = solver
        problem = solver.problem
        dist = problem.dist
        self.dist = dist
        dim = dist.dim
        self.device = solver.device
        arena = solver.eq_arena
        self.static_entries = []      # (arena offset, value) for constant RHS
        self.linear_copies = {}       # (equation, comp) -> [(coef, field, field comp)]: coefficient-space right-hand sides
        self.program_copies = {}      # equation -> ExpressionProgram of a lower-dimensional right-hand side
        inputs = {}                   # (id(field), comp, derivs) -> index
        self.input_keys = []
        outputs = []                  # (eq index, comp, terms)
        for ie, eq in enumerate(problem.equations):
            rhs = eq['RHS']
            if isinstance(rhs, numbers.Number):
                if rhs != 0:
                    self._add_constant(ie, eq, float(rhs))
                continue
            try:
                low = lower(rhs)
            except NonPolynomialError:
                if any(b is None for b in eq['bases']):
                    # boundary data given as an expression ("u(z=0) = f(z=0)"): evaluated stand-alone (reductions of fields), copied in
                    self.program_copies[ie] = ExpressionProgram(rhs)
                    continue
                raise
            for comp, terms in low.items():
                const = sum(c for c, f in terms if len(f) == 0)
                terms = [(c, f) for c, f in terms if len(f) > 0]
                if const != 0:
                    self._add_constant(ie, eq, float(const), comp)
                if not terms:
                    continue
                if any(b is None for b in eq['bases']):
                    # lower-dimensional equation (boundary conditions with data, "b(z=0) = g"): terms linear in fields that live on
                    # exactly the equation's bases are copied in coefficient space -- no transforms (reference: the F expression of
                    # such an equation is the field itself, core/problems.py:84-100)
                    for coef, facs in terms:
                        ok = len(facs) == 1 and not any(facs[0][2]) and all(
                            (fb is None and eb is None) or (fb is not None and eb is not None and fb == eb)
                            for fb, eb in zip(facs[0][0].bases, eq['bases']))
                        if not ok:
                            raise NotImplementedError("Right-hand sides of lower-dimensional equations must be linear in fields on the equation's bases.")
                        self.linear_copies.setdefault((ie, comp), []).append((float(coef), facs[0][0], facs[0][1]))
                    continue
                tl = []
                for coef, facs in terms:
                    idxs = []
                    for (f, c, dv) in facs:
                        if any(b is None for b in f.bases) and (any(dv) or dist.size > 1):
                            raise NotImplementedError("RHS factors without bases along some axis (background profiles, forcings) are broadcast "
                                                      "on the grid on one GPU and cannot be differentiated: precompute the derivative field.")
                        key = (id(f), c, dv)
                        if key not in inputs:
                            inputs[key] = len(self.input_keys)
                            self.input_keys.append((f, c, dv))
                        idxs.append(inputs[key])
                    tl.append((coef, idxs))
                outputs.append((ie, comp, tl))
        self.outputs = outputs
        self.n_in, self.n_out = len(self.input_keys), len(outputs)
        self.copy_dest = {}
        for (ie, comp) in self.linear_copies:
            tsh, shp = arena.shapes[ie]
            self.copy_dest[(ie, comp)] = (arena.offsets[ie] + comp * int(np.prod(shp)), shp)
        if self.n_out == 0:
            return
        # ---- bases / shapes (all inputs share the variable bases up to Jacobi parameters)
        f0 = self.input_keys[0][0]
        self.bases = f0.bases
        self.dealias = tuple(b.dealias[0] for b in self.bases)
        self.cshape = tuple(dist.coeff_local_slice(ax, b).stop - dist.coeff_local_slice(ax, b).start for ax, b in enumerate(self.bases))
        self.gshape_full = tuple(b.grid_size(s) for b, s in zip(self.bases, self.dealias))
        self.P = dist.size
        if self.P > 1:
            from .transposes import check_divisible, get_planner
            if dim < 2:
                raise NotImplementedError("1-D problems cannot be distributed.")
            check_divisible(dist, self.bases, self.dealias)
            self.planner = get_planner(dist)
            # full grid layout: axis 1 distributed (after the single transpose hop)
            self.gshape = (self.gshape_full[0], self.gshape_full[1] // self.P) + tuple(self.gshape_full[2:])
        else:
            self.gshape = self.gshape_full
        self.npoints = int(np.prod(self.gshape))
        # ---- pointwise program
        term_ptr, coef, fac_ptr, fac = [0], [], [0], []
        for ie, comp, tl in outputs:
            for c, idxs in tl:
                coef.append(c); fac.extend(idxs); fac_ptr.append(len(fac))
            term_ptr.append(len(coef))
        dev = self.device
        self.term_ptr = torch.tensor(term_ptr, dtype=torch.int32, device=dev)
        self.coef = torch.tensor(coef, dtype=torch.float64, device=dev)
        self.fac_ptr = torch.tensor(fac_ptr, dtype=torch.int32, device=dev)
        self.fac = torch.tensor(fac, dtype=torch.int32, device=dev)
        self.nfac = len(fac)
        # quadratic programs (every term a product of one or two inputs) take the packed-record kernel
        self.pairs = None
        nf = np.diff(fac_ptr)
        if len(coef) and nf.min() >= 1 and nf.max() <= 2 and self.npoints % 2 == 0 and 2 * self.n_in * 128 * 16 <= 227 * 1024:
            rec = np.zeros(len(coef), dtype=np.dtype([('coef', '<f8'), ('a', '<i4'), ('b', '<i4')]))      # db_pair_term
            rec['coef'] = coef
            rec['a'] = [fac[fac_ptr[t]] for t in range(len(coef))]
            rec['b'] = [fac[fac_ptr[t] + 1] if nf[t] == 2 else -1 for t in range(len(coef))]
            self.pairs = torch.from_numpy(np.frombuffer(rec.tobytes(), dtype=np.uint8).copy()).to(dev)
        # ---- backward prefix tree: level order = axes from last to first
        self.axes_order = list(range(dim - 1, -1, -1))
        self._build_tree()
        # ---- grid buffers of the separate passes (allocated on first use: the fused x pass does not need them)
        self._grid_in = self._grid_out = None
        # ---- fused x pass (backward x transforms + products + forward x transforms in one kernel), or None
        self.xprod = self._build_x_products()
        self.use_x_products = self.xprod is not None
        # ---- output destinations in the equation arena and forward plans
        self.out_dest = []
        for ie, comp, tl in outputs:
            eq = problem.equations[ie]
            tsh, shp = arena.shapes[ie]
            off = arena.offsets[ie] + comp * int(np.prod(shp))
            self.out_dest.append((off, shp, eq['bases']))

    @property
    def grid_in(self):
        if self._grid_in is None:
            import torch
            self._grid_in = torch.empty((self.n_in,) + self.gshape, dtype=torch.float64, device=self.device)
        return self._grid_in

    @property
    def grid_out(self):
        if self._grid_out is None:
            import torch
            self._grid_out = torch.empty((self.n_out,) + self.gshape, dtype=torch.float64, device=self.device)
        return self._grid_out

    def _build_x_products(self):
        """Schedule of the fused x pass (csrc/rfft_regs.cu k_rfft_x_products), or None where the separate passes stay.

        The x axis is the last backward and the first forward pass, so a tile of 16 adjacent lines holds everything the products
        need once its lines are transformed along x: the inputs' level-(dim-2) coefficient arrays are read once and the outputs'
        x coefficients written once, with no grid array in global memory.  Inputs that appear in more than one term (the velocity
        components of u.grad(u), u.grad(b)) are held on chip for the whole tile; every other input is transformed right before
        its one term.  DB_RHS_FUSED=0 keeps the separate passes (for A/B timing)."""
        import os, torch
        from collections import Counter
        from .transforms import cached_plan, RealFourierTransform
        dim = self.dist.dim
        if os.environ.get("DB_RHS_FUSED", "1") == "0":
            return None
        if self.P != 1 or dim < 2 or self.grid_leaves or self.broadcast_leaves or self.pairs is None:
            return None
        px = cached_plan(self.bases[0], self.dealias[0])
        if not isinstance(px, RealFourierTransform):
            return None
        final, parents = self.levels[dim - 1], self.levels[dim - 2]
        src, deriv = [], []
        for key in self.leaf_of_input:
            nd = final[key]
            p = cached_plan(nd['field'].bases[0], self.dealias[0])
            if not isinstance(p, RealFourierTransform) or (p.N, p.M, p.kscale) != (px.N, px.M, px.kscale):
                return None
            src.append(parents[nd['parent']]['index']); deriv.append(nd['deriv'])
        terms = [(o, coef, idxs) for o, (ie, comp, tl) in enumerate(self.outputs) for coef, idxs in tl]
        count = Counter(i for _, _, idxs in terms for i in idxs)
        held = {}
        for _, _, idxs in terms:
            for i in idxs:
                if count[i] > 1 and i not in held:
                    held[i] = len(held)
            if len(idxs) == 2 and all(count[i] == 1 for i in idxs):
                held[idxs[0]] = len(held)             # a product of two single-use inputs: hold the first, stream the second
        inner = int(np.prod(self.gshape[1:], dtype=np.int64))
        if not px.x_products_supported(inner, len(held)):
            return None
        rec = []                                      # db_xprod_item: coef, src, deriv, a, b, out, flags
        for i, slot in held.items():
            rec.append((0.0, src[i], deriv[i], slot, -1, -1, 1))                                   # DB_XPROD_HELD
        for k, (o, coef, idxs) in enumerate(terms):
            streamed = [i for i in idxs if i not in held]
            code = [held.get(i, 3) for i in idxs] + [-1]                                          # 3: the streamed input
            last = k + 1 == len(terms) or terms[k + 1][0] != o
            rec.append((coef, src[streamed[0]] if streamed else -1, deriv[streamed[0]] if streamed else 0,
                        code[0], code[1], o, 2 if last else 0))                                    # DB_XPROD_LAST
        items = np.array(rec, dtype=np.dtype([('coef', '<f8'), ('src', '<i4'), ('deriv', '<i4'), ('a', '<i4'), ('b', '<i4'),
                                              ('out', '<i4'), ('flags', '<i4')]))
        loads = items['src'][items['src'] >= 0]
        if len(loads) == 0:
            return None
        return dict(plan=px, inner=inner, n_held=len(held), n_items=len(items),
                    items=torch.from_numpy(np.frombuffer(items.tobytes(), dtype=np.uint8).copy()).to(self.device),
                    loads=torch.from_numpy(loads.astype(np.int32)).to(self.device))

    def _x_products(self, cin):
        """Fused x pass from the level-(dim-2) stack into the x-forward scratch that the next forward pass reads."""
        from .solvers import Timed
        xp = self.xprod
        px, inner = xp['plan'], xp['inner']
        out = self._scratch(('fwd', 0), (self.n_out, px.M) + tuple(self.gshape[1:]))
        with Timed(self.solver.prof, "rhs_x_products", 8 * (self.n_in + self.n_out) * px.M * inner):
            px.x_products(cin, out, inner, xp['items'], xp['n_items'], xp['loads'], xp['n_held'])
        return out

    # ------------------------------------------------------------------------------------------------
    def _add_constant(self, ie, eq, value, comp=0):
        """Constant RHS: coefficient of the constant mode of the equation's domain (group (0,..,0), cos slot)."""
        arena = self.solver.eq_arena
        tsh, shp = arena.shapes[ie]
        factor = 1.0
        for ax, b in enumerate(eq['bases']):
            if b is None:
                continue
            sl = self.dist.coeff_local_slice(ax, b)
            if sl.start != 0:
                return            # mode 0 lives on another rank
            if isinstance(b, Jacobi):
                factor /= b.constant_mode_value
        off = arena.offsets[ie] + comp * int(np.prod(shp))
        self.static_entries.append((off, value * factor))

    def _build_tree(self):
        """nodes[level] = list of dicts(parent, field, comp, deriv) ; leaves map to grid-input slots."""
        from .transforms import cached_plan
        dim = self.dist.dim
        levels = [dict() for _ in range(dim)]
        self.leaf_of_input = []
        self.grid_leaves = []        # (input slot, field, comp): grid-function results enter the products without a coefficient round trip
        self.broadcast_leaves = []   # (input slot, field, comp): factors without bases along some axis
        for slot, (f, c, dv) in enumerate(self.input_keys):
            if getattr(f, '_grid_leaf', False) and not any(dv):
                self.leaf_of_input.append(('gridleaf', id(f), c))
                self.grid_leaves.append((slot, f, c))
                continue
            if any(b is None for b in f.bases):
                # a factor that is constant along some axis (a background profile b0(z), a forcing f(x)): its own low-dimensional
                # transform, then broadcast into the product's input slot (reference: numpy broadcasting in MultiplyFields.operate)
                self.leaf_of_input.append(('broadcast', id(f), c))
                self.broadcast_leaves.append((slot, f, c))
                continue
            parent = None
            for lvl, ax in enumerate(self.axes_order):
                key = (id(f), c) + tuple(dv[a] for a in self.axes_order[:lvl + 1])
                if key not in levels[lvl]:
                    levels[lvl][key] = dict(parent=parent, field=f, comp=c, axis=ax, deriv=dv[ax], index=len(levels[lvl]))
                parent = key
            self.leaf_of_input.append(parent)
        self.levels = levels
        # shapes after each level (before the transpose hop axis 1 is still complete and axis 0 block-local)
        shp = list(self.cshape)
        self.level_shapes = []
        for lvl, ax in enumerate(self.axes_order):
            shp[ax] = self.gshape_full[ax]
            self.level_shapes.append(tuple(shp))

    def set_static(self, arena_tensor):
        for off, val in self.static_entries:
            arena_tensor[off] = val

    # ------------------------------------------------------------------------------------------------
    def evaluate(self, eq_arena_tensor, grid_only=False):
        """Evaluate all RHS outputs into eq_arena_tensor (state fields must be in coefficient space on device).
        grid_only: stop after the products and return the (n_out, grid) values on the dealiased grid."""
        import torch, ctypes as C
        from .transforms import cached_plan, _dptr, _stream
        from .lib import get_lib
        from .solvers import Timed
        for ie, prog in self.program_copies.items():
            res = prog.run()
            res.change_layout('c')
            tsh, shp = self.solver.eq_arena.shapes[ie]
            n = int(np.prod(tsh, dtype=int)) * int(np.prod(shp, dtype=int))
            off = self.solver.eq_arena.offsets[ie]
            eq_arena_tensor[off:off + n].copy_(res.device_data().reshape(-1))
        for key, terms in self.linear_copies.items():
            off, shp = self.copy_dest[key]
            dst = eq_arena_tensor[off:off + int(np.prod(shp))].view(shp)
            for i, (coef, f, c) in enumerate(terms):
                if f.layout != 'c':
                    f.change_layout('c')
                src = f.device_data()[self._comp_index(f, c)].reshape(shp)
                if i == 0:
                    torch.mul(src, coef, out=dst)
                else:
                    dst.add_(src, alpha=coef)
        if self.n_out == 0:
            return
        dim = self.dist.dim
        dev = self.device
        last = dim - 1
        # ---- phase 1: backward transforms along the prefix tree
        for slot, f, c in self.grid_leaves:
            if f.layout != 'g' or tuple(f.scales) != tuple(self.dealias):
                raise RuntimeError("grid-function result is not on the dealiased grid")
            self.grid_in[slot].copy_(f.device_data()[self._comp_index(f, c)])
        if self.broadcast_leaves:
            grids = {}
            for slot, f, c in self.broadcast_leaves:
                if id(f) not in grids:
                    grids[id(f)] = f.copy_device_to_grid()
                self.grid_in[slot].copy_(grids[id(f)][self._comp_index(f, c)].expand(self.gshape))
        in_tree = {id(nd['field']): nd['field'] for nd in self.levels[0].values()}
        for f in in_tree.values():
            if f.layout != 'c':
                f.change_layout('c')          # non-state fields (forcings, NCCs) may have been set on the grid
        fused = self.use_x_products and not grid_only
        bufs = [None] * dim
        for lvl, ax in enumerate(self.axes_order if in_tree else []):
            nodes = self.levels[lvl]
            final = (lvl == dim - 1)
            if final and fused:
                break
            prev = bufs[lvl - 1] if lvl > 0 else None
            if self.P > 1 and dim >= 3 and lvl == dim - 2 and self._blocked_bwd_ok():
                # the y pass writes the all-to-all send buffer directly and the x pass reads the receive buffer directly
                self._backward_blocked_levels(prev, lvl)
                break
            if not final:
                bufs[lvl] = self._scratch(('bwd', lvl), (len(nodes),) + self.level_shapes[lvl])
            if final and self.P > 1:
                # transpose hop (axis 0 <-> axis 1) for the whole stack of level-(dim-2) arrays in ONE all-to-all
                nn = prev.shape[0]
                n1loc, n2 = prev.shape[1], prev.shape[2]
                n3 = int(np.prod(prev.shape[3:], dtype=int))
                tshape = (nn, n1loc * self.P, n2 // self.P) + tuple(prev.shape[3:])
                tr = self._scratch(('tr_bwd',), tshape)
                with Timed(self.solver.prof, "transpose_bwd", 8 * 2 * prev.numel()):
                    self.planner.localize_columns(prev.view(nn, n1loc, n2, n3), tr.view(nn, n1loc * self.P, n2 // self.P, n3))
                prev = tr
            for key, nd in nodes.items():
                f = nd['field']
                basis = f.bases[ax]
                plan = cached_plan(basis, self.dealias[ax])
                if lvl == 0:
                    src = f.device_data()[self._comp_index(f, nd['comp'])]
                else:
                    src = prev[self.levels[lvl - 1][nd['parent']]['index']]
                if final:
                    dst = self.grid_in[self._input_slot(key)]
                else:
                    dst = bufs[lvl][nd['index']]
                with Timed(self.solver.prof, f"transform_bwd_axis{ax}", 8 * (src.numel() + dst.numel())):
                    plan.backward(src, dst, ax, deriv=nd['deriv'])
        if fused:
            # ---- phases 2 and the x pass of phase 3 in one kernel
            cur = self._x_products(bufs[dim - 2])
        else:
            cur = self._products()
        if grid_only:
            return cur
        # ---- phase 3: forward transforms (axes first -> last), all outputs stacked
        blocked_fwd = self.P > 1 and dim >= 3 and self._blocked_fwd_ok()
        for ax in range(1 if fused else 0, dim):
            basis = self.bases[ax]
            if blocked_fwd and ax == 0:
                cur = self._forward_blocked_xy(cur)
                continue
            if blocked_fwd and ax == 1:
                continue
            if ax < last:
                plan = cached_plan(basis, self.dealias[ax])
                shp = list(cur.shape); shp[1 + ax] = plan.M
                out = self._scratch(('fwd', ax), tuple(shp))
                with Timed(self.solver.prof, f"transform_fwd_axis{ax}", 8 * (cur.numel() + out.numel())):
                    plan.forward(cur, out, 1 + ax)
                cur = out
                if ax == 0 and self.P > 1:
                    nn, n1, n2loc = cur.shape[0], cur.shape[1], cur.shape[2]
                    n3 = int(np.prod(cur.shape[3:], dtype=int))
                    tshape = (nn, n1 // self.P, n2loc * self.P) + tuple(cur.shape[3:])
                    tr = self._scratch(('tr_fwd',), tshape)
                    with Timed(self.solver.prof, "transpose_fwd", 8 * 2 * cur.numel()):
                        self.planner.localize_rows(cur.view(nn, n1, n2loc, n3), tr.view(nn, n1 // self.P, n2loc * self.P, n3))
                    cur = tr
            else:
                for o, (off, shp, eq_bases) in enumerate(self.out_dest):
                    eqb = eq_bases[ax]
                    if isinstance(basis, Jacobi):
                        prod_basis = basis.clone_with(a=basis.a0, b=basis.b0)
                        tb = eqb if eqb is not None else prod_basis
                        plan = self._fwd_plan_last(prod_basis, tb)
                    else:
                        plan = cached_plan(basis, self.dealias[ax])
                    n = int(np.prod(shp))
                    dst = eq_arena_tensor[off:off + n].view(shp)
                    with Timed(self.solver.prof, f"transform_fwd_axis{ax}", 8 * (cur[o].numel() + dst.numel())):
                        plan.forward(cur[o], dst, ax)

    def _products(self):
        """Phase 2 of the separate passes: products of the backward-transformed inputs on the grid into grid_out."""
        from .transforms import _dptr, _stream
        from .lib import get_lib
        from .solvers import Timed
        with Timed(self.solver.prof, "pointwise", 8 * self.npoints * (self.n_in + self.n_out)):
          if self.pairs is not None and self.grid_in.data_ptr() % 16 == 0 and self.grid_out.data_ptr() % 16 == 0:
              get_lib().call("db_pointwise_pairs", _dptr(self.grid_in), _dptr(self.grid_out), self.npoints, self.n_in, self.n_out,
                             _dptr(self.term_ptr), _dptr(self.pairs), _stream())
          else:
              get_lib().call("db_pointwise", _dptr(self.grid_in), _dptr(self.grid_out), self.npoints, self.n_in, self.n_out,
                             _dptr(self.term_ptr), _dptr(self.coef), _dptr(self.fac_ptr), _dptr(self.fac), self.nfac, _stream())
        return self.grid_out

    def _fwd_plan_last(self, prod_basis, target_basis):
        from .transforms import FastChebyshevTransform, cached_plan
        key = ('fwdlast', target_basis)
        if not hasattr(self, '_plans'):
            self._plans = {}
        if key not in self._plans:
            N = prod_basis.grid_size(self.dealias[-1])
            if prod_basis.a0 == prod_basis.b0 == -0.5:
                self._plans[key] = FastChebyshevTransform(N, prod_basis.size, target_basis.a, target_basis.b, -0.5, -0.5,
                                                          stretch=prod_basis.COV.stretch)
            else:
                from .transforms import JacobiMatrixTransform
                self._plans[key] = JacobiMatrixTransform(N, prod_basis.size, target_basis.a, target_basis.b, prod_basis.a0, prod_basis.b0)
        return self._plans[key]

    # ---- distributed path without pack / unpack kernels (X1): blocked row addressing in the real-Fourier kernels
    def _xy_plans(self):
        from .transforms import cached_plan, RealFourierTransform
        px, py = cached_plan(self.bases[0], self.dealias[0]), cached_plan(self.bases[1], self.dealias[1])
        if not (isinstance(px, RealFourierTransform) and isinstance(py, RealFourierTransform)):
            return None
        return px, py

    def _blocked_bwd_ok(self):
        if not hasattr(self, '_blk_bwd'):
            ok = False
            plans = self._xy_plans()
            if plans is not None:
                px, py = plans
                n1loc, n2, n3 = self.level_shapes[self.dist.dim - 2][0], self.gshape_full[1], int(np.prod(self.gshape_full[2:], dtype=int))
                n2loc = n2 // self.P
                ok = (py.blocked_supported(n3) and px.blocked_supported(n2loc * n3) and (n1loc * n2loc * n3) % 2 == 0
                      and px.M == n1loc * self.P)
            self._blk_bwd = ok
        return self._blk_bwd

    def _blocked_fwd_ok(self):
        if not hasattr(self, '_blk_fwd'):
            ok = False
            plans = self._xy_plans()
            if plans is not None:
                px, py = plans
                n2loc, n3 = self.gshape[1], int(np.prod(self.gshape[2:], dtype=int))
                ok = (px.blocked_supported(n2loc * n3) and py.blocked_supported(n3) and px.M % self.P == 0
                      and ((px.M // self.P) * n2loc * n3) % 2 == 0 and py.N == n2loc * self.P)
            self._blk_fwd = ok
        return self._blk_fwd

    def _peer(self):
        """PeerExchange of this plan's process mesh (None: NCCL all-to-all path).  Created collectively on first use."""
        if not hasattr(self, '_peer_x'):
            from .transposes import PeerExchange
            self._peer_x = PeerExchange.create(self.dist) if self.P > 1 else None
        return self._peer_x

    @staticmethod
    def _groups(n, want):
        g = max(1, min(want, n))
        cuts = [round(i * n / g) for i in range(g + 1)]
        return [(cuts[i], cuts[i + 1]) for i in range(g) if cuts[i + 1] > cuts[i]]

    def _backward_blocked_levels(self, prev, lvl):
        """Levels dim-2 (y pass) and dim-1 (x pass) of the backward tree with the all-to-all in between.  The stack of y-level
        arrays is exchanged in groups: the all-to-all of one group runs (on the communicator's stream) while the y passes of
        the next group and the x passes of the previous one occupy the SMs."""
        from .solvers import Timed
        px, py = self._xy_plans()
        nodes = self.levels[lvl]
        order = sorted(nodes.items(), key=lambda kv: kv[1]['index'])
        nn = len(order)
        n1loc = self.level_shapes[lvl][0]
        n2 = self.gshape_full[1]; n2loc = n2 // self.P
        n3 = int(np.prod(self.gshape_full[2:], dtype=int))
        per_field = n1loc * n2loc * n3
        peer = self._peer()
        if peer is not None:
            # the y passes store every peer's rows straight into that peer's receive buffer (NVLink peer memory): no send
            # buffer, no communication kernel; ONE device-side barrier orders the x passes after all writers
            recv, peer_ptrs, peer_h = peer.buffers('bwd', self.P * nn * per_field)
            rank = self.dist.rank
            groups = [(0, nn)]
        else:
            send = self._scratch(('blk_send_bwd',), (self.P * nn * per_field,))
            recv = self._scratch(('blk_recv_bwd',), (self.P * nn * per_field,))
            groups = self._groups(nn, 3)
        handles, group_of, base_of = [], {}, {}
        for gi, (g0, g1) in enumerate(groups):
            ng = g1 - g0
            off = self.P * g0 * per_field                        # groups are laid out one after the other
            for key, nd in order[g0:g1]:
                f = nd['field']
                src = (f.device_data()[self._comp_index(f, nd['comp'])] if lvl == 0 else prev[self.levels[lvl - 1][nd['parent']]['index']])
                local = nd['index'] - g0
                group_of[key] = gi; base_of[key] = (off + local * per_field, ng * per_field)
                with Timed(self.solver.prof, "transform_bwd_axis1", 8 * (src.numel() + n1loc * n2 * n3)):
                    if peer is not None:
                        # block for peer p lands where the all-to-all would have put it: slot `rank` of p's group region
                        dst = [peer_ptrs[p] + 8 * (off + rank * ng * per_field + local * per_field) for p in range(self.P)]
                        py.backward_peer(src.data_ptr(), recv.data_ptr(), n1loc, n3, self.device, n2loc, dst, deriv=nd['deriv'])
                    else:
                        py.backward_blocked(src.data_ptr(), send.data_ptr() + 8 * (off + local * per_field), n1loc, n3, self.device,
                                            deriv=nd['deriv'], out_block=(n2loc, ng * per_field))
            sl = slice(off, off + self.P * ng * per_field)
            with Timed(self.solver.prof, "transpose_bwd", 8 * 2 * self.P * ng * per_field):
                if peer is not None:
                    peer.barrier(peer_h)
                    handles.append(None)
                else:
                    handles.append(self.planner.alltoall_async(recv[sl], send[sl]))
        inner = n2loc * n3
        waited = set()
        children = sorted(self.levels[lvl + 1].items(), key=lambda kv: group_of[kv[1]['parent']])
        for key, nd in children:
            gi = group_of[nd['parent']]
            if gi not in waited:
                waited.add(gi)
                if handles[gi] is not None:
                    with Timed(self.solver.prof, "transpose_bwd", 0):
                        handles[gi].wait()
            dst = self.grid_in[self._input_slot(key)]
            base, stride = base_of[nd['parent']]
            with Timed(self.solver.prof, "transform_bwd_axis0", 8 * (n1loc * self.P * inner + dst.numel())):
                px.backward_blocked(recv.data_ptr() + 8 * base, dst.data_ptr(), 1, inner, self.device,
                                    deriv=nd['deriv'], in_block=(n1loc, stride))

    def _forward_blocked_xy(self, cur):
        """x pass into the send buffer, all-to-all, y pass out of the receive buffer (in two groups of outputs so that the
        exchange of one overlaps the passes of the other); returns the (n_out, n1loc, My, ...) stack."""
        from .solvers import Timed
        px, py = self._xy_plans()
        n_out = cur.shape[0]
        n2loc = cur.shape[2]
        n3 = int(np.prod(cur.shape[3:], dtype=int))
        inner = n2loc * n3
        n1loc = px.M // self.P
        per_out_g = px.N * inner                                  # grid elements per output
        per_out_c = px.M * inner                                  # coefficient elements per output (all peers' blocks)
        peer = self._peer()
        if peer is not None:
            recv, peer_ptrs, peer_h = peer.buffers('fwd', n_out * per_out_c)
            rank = self.dist.rank
            groups = [(0, n_out)]
        else:
            send = self._scratch(('blk_send_fwd',), (n_out * per_out_c,))
            recv = self._scratch(('blk_recv_fwd',), (n_out * per_out_c,))
            groups = self._groups(n_out, 2)
        out = self._scratch(('fwd', 1), (n_out, n1loc, py.M) + tuple(cur.shape[3:]))
        flat_in = cur.reshape(-1)
        handles = []
        for g0, g1 in groups:
            ng = g1 - g0
            sl = slice(g0 * per_out_c, g1 * per_out_c)
            with Timed(self.solver.prof, "transform_fwd_axis0", 8 * ng * (per_out_g + per_out_c)):
                if peer is not None:
                    # peer p's block (its n1loc coefficient rows of all ng outputs) -> slot `rank` of p's receive buffer
                    dst = [peer_ptrs[p] + 8 * (g0 * per_out_c + rank * ng * n1loc * inner) for p in range(self.P)]
                    px.forward_peer(flat_in.data_ptr() + 8 * g0 * per_out_g, recv.data_ptr(), ng, inner, self.device, n1loc, dst)
                else:
                    px.forward_blocked(flat_in.data_ptr() + 8 * g0 * per_out_g, send.data_ptr() + 8 * g0 * per_out_c, ng, inner, self.device,
                                       out_block=(n1loc, ng * n1loc * inner))
            with Timed(self.solver.prof, "transpose_fwd", 8 * 2 * ng * per_out_c):
                if peer is not None:
                    peer.barrier(peer_h)
                    handles.append(None)
                else:
                    handles.append(self.planner.alltoall_async(recv[sl], send[sl]))
        per_out_y = n1loc * py.M * n3
        for (g0, g1), h in zip(groups, handles):
            ng = g1 - g0
            if h is not None:
                with Timed(self.solver.prof, "transpose_fwd", 0):
                    h.wait()
            outer = ng * n1loc
            with Timed(self.solver.prof, "transform_fwd_axis1", 8 * ng * (per_out_c + per_out_y)):
                py.forward_blocked(recv.data_ptr() + 8 * g0 * per_out_c, out.reshape(-1).data_ptr() + 8 * g0 * per_out_y, outer, n3, self.device,
                                   in_block=(n2loc, outer * n2loc * n3))
        return out

    def _scratch(self, key, shape):
        import torch
        if not hasattr(self, '_scr'):
            self._scr = {}
        t = self._scr.get(key)
        if t is None or tuple(t.shape) != tuple(shape):
            t = torch.empty(shape, dtype=torch.float64, device=self.device)
            self._scr[key] = t
        return t

    def _comp_index(self, f, comp):
        if not f.tensorsig:
            return ()
        return tuple(int(i) for i in np.unravel_index(comp, f.tshape))

    def _input_slot(self, leaf_key):
        if not hasattr(self, '_slot'):
            self._slot = {}
            for i, lk in enumerate(self.leaf_of_input):
                self._slot[lk] = i
        return self._slot[leaf_key]


class _ExpressionHost:
    """What RHSPlan needs from a solver, for expressions evaluated outside a solver (analysis tasks, flow properties)."""

    def __init__(self, expr):
        from types import SimpleNamespace
        from .pencils import Arena
        from .lib import compute_device
        dist = expr.dist
        self.dist = dist
        self.device = compute_device()
        dist.device = self.device
        self.prof = None
        self.problem = SimpleNamespace(dist=dist, equations=[dict(RHS=expr, bases=expr.bases, tensorsig=expr.tensorsig)])
        self.eq_arena = Arena(dist, [(tuple(cs.dim for cs in expr.tensorsig), expr.bases)])


# numpy ufunc -> torch function applied to the device grid values
_TORCH_NAMES = {'absolute': 'abs', 'arcsin': 'asin', 'arccos': 'acos', 'arctan': 'atan', 'arcsinh': 'asinh', 'arccosh': 'acosh',
                'arctanh': 'atanh', 'conjugate': 'conj'}


class Stager:
    """Rewrites an expression into stages + a polynomial remainder that one RHSPlan can evaluate:
      * a grid function np.f(arg) (reference UnaryGridFunction, operators.py:505-640) becomes "polynomial part of arg on the
        dealiased grid -> f pointwise -> temporary field on the grid", which enters later products without a coefficient round trip;
      * a differential operator applied to a product (div(u*b), the reference evaluates the product, transforms it to coefficient
        space and differentiates there) becomes "product -> temporary field in coefficient space".
    Stages run in order before the remainder; every stage is an RHSPlan of its own (same transform / product kernels)."""

    _DIFF = (ops.Differentiate, ops.Gradient, ops.Divergence, ops.Laplacian)
    _PRODUCTS = (ops.Multiply, ops.DotProduct, ops.Power)

    def __init__(self):
        self.stages = []           # ('grid', plan, torch function, field) | ('coeff', plan, arena tensor, view, field)

    @staticmethod
    def plan(e):
        plan = RHSPlan(_ExpressionHost(e))
        if plan.n_out == 0 and not plan.static_entries:
            raise NotImplementedError("expression evaluates to zero")
        return plan

    @classmethod
    def _has_product(cls, e):
        if isinstance(e, cls._PRODUCTS) or getattr(e, '_grid_leaf', False):
            return True
        return any(cls._has_product(a) for a in getattr(e, 'args', []) if isinstance(a, Operand))

    def rewrite(self, e):
        import copy, torch
        if isinstance(e, ops.UnaryGridFunction):
            arg = self.rewrite(e.args[0])
            plan = self.plan(arg)
            if plan.static_entries:
                raise NotImplementedError("constants inside grid functions")
            name = getattr(e.func, '__name__', str(e.func))
            fn = getattr(torch, _TORCH_NAMES.get(name, name), None)
            if fn is None:
                raise NotImplementedError(f"grid function {name!r} has no device implementation")
            if any(b is None for b in e.bases):
                raise NotImplementedError("grid functions of lower-dimensional operands")
            tmp = Field(e.dist, bases=tuple(dict.fromkeys(e.bases)), tensorsig=e.tensorsig, dtype=e.dtype)
            e.dist._fields.pop()
            tmp._grid_leaf = True
            self.stages.append(('grid', plan, fn, tmp))
            return tmp
        if isinstance(e, Field) or not isinstance(e, Operand):
            return e
        new = copy.copy(e)
        new.args = [self.rewrite(a) for a in e.args]
        if isinstance(e, self._DIFF) and self._has_product(new.args[0]):
            inner = new.args[0]
            if any(b is None for b in inner.bases):
                raise NotImplementedError("derivatives of lower-dimensional products")
            plan = self.plan(inner)
            host = plan.solver
            out_t = torch.zeros(host.eq_arena.size, dtype=torch.float64, device=host.device)
            plan.set_static(out_t)
            tmp = Field(inner.dist, bases=tuple(dict.fromkeys(inner.bases)), tensorsig=inner.tensorsig, dtype=inner.dtype)
            inner.dist._fields.pop()
            tsh, shp = host.eq_arena.shapes[0]
            self.stages.append(('coeff', plan, out_t, out_t.view(tuple(tsh) + tuple(shp)), tmp))
            new.args = [tmp]
        return new

    @staticmethod
    def run(stages):
        for st in stages:
            if st[0] == 'grid':
                _, plan, fn, tmp = st
                vals = fn(plan.evaluate(None, grid_only=True))
                tmp.set_device_data(vals.reshape(tuple(cs.dim for cs in tmp.tensorsig) + tuple(plan.gshape)), 'g', scales=plan.dealias)
            else:
                _, plan, out_t, view, tmp = st
                plan.evaluate(out_t)
                tmp.set_device_data(view, 'c')


class StagedRHSPlan:
    """Right-hand sides that are not polynomial in derivatives of fields -- grid functions (np.tanh(b)) and derivatives of products
    (div(u*b)): the Stager's stages, then the ordinary RHSPlan over the rewritten equations.  Same interface as RHSPlan."""

    def __init__(self, solver):
        stager = Stager()
        eqs = []
        for eq in solver.problem.equations:
            new = dict(eq)
            if isinstance(eq['RHS'], Operand):
                new['RHS'] = stager.rewrite(eq['RHS'])
            eqs.append(new)
        self.stages = stager.stages
        self.plan = RHSPlan(_ProfProxy(solver, eqs))

    def set_static(self, arena_tensor):
        self.plan.set_static(arena_tensor)

    def evaluate(self, eq_arena_tensor):
        Stager.run(self.stages)
        self.plan.evaluate(eq_arena_tensor)

    def __getattr__(self, name):                      # bench / tests look at the main plan's attributes (_blocked_bwd_ok, ...)
        return getattr(self.plan, name)


class _ProfProxy:
    """The solver as the main RHSPlan sees it, with the rewritten equations."""

    def __init__(self, solver, equations):
        from types import SimpleNamespace
        self._solver = solver
        self.problem = SimpleNamespace(dist=solver.problem.dist, equations=equations)

    def __getattr__(self, name):
        return getattr(self._solver, name)


class ExpressionProgram:
    """Stand-alone evaluation of an operator expression of Cartesian fields into a new Field (reference Future.evaluate,
    core/future.py:149-206, used by output handlers and flow properties -- not part of the per-step path).

    The expression is compiled once: every grid function np.f(arg) (reference UnaryGridFunction, operators.py:505-640)
    becomes a stage "polynomial part of arg on the dealiased grid -> f pointwise -> temporary field", and what remains is a
    polynomial expression of fields that one RHSPlan evaluates into coefficient space -- the same transform and product
    kernels as the solver's right-hand sides."""

    def __init__(self, expr):
        # outer reductions -- integ / ave / interpolation, possibly nested and scaled (Nusselt numbers, profiles, mid-plane values):
        # contractions of the coefficient data with the basis' row vectors (reference IntegrateJacobi / InterpolateRealFourier ...,
        # core/basis.py:721-789, 1037-1290), applied to the result of the remaining expression
        self.reductions = []
        while True:
            if isinstance(expr, ops.ScalarMul) and isinstance(expr.args[0], (ops.Integrate, ops.Interpolate)):
                self.reductions.append(('scale', expr.c)); expr = expr.args[0]
            elif isinstance(expr, ops.Integrate):
                self.reductions.append(('integ', expr.axes, expr.average)); expr = expr.args[0]
            elif isinstance(expr, ops.Interpolate) and not expr.trivial:
                self.reductions.append(('interp', expr.axis, expr.position)); expr = expr.args[0]
            elif isinstance(expr, ops.Lift):
                self.reductions.append(('lift', expr.axis, expr.basis, expr.n)); expr = expr.args[0]
            else:
                break
        self.reductions.reverse()

        stager = Stager()
        self.stages = stager.stages
        sub = stager.rewrite
        final = sub(expr)
        self.result_field = final if isinstance(final, Field) else None
        if self.result_field is None:
            self.final = self._plan(final)
            host = self.final.solver
            import torch
            self.out_t = torch.zeros(host.eq_arena.size, dtype=torch.float64, device=host.device)
            self.final.set_static(self.out_t)
            self.out = Field(expr.dist, bases=tuple(dict.fromkeys(b for b in expr.bases if b is not None)), tensorsig=expr.tensorsig, dtype=expr.dtype)
            expr.dist._fields.pop()
            tsh, shp = host.eq_arena.shapes[0]
            self.out_view = self.out_t.view(tuple(tsh) + tuple(shp))

    @staticmethod
    def _plan(e):
        return Stager.plan(e)

    def run(self):
        Stager.run(self.stages)
        if self.result_field is not None:
            out = self.result_field
        else:
            self.final.evaluate(self.out_t)
            self.out.set_device_data(self.out_view, 'c')
            out = self.out
        # like the reference's evaluation, which moves the operands to the dealiased grid in place (core/future.py:149-206): the
        # fields of the expression are left at their dealias scales (their coefficients are untouched)
        plans = [st[1] for st in self.stages] + ([self.final] if self.result_field is None else [])
        for plan in plans:
            for f, c, dv in getattr(plan, 'input_keys', []):
                if not getattr(f, '_grid_leaf', False) and f.layout == 'c':
                    f.change_scales(f.dealias)
        return self._reduce(out) if self.reductions else out

    def _reduce(self, f):
        """Apply the outer integrations / averages / interpolations to the coefficient data of f."""
        import torch
        dist = f.dist
        f.change_layout('c')
        data = f.device_data()
        bases = list(f.bases)
        nt = len(f.tshape)
        for red in self.reductions:
            if red[0] == 'scale':
                data = data * red[1]
                continue
            if red[0] == 'lift':
                # operand times the n-th polynomial of the lift basis: its value lands in mode n (reference LiftJacobi, basis.py:790-814)
                _, ax, lb, n = red
                if lb.dim != 1 or bases[ax] is not None:
                    raise NotImplementedError("stand-alone Lift: one-dimensional lift bases over an axis without basis")
                shape = list(data.shape); shape[nt + ax] = lb.size
                lifted = torch.zeros(shape, dtype=data.dtype, device=data.device)
                lifted.select(nt + ax, n % lb.size).copy_(data.select(nt + ax, 0))
                data = lifted
                bases[ax] = lb
                continue
            axes = red[1] if red[0] == 'integ' else (red[1],)
            for ax in axes:
                b = bases[ax]
                if b is None:
                    continue
                if red[0] == 'interp':
                    row = b.interpolation_vector(red[2])
                elif red[2] and hasattr(b, 'average_vector'):
                    row = b.average_vector()
                else:
                    row = b.integration_vector()
                    if red[2]:
                        row = row / b.COV.problem_length
                row = np.asarray(row.todense()).ravel()
                if np.iscomplexobj(row) and not np.iscomplexobj(np.zeros(0, dtype=f.dtype)):
                    row = row.real
                w = torch.from_numpy(np.ascontiguousarray(row[dist.coeff_local_slice(ax, b)])).to(data.device).to(data.dtype)
                shape = [1] * data.dim(); shape[nt + ax] = -1
                data = (data * w.reshape(shape)).sum(dim=nt + ax, keepdim=True)
                if ax == 0 and dist.size > 1:
                    import torch.distributed as td
                    td.all_reduce(data, op=td.ReduceOp.SUM)
                bases[ax] = None
        out = Field(dist, bases=tuple(dict.fromkeys(b for b in bases if b is not None)), tensorsig=f.tensorsig, dtype=f.dtype)
        dist._fields.pop()
        out.set_device_data(data.contiguous(), 'c')
        return out


def evaluate_expression(expr):
    """Stand-alone evaluation (reference Future.evaluate): output expressions on the sphere / shell (dedalus_b200/analysis.py), and
    any polynomial / grid-function expression of Cartesian fields (compiled program cached on the expression)."""
    if getattr(expr.dist.coordsys, 'curvilinear', False):
        from .analysis import evaluate_curvilinear
        return evaluate_curvilinear(expr)
    prog = getattr(expr, '_program', None)
    if prog is None:
        prog = expr._program = ExpressionProgram(expr)
    return prog.run()
