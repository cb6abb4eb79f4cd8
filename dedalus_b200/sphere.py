"""S2 sphere basis (spin-weighted spherical harmonics) and the device transform chain of sphere fields.

Reference: core/basis.py:1561-1717 (SpinRecombinationBasis / SpinBasis), 2672-3277 (SphereBasis), core/coords.py:201-252
(S2Coordinates), core/transforms.py:1251-1340 (SWSHColatitudeTransform), libraries/spin_recombination.pyx.

Layouts (real dtype; the only one built):
  grid          (comps, Nphi_g, Ntheta_g)      coordinate components (phi, theta)
  coefficient   (comps, Nphi / 2, Lmax + 1 + shift)   spin components (-, +); rows 2j, 2j + 1 = cos / -sin part (real and
                imaginary part of the exp(i m phi) coefficient) of m = j at columns l + shift (l >= m) AND of the folded
                partner m' = Nphi/2 - 1 - j at columns Lmax - l: the reference's repacked triangular truncation
                (core/basis.py:2800-2809, 2872-2914), reproduced exactly so that f['c'] is interchangeable.
The intermediate (azimuthal coefficient, colatitude grid) layout is internal here and keeps the FFT's natural m order: the
reference's azimuthal permutation (basis.py:2757-2777) only serves its MPI block decomposition and is folded into the
m_maps handed to the colatitude transform.

Device chain towards the grid: SWSH colatitude transform per spin weight (csrc/pointwise.cu k_ragged_matvec) -> spin to
component recombination (csrc/banded.cu k_pair_lincomb) -> azimuthal real FFT (csrc/rfft_regs.cu / fft.cu).
"""
import numpy as np
from .basis import Basis
from .coords import S2Coordinates


class SphereBasis(Basis):
    dim = 2
    kind = "Sphere"
    constant_mode_value = 1 / np.sqrt(2)

    def __init__(self, coordsys, shape, dtype=np.float64, radius=1, dealias=(1, 1), azimuth_library=None, colatitude_library=None):
        from .coords import SphericalCoordinates
        if not isinstance(coordsys, (S2Coordinates, SphericalCoordinates)):
            raise ValueError("Sphere coordsys must be S2Coordinates.")
        shape = tuple(int(n) for n in shape)
        if len(shape) != 2:
            raise ValueError("Sphere shape must have length 2.")
        if radius < 0:
            raise ValueError("Sphere radius must be non-negative.")
        if isinstance(dealias, (int, float)):
            dealias = (dealias,) * 2
        dealias = tuple(dealias)
        if len(dealias) != 2:
            raise ValueError("Sphere dealias must have length 2.")
        if np.dtype(dtype) != np.float64:
            raise NotImplementedError("only real (float64) sphere fields are built")
        if shape[0] % 4 != 0:
            raise ValueError("Don't use a phi resolution that isn't divisible by 4, please")
        self.coordsys, self.coord = coordsys, coordsys.coords[0]
        self.shape, self.dtype, self.radius, self.dealias = shape, np.float64, radius, dealias
        self.volume = 4 * np.pi * radius**2
        self.mmax = (shape[0] - 1) // 2
        self.Lmax = max(0, shape[1] - 2)                      # real dtype (reference basis.py:2723-2724)
        self.shift = max(0, self.Lmax + 2 - shape[0] // 2)
        self.coeff_shape = (shape[0] // 2, self.Lmax + 1 + self.shift)
        self._key = (coordsys, shape, radius, dealias)
        self._ctor_args = dict(coordsys=coordsys, shape=shape, dtype=np.float64, radius=radius, dealias=dealias)
        self._plans = {}

    @classmethod
    def _make(cls, **kw):
        return cls(**kw)

    def __repr__(self):
        return f"SphereBasis({self.shape}, R={self.radius})"

    # ---- per-axis accessors used by Field / Distributor
    def axis_size(self, sub=0):
        return self.coeff_shape[sub]

    def axis_grid_size(self, scale, sub=0):
        return int(np.ceil(scale * self.shape[sub]))

    def axis_dealias(self, sub=0):
        return self.dealias[sub]

    def axis_group_size(self, sub=0):
        return (2, 1)[sub]

    def grid_shape(self, scales):
        return tuple(self.axis_grid_size(s, i) for i, s in enumerate(scales))

    # ---- basis algebra (reference basis.py:2916-2938)
    def __add__(self, other):
        if other is None or other == self:
            return self
        if isinstance(other, SphereBasis) and (self.coordsys, self.radius, self.dealias) == (other.coordsys, other.radius, other.dealias):
            return self.clone_with(shape=tuple(np.maximum(self.shape, other.shape)))
        if getattr(other, 'kind', None) == "Shell":        # a sphere basis met on the angular axes of a shell expression
            return other
        return NotImplemented
    __radd__ = __add__
    __mul__ = __add__
    __rmul__ = __add__

    def derivative_basis(self, order=1):
        return self

    # ---- grids (reference basis.py:3013-3045)
    def global_grid_azimuth(self, scale):
        N = self.axis_grid_size(scale, 0)
        return (2 * np.pi / N) * np.arange(N)

    def colatitude_quadrature(self, scale):
        """cos(theta) nodes (ascending) and weights: Gauss-Legendre on N = ceil(scale * Ntheta) points."""
        from scipy.special import roots_jacobi
        return roots_jacobi(self.axis_grid_size(scale, 1), 0.0, 0.0)

    def global_grid_colatitude(self, scale):
        return np.arccos(self.colatitude_quadrature(scale)[0])

    def global_colatitude_weights(self, scale=1):
        return self.colatitude_quadrature(scale)[1]

    def local_grids(self, dist, scales):
        ax = dist.get_basis_axis(self)
        out = []
        for sub, g in enumerate((self.global_grid_azimuth(scales[0]), self.global_grid_colatitude(scales[1]))):
            g = g[dist.grid_local_slice(ax + sub, self, scales[sub])]          # colatitude (axis 1) is distributed on the grid
            shp = [1] * dist.dim
            shp[ax + sub] = g.size
            out.append(g.reshape(shp))
        return tuple(out)

    def global_grids(self, dist, scales):
        return self.local_grids(dist, scales)

    # ---- coefficient packing (reference elements_to_groups, basis.py:2872-2914)
    def elements_to_groups(self):
        """(m, l) of every coefficient element, arrays of shape coeff_shape (negative l never occurs; elements without a
        mode -- l > Lmax -- carry l beyond Lmax)."""
        if 'groups' in self._plans:
            return self._plans['groups']
        Nphi, Lmax, shift = self.shape[0], self.Lmax, self.shift
        i, j = np.indices(self.coeff_shape)
        m = i // 2
        ell = j - shift
        neg = ell < m
        m = np.where(neg, (Nphi // 2 - 1) - m, m)
        ell = np.where(neg, Lmax - j, ell)
        zero = i < 2
        m = np.where(zero, 0, m)
        ell = np.where(zero, j, ell)
        mmax_ = zero & (j > Lmax)
        m = np.where(mmax_, Nphi // 2 - 1, m)
        ell = np.where(mmax_, j - shift, ell)
        self._plans['groups'] = (m, ell)
        return m, ell

    def spin_weights(self, tensorsig):
        """Spin total of every tensor component, shape (2,) * rank (spin ordering -, +)."""
        S = np.zeros(tuple(cs.dim for cs in tensorsig), dtype=int)
        for i, cs in enumerate(tensorsig):
            if not hasattr(cs, 'spin_ordering'):
                raise NotImplementedError("tensor indices over non-curvilinear coordinate systems on a sphere basis")
            shp = [1] * len(tensorsig); shp[i] = cs.dim           # S2: (-, +); spherical: (-, +, 0)
            S = S + np.array(cs.spin_ordering).reshape(shp)
        return S

    def valid_elements(self, tensorsig):
        """Boolean mask over (components, coeff_shape) of the modes that exist (reference basis.py:3178-3211)."""
        m, ell = self.elements_to_groups()
        S = self.spin_weights(tensorsig).reshape(-1)
        part = np.indices(self.coeff_shape)[0] % 2
        valid = np.ones((S.size,) + self.coeff_shape, dtype=bool)
        for c, s in enumerate(S):
            valid[c] = (ell >= np.maximum(m, abs(s))) & (ell <= self.Lmax)
            if len(tensorsig) <= 1:
                valid[c] &= ~((ell == 0) & (part == 1))       # -sin part of l = 0
        return valid

    def mode_columns(self, m):
        """(pair index j, column indices of l = m .. Lmax) of azimuthal wavenumber m in the coefficient packing."""
        ms, ells = self.elements_to_groups()
        rows, cols = np.nonzero((ms[0::2] == m) & (ells[0::2] <= self.Lmax) & (ells[0::2] >= m))
        if rows.size == 0:
            return None, np.zeros(0, dtype=int)
        j = int(rows[0])
        assert np.all(rows == j)
        order = np.argsort(ells[2 * j, cols])
        cols = cols[order]
        assert np.array_equal(ells[2 * j, cols], np.arange(m, self.Lmax + 1))
        return j, cols

    def local_pairs(self, dist=None):
        """Block [j0, j1) of the azimuthal pairs of the coefficient packing owned by this rank (all of them on one GPU).  Pair
        j carries m = j and its folded partner Nphi/2 - 1 - j: the reference's load-balanced layout, core/basis.py:2757-2777."""
        npairs = self.shape[0] // 4
        if dist is None or dist.size == 1:
            return 0, npairs
        return dist.block_range(npairs, dist.size, dist.rank)

    def local_wavenumbers(self, dist=None):
        """[(m, row of its cos part in the rank's (azimuthal coefficient, colatitude grid) array)]: single GPU: natural FFT order
        (row 2 m); distributed: the unfolded wavenumbers of the rank's pairs ascending, then their folded partners ascending."""
        N2 = self.shape[0] // 2
        if dist is None or dist.size == 1:
            return [(m, 2 * m) for m in range(N2)]
        j0, j1 = self.local_pairs(dist)
        npl = j1 - j0
        out = [(j, 2 * (j - j0)) for j in range(j0, j1)]
        out += [(N2 - 1 - j, 2 * npl + 2 * (j1 - 1 - j)) for j in range(j1 - 1, j0 - 1, -1)]
        return out

    def m_maps(self, dist=None):
        """Rows (m, mg0, mg1, mc0, mc1, ell_start, ell_stop or -1, ell_step) for SWSHColatitudeTransform: the reference's
        m_maps (basis.py:2940-2970) for the wavenumbers of this rank, positions as in local_wavenumbers()."""
        j0, _ = self.local_pairs(dist)
        rows = []
        for m, row in self.local_wavenumbers(dist):
            j, cols = self.mode_columns(m)
            if j is None:
                # |m| > Lmax: no coefficients; the transform zero-fills these grid lines on the way back
                rows.append((m, row, row + 2, 0, 2, 0, 0, 1))
                continue
            step = 1 if (cols.size < 2 or cols[1] > cols[0]) else -1
            assert np.all(np.diff(cols) == step)
            stop = int(cols[-1]) + step
            rows.append((m, row, row + 2, 2 * (j - j0), 2 * (j - j0) + 2, int(cols[0]), -1 if stop < 0 else stop, step))
        return rows

    # ---- operator symbols (reference basis.py:3150-3152, libraries/dedalus_sphere/sphere.py k_element)
    @staticmethod
    def k(l, s, mu):
        l = np.asarray(l, dtype=float)
        return -mu * np.sqrt(np.maximum(0, (l - mu * s) * (l + mu * s + 1) / 2))

    def cos_matrix(self, m, s):
        """cos(theta) multiplication on l = Lmin .. Lmax, Lmin = max(|m|, |s|): the Jacobi operator Z on (a, b) = (|m+s|, |m-s|)
        truncated (reference operators.py:3043-3050 -> libraries/dedalus_sphere/sphere.py:91-95)."""
        from . import jacobi
        Lmin = max(abs(m), abs(s))
        n = self.Lmax + 1 - Lmin
        if n <= 0:
            return None, Lmin
        return jacobi.jacobi_matrix(n, abs(m + s), abs(m - s)), Lmin

    # ---- device transforms
    def colatitude_plan(self, Ntheta_g, s, dist=None):
        P, rank = (1, 0) if (dist is None or dist.size == 1) else (dist.size, dist.rank)
        key = (int(Ntheta_g), int(s), P, rank)
        if key not in self._plans:
            from .transforms import SWSHColatitudeTransform
            self._plans[key] = SWSHColatitudeTransform(Ntheta_g, self.Lmax, self.m_maps(dist), s)
        return self._plans[key]

    def hop(self, dist):
        key = ('hop', dist.size, dist.rank)
        if key not in self._plans:
            self._plans[key] = SphereHop(self, dist)
        return self._plans[key]

    def azimuth_plan(self, Nphi_g):
        key = ('az', int(Nphi_g))
        if key not in self._plans:
            from .transforms import RealFourierTransform
            self._plans[key] = RealFourierTransform(Nphi_g, self.shape[0], kscale=1.0)
        return self._plans[key]

    def recombination_table(self, rank, forward, device, cs=S2Coordinates):
        """Device program of db_pair_lincomb for the component <-> spin recombination of a rank-`rank` tensor over `cs` (one
        coordinate-system class for every index, or a tuple of them: spherical and S2 indices mixed)."""
        css = tuple(cs) if isinstance(cs, tuple) else (cs,) * rank
        key = ('rec', bool(forward), str(device), tuple(c.dim for c in css))
        if key not in self._plans:
            U = np.ones((1, 1))
            for c in css:
                U = np.kron(U, c.U_forward(1) if forward else c.U_backward(1))
            self._plans[key] = PairProgram.from_matrix(U, device)
        return self._plans[key]


class SphereHop:
    """Transpose between the two distributed intermediate layouts of a sphere transform chain (P GPUs):
        A  (comps, rows of the rank's wavenumbers, ALL colatitude points, trailing)    after / before the colatitude transform
        B  (comps, ALL azimuthal rows in natural FFT order, the rank's colatitude block, trailing)   before / after the FFT
    = pack -> all-to-all -> unpack (dedalus_b200/transposes.py TransposePlanner, csrc/pointwise.cu k_tr_chunks) plus a row
    permutation (db_index_move_runs) between the rank-major row order the exchange delivers and the FFT's natural order.
    Replaces the reference's azimuth <-> colatitude Transpose of a curvilinear layout chain (core/distributor.py:696-924)."""

    def __init__(self, basis, dist):
        import torch
        from .transposes import get_planner
        self.basis, self.dist = basis, dist
        self.P = dist.size
        self.planner = get_planner(dist)
        Nphi = basis.shape[0]
        N2 = Nphi // 2
        npairs = Nphi // 4
        npl = npairs // self.P
        # natural row of each row of the rank-major order delivered by the exchange
        nat = np.zeros(Nphi, dtype=np.int64)
        for p in range(self.P):
            j0, j1 = p * npl, (p + 1) * npl
            rows = [(j, 2 * (j - j0)) for j in range(j0, j1)] + [(N2 - 1 - j, 2 * npl + 2 * (j1 - 1 - j)) for j in range(j1 - 1, j0 - 1, -1)]
            for m, r in rows:
                nat[p * 4 * npl + r], nat[p * 4 * npl + r + 1] = 2 * m, 2 * m + 1
        self.nat = nat
        self._idx = {}

    def _table(self, ncomp, run, device):
        import torch
        key = (ncomp, run, str(device))
        if key not in self._idx:
            Nphi = self.basis.shape[0]
            idx = (np.arange(ncomp)[:, None] * Nphi + self.nat[None, :]) * run          # entry (c, rank-major row) -> natural row offset
            self._idx[key] = torch.from_numpy(np.ascontiguousarray(idx.ravel())).to(device)
        return self._idx[key]

    def to_grid_side(self, A):
        """A (ncomp, 4 npl, Ntheta_g, trail) -> B (ncomp, Nphi, Ntheta_g / P, trail)."""
        import torch
        from .lib import get_lib, current_stream
        ncomp, rows, Nt, trail = A.shape
        tb = Nt // self.P
        rm = torch.empty((ncomp, rows * self.P, tb, trail), dtype=A.dtype, device=A.device)
        self.planner.localize_columns(A, rm)
        B = torch.empty_like(rm)
        run = tb * trail
        get_lib().call("db_index_move_runs", self._table(ncomp, run, A.device).data_ptr(), ncomp * rows * self.P, run,
                       B.data_ptr(), rm.data_ptr(), 0, current_stream())                # scatter: B[natural row] = rank-major row
        return B

    def to_coeff_side(self, B):
        import torch
        from .lib import get_lib, current_stream
        ncomp, Nphi, tb, trail = B.shape
        rm = torch.empty_like(B)
        run = tb * trail
        get_lib().call("db_index_move_runs", self._table(ncomp, run, B.device).data_ptr(), ncomp * Nphi, run,
                       B.data_ptr(), rm.data_ptr(), 1, current_stream())                # gather: rank-major row = B[natural row]
        A = torch.empty((ncomp, Nphi // self.P, tb * self.P, trail), dtype=B.dtype, device=B.device)
        self.planner.localize_rows(rm, A)
        return A


class PairProgram:
    """Term table of db_pair_lincomb (include/dedalus_b200.h): out[o] = sum_t (re + i im) * sym * in[src]."""

    def __init__(self, rows, device, syms=None):
        """rows: list over outputs of lists of (src, complex coefficient, symbol offset or -1)."""
        import torch
        from .lib import PairLinTerm
        nterm = sum(len(r) for r in rows)
        arr = (PairLinTerm * max(nterm, 1))()
        ptr = [0]
        t = 0
        for r in rows:
            for src, coef, sym_off in r:
                arr[t].re, arr[t].im, arr[t].sym_off, arr[t].src = float(np.real(coef)), float(np.imag(coef)), int(sym_off), int(src)
                t += 1
            ptr.append(t)
        self.n_out = len(rows)
        self.terms = torch.from_numpy(np.frombuffer(bytes(arr), dtype=np.uint8).copy()).to(device)
        self.ptr = torch.from_numpy(np.array(ptr, dtype=np.int32)).to(device)
        self.syms = syms if syms is not None else torch.zeros(1, dtype=torch.float64, device=device)

    @classmethod
    def from_matrix(cls, U, device):
        rows = [[(j, U[i, j], -1) for j in range(U.shape[1]) if U[i, j] != 0] for i in range(U.shape[0])]
        return cls(rows, device)

    def apply(self, inp, out, npair, ncol, sym_div=1):
        from .lib import get_lib, current_stream
        get_lib().call("db_pair_lincomb", inp.data_ptr(), out.data_ptr(), int(npair), int(ncol), self.n_out,
                       self.ptr.data_ptr(), self.terms.data_ptr(), self.syms.data_ptr(), int(sym_div), current_stream())


def sphere_basis_of(field_or_bases):
    bases = getattr(field_or_bases, 'bases', field_or_bases)
    for b in bases:
        if isinstance(b, SphereBasis):
            return b
    return None


def _distributed(dist):
    return dist is not None and dist.size > 1


def components_to_grid(basis, cdata, spins, rank, scales, cs=S2Coordinates, dist=None):
    """Coefficient data (ncomp, local Nphi/2 rows, Nl) of spin components -> grid data (ncomp, Nphi_g, local Ntheta_g) of
    coordinate components; components of a rank-`rank` tensor in C order.  Components of equal spin weight that are ADJACENT
    share one launch of the colatitude transform (one pass over that spin weight's matrices).  On P GPUs the azimuth <->
    colatitude transpose (SphereHop) sits between the spin recombination and the azimuthal FFT."""
    import torch
    ncomp = cdata.shape[0]
    Ng_phi, Ng_theta = basis.grid_shape(scales)
    rows = 2 * len(basis.local_wavenumbers(dist))
    cg = torch.empty((ncomp, rows, Ng_theta), dtype=cdata.dtype, device=cdata.device)
    c = 0
    while c < ncomp:
        c1 = c
        while c1 < ncomp and spins[c1] == spins[c]:
            c1 += 1
        basis.colatitude_plan(Ng_theta, spins[c], dist).backward(cdata[c:c1], cg[c:c1], 2)
        c = c1
    if rank > 0:
        cg2 = torch.empty_like(cg)
        basis.recombination_table(rank, False, cdata.device, cs).apply(cg, cg2, rows // 2, Ng_theta)
        cg = cg2
    if _distributed(dist):
        cg = basis.hop(dist).to_grid_side(cg.unsqueeze(-1)).squeeze(-1)
    g = torch.empty((ncomp, Ng_phi, cg.shape[2]), dtype=cdata.dtype, device=cdata.device)
    basis.azimuth_plan(Ng_phi).backward(cg.contiguous(), g, 1)
    return g


def grid_to_components(basis, gdata, spins, rank, out=None, cs=S2Coordinates, dist=None):
    """Inverse chain of components_to_grid."""
    import torch
    ncomp, Ng_phi, tb = gdata.shape
    cg = torch.empty((ncomp, basis.shape[0], tb), dtype=gdata.dtype, device=gdata.device)
    basis.azimuth_plan(Ng_phi).forward(gdata, cg, 1)
    if _distributed(dist):
        cg = basis.hop(dist).to_coeff_side(cg.unsqueeze(-1)).squeeze(-1).contiguous()
    rows, Ng_theta = cg.shape[1], cg.shape[2]
    if rank > 0:
        cg2 = torch.empty_like(cg)
        basis.recombination_table(rank, True, gdata.device, cs).apply(cg, cg2, rows // 2, Ng_theta)
        cg = cg2
    if out is None:
        j0, j1 = basis.local_pairs(dist)
        out = torch.zeros((ncomp, 2 * (j1 - j0), basis.coeff_shape[1]), dtype=gdata.dtype, device=gdata.device)
    c = 0
    while c < ncomp:
        c1 = c
        while c1 < ncomp and spins[c1] == spins[c]:
            c1 += 1
        basis.colatitude_plan(Ng_theta, spins[c], dist).forward(cg[c:c1], out[c:c1], 2)
        c = c1
    return out


def transform_sphere_field(field, layout):
    """field['c'] <-> field['g'] for fields on a SphereBasis (single GPU)."""
    basis = sphere_basis_of(field)
    if any(b is not None and b is not basis for b in field.bases):
        raise NotImplementedError("sphere basis combined with other bases")
    ax = field.dist.get_basis_axis(basis)
    scales = field.scales[ax:ax + 2]
    rank = len(field.tensorsig)
    cs = tuple(type(c) for c in field.tensorsig) if rank else S2Coordinates
    trail = (1,) * (field.dist.dim - ax - 2)             # a sphere inside a 3-D distributor: trailing constant axis
    spins = [int(s) for s in basis.spin_weights(field.tensorsig).reshape(-1)]
    data = field.device_data()
    ncomp = max(1, len(spins))
    dist = field.dist
    if layout == 'g':
        cdata = data.reshape((ncomp,) + tuple(data.shape[len(field.tshape):len(field.tshape) + 2])).contiguous()
        g = components_to_grid(basis, cdata, spins, rank, scales, cs, dist)
        field.set_device_data(g.reshape(field.tshape + tuple(g.shape[1:]) + trail), 'g')
    else:
        gdata = data.reshape((ncomp,) + tuple(data.shape[len(field.tshape):len(field.tshape) + 2])).contiguous()
        c = grid_to_components(basis, gdata, spins, rank, cs=cs, dist=dist)
        field.set_device_data(c.reshape(field.tshape + tuple(c.shape[1:]) + trail), 'c')


# ------------------------------------------------------------------------------------------------------------
# Linear operators on sphere fields (host side): symbols per degree and per-m matrices
# ------------------------------------------------------------------------------------------------------------
def _grad_symbol(basis, s_in, mu):
    """k(l, s, mu) / R over l = 0 .. Lmax, zero where the input or output spin exceeds l (reference basis.py:3370-3377)."""
    ell = np.arange(basis.Lmax + 1)
    k = SphereBasis.k(ell, s_in, mu)
    k[np.abs(s_in) > ell] = 0
    k[np.abs(s_in + mu) > ell] = 0
    return k / basis.radius


def _lap_symbol(basis, s):
    """Laplacian symbol (reference basis.py:3408-3419)."""
    ell = np.arange(basis.Lmax + 1)
    k = SphereBasis.k
    k_lap = k(ell, s + 1, -1) * k(ell, s, +1) + k(ell, s - 1, +1) * k(ell, s, -1)
    k_lap[np.abs(s) > ell] = 0
    return k_lap / basis.radius**2


def _spins(basis, operand):
    return [int(s) for s in basis.spin_weights(operand.tensorsig).reshape(-1)]


def diag_linear(e, basis, is_leaf):
    """Lower an expression built from operators that are DIAGONAL in (m, l) -- gradient, divergence, Laplacian, skew, sums
    and numeric factors -- over leaves accepted by `is_leaf`.  Returns one list per output component of terms
    (leaf, leaf component, complex coefficient, real symbol over l = 0 .. Lmax)."""
    from . import operators as ops
    ones = np.ones(basis.Lmax + 1)
    if is_leaf(e):
        return [[(e, c, 1.0 + 0j, ones)] for c in range(max(e.ncomp, 1))]
    if isinstance(e, ops.Add):
        out = None
        for a in e.args:
            if not isinstance(a, ops.Operand):
                raise NotImplementedError("numbers added to sphere fields")
            sub = diag_linear(a, basis, is_leaf)
            out = sub if out is None else [x + y for x, y in zip(out, sub)]
        return out
    if isinstance(e, ops.ScalarMul):
        return [[(l, c, coef * e.c, sym) for l, c, coef, sym in terms] for terms in diag_linear(e.args[0], basis, is_leaf)]
    if isinstance(e, ops.Convert):
        return diag_linear(e.args[0], basis, is_leaf)
    if isinstance(e, ops.Gradient):
        A = e.args[0]
        sub = diag_linear(A, basis, is_leaf)
        sp = _spins(basis, A)
        out = []
        for mu in e.cs.spin_ordering:
            for ca, terms in enumerate(sub):
                sym = _grad_symbol(basis, sp[ca], mu)
                out.append([(l, c, coef, s0 * sym) for l, c, coef, s0 in terms])
        return out
    if isinstance(e, ops.Divergence):
        A = e.args[0]
        sub = diag_linear(A, basis, is_leaf)
        sp = _spins(basis, A)
        nrest = len(sub) // 2
        out = [[] for _ in range(nrest)]
        for i, sigma in enumerate(e.cs.spin_ordering):
            for r in range(nrest):
                ca = i * nrest + r
                sym = _grad_symbol(basis, sp[ca], -sigma)
                out[r].extend((l, c, coef, s0 * sym) for l, c, coef, s0 in sub[ca])
        return out
    if isinstance(e, ops.Laplacian):
        A = e.args[0]
        sub = diag_linear(A, basis, is_leaf)
        sp = _spins(basis, A)
        return [[(l, c, coef, s0 * _lap_symbol(basis, sp[ca])) for l, c, coef, s0 in terms] for ca, terms in enumerate(sub)]
    if isinstance(e, ops.Skew):
        if e.index != 0:
            raise NotImplementedError("Skew along index 0 only")
        sub = diag_linear(e.args[0], basis, is_leaf)
        nrest = len(sub) // 2
        out = []
        for i, sigma in enumerate(e.cs.spin_ordering):            # spin components are multiplied by sigma * 1j
            for r in range(nrest):
                out.append([(l, c, coef * (1j * sigma), s0) for l, c, coef, s0 in sub[i * nrest + r]])
        return out
    raise NotImplementedError(f"{type(e).__name__} is not a separable sphere operator")


def lhs_blocks(e, variables, basis, m):
    """{time-derivative order: {(out comp, variable index, variable comp): complex sparse matrix over l = m .. Lmax}} of an
    expression linear in the problem variables, for azimuthal wavenumber m (reference subproblem_matrix of the separable
    sphere operators, operators.py:2758-2800, SpinSkew 2133-2148, and of MulCosine, 2936-2968 / 3036-3050)."""
    from . import operators as ops
    from scipy import sparse
    NL = basis.Lmax + 1 - m
    ell = slice(m, basis.Lmax + 1)

    def scale(blocks, f):
        return {t: {k: f(k, B) for k, B in d.items()} for t, d in blocks.items()}

    def constant(x):
        return all(b is None for b in x.bases)
    E00 = sparse.csr_matrix(([1.0 + 0j], ([0], [0])), shape=(NL, NL))       # the (l = 0) -> (l = 0) entry, wavenumber 0 only

    def rec(e):
        for iv, v in enumerate(variables):
            if e is v:
                if constant(v):
                    # a constant unknown lives in the (m = 0, l = 0) cosine coefficient (LBVP gauge constants: "+ c", "ave(h) = 0")
                    if v.tensorsig:
                        raise NotImplementedError("constant tensor unknowns in sphere problems")
                    return {0: {(0, iv, 0): E00}} if m == 0 else {}
                return {0: {(c, iv, c): sparse.identity(NL, dtype=complex, format='csr') for c in range(max(v.ncomp, 1))}}
        if isinstance(e, ops.Add):
            out = {}
            for a in e.args:
                if not isinstance(a, ops.Operand):
                    raise ValueError("LHS must be homogeneous in the variables")
                # constant + sphere field: the constant is converted, unit amplitude 1 / constant_mode_value = sqrt(2)
                # (reference ConvertConstantSphere.symbol, basis.py:3293-3296)
                lift = np.sqrt(2.0) if (constant(a) and not constant(e)) else 1.0
                for t, d in rec(a).items():
                    o = out.setdefault(t, {})
                    for k, B in d.items():
                        B = B * lift if lift != 1.0 else B
                        o[k] = o[k] + B if k in o else B
            return out
        if isinstance(e, ops.Integrate):
            if not (e.average and sphere_basis_of(e.args[0]) is not None and not e.args[0].tensorsig):
                raise NotImplementedError("only ave(scalar sphere field) is supported on the LHS of sphere problems")
            if m != 0:
                return {}
            # reference SphereAverage.symbol (basis.py:5315-5317): 1 at l = 0, the l = 0 coefficient passes through
            return {t: {k: E00 @ B for k, B in d.items()} for t, d in rec(e.args[0]).items()}
        if isinstance(e, ops.ScalarMul):
            return scale(rec(e.args[0]), lambda k, B: B * e.c)
        if isinstance(e, ops.Convert):
            return rec(e.args[0])
        if isinstance(e, ops.TimeDerivative):
            return {t + 1: d for t, d in rec(e.args[0]).items()}
        A = e.args[0] if getattr(e, 'args', None) else None
        if isinstance(e, (ops.Gradient, ops.Divergence, ops.Laplacian, ops.Skew, ops.MulCosine)):
            sub = rec(A)
            sp = _spins(basis, A)
            na = len(sp)
            out = {}
            for t, d in sub.items():
                o = out.setdefault(t, {})

                def put(co, iv, ci, B):
                    key = (co, iv, ci)
                    o[key] = o[key] + B if key in o else B
                for (ca, iv, ci), B in d.items():
                    if isinstance(e, ops.Gradient):
                        for i, mu in enumerate(e.cs.spin_ordering):
                            put(i * na + ca, iv, ci, sparse.diags(_grad_symbol(basis, sp[ca], mu)[ell]) @ B)
                    elif isinstance(e, ops.Divergence):
                        nrest = na // 2
                        i, r = divmod(ca, nrest)
                        put(r, iv, ci, sparse.diags(_grad_symbol(basis, sp[ca], -e.cs.spin_ordering[i])[ell]) @ B)
                    elif isinstance(e, ops.Laplacian):
                        put(ca, iv, ci, sparse.diags(_lap_symbol(basis, sp[ca])[ell]) @ B)
                    elif isinstance(e, ops.Skew):
                        nrest = na // 2
                        put(ca, iv, ci, (1j * e.cs.spin_ordering[ca // nrest]) * B)
                    else:   # MulCosine
                        Cm, Lmin = basis.cos_matrix(m, sp[ca])
                        if Cm is None:
                            continue
                        full = sparse.lil_matrix((NL, NL))
                        full[Lmin - m:, Lmin - m:] = Cm
                        put(ca, iv, ci, full.tocsr() @ B)
            return out
        raise NotImplementedError(f"{type(e).__name__} is not supported on the LHS of sphere problems")

    return rec(e)


class SphereSystems:
    """Per-m banded pencil systems of a sphere IVP on the device, behind the interface the IMEX loops of
    dedalus_b200/solvers.py use (move / matvec / solve / factor_verified), served by csrc/banded.cu.

    Unknowns of the system of wavenumber m: index ((l - m) * NC + component) * 2 + part, components of all variables in
    order, part 0 / 1 = cos / -sin coefficient.  A complex operator entry a becomes the real block [[Re a, -Im a], [Im a, Re a]]
    (reference: cos / -sin expansion of SpinSkew, operators.py:2141-2147).  Modes that do not exist (l < |s|, the -sin part of
    l = 0) keep a unit diagonal and a zero right-hand side."""

    VERIFY_TOL = 1e-10

    def __init__(self, solver, nslots, nlu):
        import torch
        from .lib import BandedSys
        self.solver = solver
        problem = solver.problem
        basis = next(b for b in map(sphere_basis_of, problem.variables) if b is not None)
        self.basis = basis
        dev = solver.device
        variables = problem.variables
        Lmax = basis.Lmax
        var_comps = [(iv, c) for iv, v in enumerate(variables) for c in range(max(v.ncomp, 1))]
        eq_comps = [(ie, c) for ie, eq in enumerate(problem.equations)
                    for c in range(max(int(np.prod([cs.dim for cs in eq['tensorsig']], dtype=int)), 1))]
        if len(var_comps) != len(eq_comps):
            raise ValueError("sphere problem: number of equation components differs from the number of unknown components")
        NC = len(var_comps)
        var_spin = [s for v in variables for s in (_spins(basis, v) or [0])]
        var_rank = [len(v.tensorsig) for v in variables for _ in range(max(v.ncomp, 1))]
        eq_spin = [s for eq in problem.equations for s in ([int(x) for x in basis.spin_weights(eq['tensorsig']).reshape(-1)] or [0])]
        eq_rank = [len(eq['tensorsig']) for eq in problem.equations
                   for _ in range(max(int(np.prod([cs.dim for cs in eq['tensorsig']], dtype=int)), 1))]
        var_base = np.cumsum([0] + [max(v.ncomp, 1) for v in variables])
        # constants (no bases): one number, carried by the (m = 0, l = 0) cosine slot of their component
        var_const = np.array([all(b is None for b in variables[iv].bases) for iv, c in var_comps])
        eq_const = np.array([all(b is None for b in problem.equations[ie]['bases']) for ie, c in eq_comps])
        dist = solver.dist
        if (var_const.any() or eq_const.any()) and dist.size > 1:
            raise NotImplementedError("constant unknowns / equations of sphere problems are single-GPU in this build")
        j0, j1 = basis.local_pairs(dist)
        plane = 2 * (j1 - j0) * basis.coeff_shape[1]                 # the rank's block of the coefficient packing
        var_off = [solver.var_arena.offsets[iv] + c * plane for iv, c in var_comps]
        eq_off = [solver.eq_arena.offsets[ie] + c * plane for ie, c in eq_comps]
        ms = sorted(m for m, _ in basis.local_wavenumbers(dist) if m <= Lmax)       # the wavenumbers of this rank's pairs
        systems = []
        kband = 0
        total_valid = 0
        for m in ms:
            NL = Lmax + 1 - m
            n = NL * NC * 2
            rows_, cols_, vals = {0: [], 1: []}, {0: [], 1: []}, {0: [], 1: []}
            for ie, eq in enumerate(problem.equations):
                blocks = lhs_blocks(eq['LHS'], variables, basis, m)
                if any(t > 1 for t in blocks):
                    raise NotImplementedError("Only first-order time derivatives are supported.")
                eq_c0 = sum(1 for q in eq_comps if q[0] < ie)
                for t, d in blocks.items():
                    for (co, iv, ci), B in d.items():
                        B = B.tocoo()
                        R = (B.row * NC + eq_c0 + co) * 2
                        Cc = (B.col * NC + int(var_base[iv]) + ci) * 2
                        re, im = B.data.real, B.data.imag
                        rows_[t] += [R, R, R + 1, R + 1]; cols_[t] += [Cc, Cc + 1, Cc, Cc + 1]; vals[t] += [re, -im, im, re]
            lidx = np.arange(n) // (2 * NC) + m
            comp = (np.arange(n) // 2) % NC
            part = np.arange(n) % 2
            def validity(spin, rank, const):
                sp = np.asarray(spin)[comp]; rk = np.asarray(rank)[comp]
                ok = (lidx >= np.maximum(m, np.abs(sp))) & ~((lidx == 0) & (part == 1) & (rk <= 1))
                return ok & ~(const[comp] & ~((lidx == 0) & (part == 0)))
            vcol, vrow = validity(var_spin, var_rank, var_const), validity(eq_spin, eq_rank, eq_const)
            if not np.array_equal(vcol, vrow):
                raise NotImplementedError("equations and variables of a sphere problem must pair up component by component")
            mats = {}
            from scipy import sparse
            for t in (0, 1):
                if rows_[t]:
                    A = sparse.coo_matrix((np.concatenate(vals[t]), (np.concatenate(rows_[t]), np.concatenate(cols_[t]))), shape=(n, n)).tocsr()
                else:
                    A = sparse.csr_matrix((n, n))
                D = sparse.diags(vrow.astype(float))
                A = (D @ A @ D).tocsr()
                A.data[np.abs(A.data) < solver.entry_cutoff] = 0
                A.eliminate_zeros()
                mats[t] = A
            mats[0] = (mats[0] + sparse.diags((~vrow).astype(float))).tocsr()       # L: unit diagonal on the missing modes
            for A in mats.values():
                coo = A.tocoo()
                if coo.nnz:
                    kband = max(kband, int(np.abs(coo.row - coo.col).max()))
            # arena positions of the unknowns / equation rows
            j, cols = basis.mode_columns(m)
            col_of = cols[lidx - m]
            pos = (2 * (j - j0) + part) * basis.coeff_shape[1] + col_of
            xi = np.where(vcol, np.asarray(var_off)[comp] + np.where(var_const[comp], 0, pos), -1)
            fi = np.where(vrow, np.asarray(eq_off)[comp] + np.where(eq_const[comp], 0, pos), -1)
            systems.append(dict(m=m, n=n, L=mats[0], M=mats[1], xi=xi, fi=fi))
            total_valid += int(vcol.sum())
        self.total_modes = total_valid
        self.kl = self.ku = kl = ku = max(kband, 1)
        ld0, ldf = kl + ku + 1, 2 * kl + ku + 1
        arr = (BandedSys * len(systems))()
        op_off = lu_off = vec_off = 0
        for i, s in enumerate(systems):
            a = arr[i]
            a.n, a.nrhs, a.op_off, a.lu_off, a.piv_off, a.vec_off = s['n'], 1, op_off, lu_off, vec_off, vec_off
            s['op_off'], s['vec_off'] = op_off, vec_off
            op_off += s['n'] * ld0; lu_off += s['n'] * ldf; vec_off += s['n']
        self.nsys, self.nvec, self.nlu_size, self.max_n = len(systems), vec_off, lu_off, max(s['n'] for s in systems)
        M_ab, L_ab = np.zeros(op_off), np.zeros(op_off)
        for s in systems:
            for name, ab in (('M', M_ab), ('L', L_ab)):
                coo = s[name].tocoo()
                ab[s['op_off'] + coo.col.astype(np.int64) * ld0 + (ku + coo.row - coo.col)] = coo.data
        t64 = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
        self.M_ab, self.L_ab = t64(M_ab), t64(L_ab)
        self.desc = torch.from_numpy(np.frombuffer(bytes(arr), dtype=np.uint8).copy()).to(dev)
        self.idx = [t64(np.concatenate([s['xi'] for s in systems]).astype(np.int64)),
                    t64(np.concatenate([s['fi'] for s in systems]).astype(np.int64))]
        self.systems = systems
        self.vecs = [torch.zeros(self.nvec, dtype=torch.float64, device=dev) for _ in range(nslots)]
        self.lu = [torch.zeros(self.nlu_size, dtype=torch.float64, device=dev) for _ in range(nlu)]
        self.ipiv = [torch.zeros(self.nvec, dtype=torch.int32, device=dev) for _ in range(nlu)]
        self.info = torch.zeros(self.nsys, dtype=torch.int32, device=dev)
        self.reorders = 0
        self.last_verify = None
        self.sum_band = op_off

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
        with Timed(self.solver.prof, "pencil_matvec", 8 * (self.sum_band * ((ym_slot >= 0) + (yl_slot >= 0)) + 3 * self.nvec)):
            self._call("db_banded_matvec", self.desc.data_ptr(), self.nsys, self.kl, self.ku, self.M_ab.data_ptr(), self.L_ab.data_ptr(),
                       self.vecs[x_slot].data_ptr(), ym, yl)

    def solve(self, lu_slot, x_slot, terms):
        import ctypes as C
        from .lib import VecComb
        from .solvers import Timed
        vc = VecComb()
        vc.nvec = len(terms)
        for k, (slot, coef) in enumerate(terms):
            vc.vec[k] = self.vecs[slot].data_ptr(); vc.coef[k] = coef
        ldf = 2 * self.kl + self.ku + 1
        with Timed(self.solver.prof, "pencil_solve", 8 * (self.nvec * ldf + self.nvec * (len(terms) + 1))):
            self._call("db_banded_solve", self.desc.data_ptr(), self.nsys, self.kl, self.ku, self.max_n, 1, self.lu[lu_slot].data_ptr(),
                       self.ipiv[lu_slot].data_ptr(), C.byref(vc), self.vecs[x_slot].data_ptr())

    def factor(self, lu_slot, a0, b0):
        self._call("db_banded_combine", self.desc.data_ptr(), self.nsys, self.kl, self.ku, float(a0), self.M_ab.data_ptr(), float(b0),
                   self.L_ab.data_ptr(), self.lu[lu_slot].data_ptr())
        self._call("db_banded_factor", self.desc.data_ptr(), self.nsys, self.kl, self.ku, self.lu[lu_slot].data_ptr(),
                   self.ipiv[lu_slot].data_ptr(), self.info.data_ptr())

    def check_info(self):
        from .lib import DedalusB200Error
        bad = int((self.info != 0).sum().item())
        if bad:
            raise DedalusB200Error(f"{bad} sphere pencil systems hit a zero / non-finite pivot during factorisation.")

    def factor_verified(self, lhs, slots):
        """Factorise a0 M + b0 L into each slot; backward error of a probe solve per factorisation (partial pivoting is
        stable, so this is a sanity check, not a safety net as in the Cartesian static-order path)."""
        import torch
        from .lib import DedalusB200Error
        s_b, s_x, s_m, s_l = slots
        worst = 0.0
        for lu_slot, a0, b0 in lhs:
            for attempt in range(3):
                self.factor(lu_slot, a0, b0)
                self.check_info()
                gen = torch.Generator(device=self.solver.device); gen.manual_seed(1234)
                self.vecs[s_b].normal_(generator=gen)
                self.solve(lu_slot, s_x, [(s_b, 1.0)])
                self.matvec(s_x, s_m, s_l)
                b, mx, lx = self.vecs[s_b], self.vecs[s_m], self.vecs[s_l]
                r = float((a0 * mx + b0 * lx - b).abs().max() / (b.abs().max() + (a0 * mx).abs().max() + (b0 * lx).abs().max()))
                if r <= self.VERIFY_TOL:
                    break
                import warnings
                warnings.warn(f"sphere pencil factorisation: backward error {r:.2e} on attempt {attempt + 1}; factorising again")
                self.reorders += 1
            worst = max(worst, r)
        self.last_verify = worst
        if not worst <= self.VERIFY_TOL:
            raise DedalusB200Error(f"sphere pencil factorisation failed verification: backward error {worst:.2e}")
        return worst


# ------------------------------------------------------------------------------------------------------------
# Right-hand sides: post-linear( polynomial( grid values of pre-linear(state) ) )
# ------------------------------------------------------------------------------------------------------------
class SphereRHSPlan:
    """Compiled evaluation of all equation right-hand sides of a sphere IVP into the equation arena (reference:
    Evaluator.evaluate_handlers walking the operator tree, core/evaluator.py:95-146).  Stages, all on the device:
      1. PRE   one db_pair_lincomb: every grid operand (a separable operator chain over state fields: u, grad(u), h, ...) in
               coefficient space, components grouped by spin weight
      2. colatitude transforms backward, ONE launch per spin weight for all operands of that weight
      3. spin -> component recombination of all operands in one db_pair_lincomb; azimuthal FFT backward of all components
      4. one pointwise kernel for all products (csrc/pointwise.cu)
      5. azimuthal FFT forward, component -> spin recombination, colatitude transforms forward per spin weight
      6. POST  one db_pair_lincomb: the separable operators outside the products (-1, -div, ...) written straight into the
               equation arena."""

    def __init__(self, solver):
        import torch
        from . import operators as ops
        from .field import Field
        self.solver = solver
        problem = solver.problem
        dev = solver.device
        basis = self.basis = next(b for b in map(sphere_basis_of, problem.variables) if b is not None)
        variables = problem.variables
        dist = self.dist = solver.dist
        ax = dist.get_basis_axis(basis)
        self.scales = tuple(basis.dealias)
        gfull = basis.grid_shape(self.scales)
        P = dist.size
        self.gshape = (gfull[0], gfull[1] // P)                      # colatitude is distributed on the grid
        self.Ngt_full = gfull[1]
        j0, j1 = basis.local_pairs(dist)
        self.Nc0 = 2 * (j1 - j0)
        self.rowsA = 2 * len(basis.local_wavenumbers(dist))
        plane_c = self.Nc0 * basis.coeff_shape[1]
        # sources of the grid operands: problem variables are read in place from the state arena (IVPs); any other sphere field
        # (LBVP right-hand sides: e.g. the velocity in the balance equation of the stock shallow-water script) is appended to a
        # source buffer that is refreshed before every evaluation
        state_comp0 = {}
        for iv, v in enumerate(variables):
            if sphere_basis_of(v) is not None:
                assert solver.var_arena.offsets[iv] % plane_c == 0
                state_comp0[id(v)] = solver.var_arena.offsets[iv] // plane_c
        self.extra_sources = []
        self.use_state = getattr(solver, 'rhs_reads_state', True)
        if not self.use_state:
            state_comp0 = {}

        def is_state(e):
            if not (isinstance(e, Field) and sphere_basis_of(e) is not None):
                return False
            if id(e) not in state_comp0:
                base = (len(solver.state_t) // plane_c if self.use_state else 0) + sum(max(f.ncomp, 1) for f in self.extra_sources)
                state_comp0[id(e)] = base
                self.extra_sources.append(e)
            return True
        nonlinear = (ops.Multiply, ops.DotProduct, ops.Power, ops.MulCosine)
        cos_id = [None]

        operands, operand_ids = [], {}        # grid operands: (expr, comps range start, spins, rank)
        n_gcomp = [0]

        def grid_operand(e):
            if id(e) not in operand_ids:
                terms = diag_linear(e, basis, is_state)
                spins = _spins(basis, e) or [0]
                operand_ids[id(e)] = len(operands)
                operands.append(dict(expr=e, terms=terms, spins=spins, rank=len(e.tensorsig), g0=n_gcomp[0]))
                n_gcomp[0] += len(spins)
            return operands[operand_ids[id(e)]]

        def poly(e):
            """{component: [(coef, (grid input ids...))]} of a grid-space polynomial expression (coordinate components)."""
            if isinstance(e, ops.Multiply):
                A, B = e.args
                ra, rb = poly(A), poly(B)
                nb = max(B.ncomp, 1)
                return {ca * nb + cb: [(x * y, fx + fy) for x, fx in ta for y, fy in tb] for ca, ta in ra.items() for cb, tb in rb.items()}
            if isinstance(e, ops.DotProduct):
                A, B = e.args
                ra, rb = poly(A), poly(B)
                d = A.tensorsig[-1].dim
                na, nb = A.ncomp // d, B.ncomp // d
                return {ia * nb + ib: [(x * y, fx + fy) for i in range(d) for x, fx in ra[ia * d + i] for y, fy in rb[i * nb + ib]]
                        for ia in range(na) for ib in range(nb)}
            if isinstance(e, ops.Power):
                base = poly(e.args[0])[0]
                cur = base
                for _ in range(e.n - 1):
                    cur = [(x * y, fx + fy) for x, fx in cur for y, fy in base]
                return {0: cur}
            if isinstance(e, ops.MulCosine):
                # on the right-hand side cos(theta) X is formed on the dealiased grid (exact: the product raises the degree by
                # one and the forward transform truncates at Lmax, as the reference's truncated operator matrix does)
                if cos_id[0] is None:
                    cos_id[0] = -1                      # resolved to the last grid input once all operands are known
                return {c: [(x, f + ('cos',)) for x, f in t] for c, t in poly(e.args[0]).items()}
            if isinstance(e, ops.Add) and any(_has(a, nonlinear) for a in e.args if isinstance(a, ops.Operand)):
                out = {}
                for a in e.args:
                    for c, t in poly(a).items():
                        out.setdefault(c, []).extend(t)
                return out
            if isinstance(e, ops.ScalarMul) and _has(e.args[0], nonlinear):
                return {c: [(x * e.c, f) for x, f in t] for c, t in poly(e.args[0]).items()}
            if _has(e, nonlinear):
                raise NotImplementedError("operators applied to products inside products on the RHS of sphere problems")
            op = grid_operand(e)
            return {c: [(1.0, (op['g0'] + c,))] for c in range(len(op['spins']))}

        products, product_ids = [], {}
        n_pcomp = [0]

        def product(e):
            if id(e) not in product_ids:
                spins = _spins(basis, e) or [0]
                product_ids[id(e)] = len(products)
                products.append(dict(expr=e, poly=poly(e), spins=spins, rank=len(e.tensorsig), p0=n_pcomp[0]))
                n_pcomp[0] += len(spins)
            return products[product_ids[id(e)]]

        # leaves of the separable operators outside: products, or plain sphere fields (right-hand sides linear in a field, "skew(f)",
        # "f + MulCosine(f)": carried through the grid like a one-factor product)
        is_product = lambda e: isinstance(e, nonlinear) or is_state(e)
        self.post_rows = []
        const_seen = False
        for eq in problem.equations:
            ncomp = max(int(np.prod([cs.dim for cs in eq['tensorsig']], dtype=int)), 1)
            rhs = eq['RHS']
            if all(b is None for b in eq['bases']):
                # constant equations ("ave(h) = 0") sit behind the sphere equations in the arena and keep a zero right-hand side
                if isinstance(rhs, ops.Operand) or rhs != 0:
                    raise NotImplementedError("constant equations of sphere problems need a zero right-hand side")
                const_seen = True
                continue
            if const_seen:
                raise NotImplementedError("constant equations must follow the sphere equations")
            if not isinstance(rhs, ops.Operand):
                if rhs != 0:
                    raise NotImplementedError("nonzero numeric right-hand sides on the sphere")
                self.post_rows += [[] for _ in range(ncomp)]
                continue
            rows = diag_linear(rhs, basis, is_product)
            for terms in rows:
                self.post_rows.append([(product(leaf)['p0'] + c, coef, sym) for leaf, c, coef, sym in terms])
        self.operands, self.products = operands, products
        self.n_g, self.n_p = n_gcomp[0], n_pcomp[0]
        self.has_cos = cos_id[0] is not None
        if self.has_cos:                                  # cos(theta) rides as one more grid input
            for pr in products:
                pr['poly'] = {c: [(x, tuple(self.n_g if q == 'cos' else q for q in f)) for x, f in t] for c, t in pr['poly'].items()}
            self.n_g += 1
        if self.n_p == 0:
            self.trivial = True
            return
        self.trivial = False
        # ---- symbol table on the coefficient packing: sym[l] -> (npair, ncol) array
        _, ell_map = basis.elements_to_groups()
        ell_pairs = ell_map[0::2][j0:j1]
        in_range = ell_pairs <= basis.Lmax
        sym_arrays, sym_index = [], {}

        def sym_off(sym):
            if np.all(sym == 1):
                return -1
            key = sym.tobytes()
            if key not in sym_index:
                sym_index[key] = len(sym_arrays) * ell_pairs.size
                sym_arrays.append(np.where(in_range, sym[np.minimum(ell_pairs, basis.Lmax)], 0.0).ravel())
            return sym_index[key]
        # ---- stage 1: PRE program, outputs grouped by spin weight
        order = sorted(((s, o, c) for o, op in enumerate(operands) for c, s in enumerate(op['spins'])), key=lambda t: t[0])
        self.pre_spins = [t[0] for t in order]
        slot_of = {(o, c): i for i, (s, o, c) in enumerate(order)}
        pre_rows = []
        for s, o, c in order:
            pre_rows.append([(state_comp0[id(leaf)] + lc, coef, sym_off(sym)) for leaf, lc, coef, sym in operands[o]['terms'][c]])
        post_rows = [[(src, coef, sym_off(sym)) for src, coef, sym in terms] for terms in self.post_rows]
        syms = torch.from_numpy(np.concatenate(sym_arrays) if sym_arrays else np.zeros(1)).to(dev)
        self.pre = PairProgram(pre_rows, dev, syms)
        # ---- stage 3: backward recombination, spin-grouped slots -> operand-major coordinate components
        rec_rows = []
        for o, op in enumerate(operands):
            U = S2Coordinates.U_backward(op['rank']) if op['rank'] else np.ones((1, 1))
            for i in range(len(op['spins'])):
                rec_rows.append([(slot_of[(o, j)], U[i, j], -1) for j in range(len(op['spins'])) if U[i, j] != 0])
        self.rec_b = PairProgram(rec_rows, dev)
        # ---- stage 4: pointwise program
        coef, fac_ptr, fac, term_ptr = [], [0], [], [0]
        for pr in products:
            for c in range(len(pr['spins'])):
                for x, f in pr['poly'].get(c, []):
                    if x == 0:
                        continue
                    coef.append(float(x)); fac.extend(f); fac_ptr.append(len(fac))
                term_ptr.append(len(coef))
        self.npoints = int(np.prod(self.gshape))
        i32 = lambda a: torch.from_numpy(np.asarray(a, dtype=np.int32)).to(dev)
        self.term_ptr, self.fac_ptr, self.fac = i32(term_ptr), i32(fac_ptr), i32(fac if fac else [0])
        self.coef = torch.from_numpy(np.asarray(coef if coef else [0.0], dtype=np.float64)).to(dev)
        self.nfac = len(fac)
        nf = np.diff(fac_ptr)
        self.pairs = None
        if len(coef) and nf.min() >= 1 and nf.max() <= 2 and self.npoints % 2 == 0 and 2 * self.n_g * 128 * 16 <= 227 * 1024:
            rec = np.zeros(len(coef), dtype=np.dtype([('coef', '<f8'), ('a', '<i4'), ('b', '<i4')]))      # db_pair_term
            rec['coef'] = coef
            rec['a'] = [fac[fac_ptr[t]] for t in range(len(coef))]
            rec['b'] = [fac[fac_ptr[t] + 1] if nf[t] == 2 else -1 for t in range(len(coef))]
            self.pairs = torch.from_numpy(np.frombuffer(rec.tobytes(), dtype=np.uint8).copy()).to(dev)
        # ---- stage 5: forward recombination, product-major coordinate components -> spin-grouped slots
        forder = sorted(((s, p, c) for p, pr in enumerate(products) for c, s in enumerate(pr['spins'])), key=lambda t: t[0])
        self.post_spins = [t[0] for t in forder]
        fslot = {(p, c): i for i, (s, p, c) in enumerate(forder)}
        rec_rows = []
        for s, p, c in forder:
            pr = products[p]
            U = S2Coordinates.U_forward(pr['rank']) if pr['rank'] else np.ones((1, 1))
            rec_rows.append([(pr['p0'] + j, U[c, j], -1) for j in range(len(pr['spins'])) if U[c, j] != 0])
        self.rec_f = PairProgram(rec_rows, dev)
        # ---- stage 6: POST program reads the spin-grouped forward results
        remap = {pr['p0'] + c: fslot[(p, c)] for p, pr in enumerate(products) for c in range(len(pr['spins']))}
        self.post = PairProgram([[(remap[src], coef, so) for src, coef, so in terms] for terms in post_rows], dev, syms)
        # ---- buffers
        Nc0, Nc1 = self.Nc0, basis.coeff_shape[1]
        Ngp, tb = self.gshape
        Ngt, rowsA = self.Ngt_full, self.rowsA
        z = lambda *shape: torch.zeros(shape, dtype=torch.float64, device=dev)
        n_t = self.n_g - (1 if self.has_cos else 0)          # transformed operands (the cos(theta) plane is static)
        self.n_t = n_t
        self.c_pre, self.cg_a, self.cg_b = z(n_t, Nc0, Nc1), z(n_t, rowsA, Ngt), z(n_t, rowsA, Ngt)
        self.g_in, self.g_out = z(self.n_g, Ngp, tb), z(self.n_p, Ngp, tb)
        if self.has_cos:
            theta = basis.global_grid_colatitude(self.scales[1])[dist.grid_local_slice(ax + 1, basis, self.scales[1])]
            self.g_in[n_t] = torch.from_numpy(np.ascontiguousarray(np.broadcast_to(np.cos(theta)[None, :], (Ngp, tb)))).to(dev)
        self.pg_a, self.pg_b, self.c_post = z(self.n_p, basis.shape[0], tb), z(self.n_p, rowsA, Ngt), z(self.n_p, Nc0, Nc1)

    def set_static(self, eq_t):
        eq_t.zero_()

    @staticmethod
    def _groups(spins):
        c = 0
        while c < len(spins):
            c1 = c
            while c1 < len(spins) and spins[c1] == spins[c]:
                c1 += 1
            yield spins[c], c, c1
            c = c1

    def evaluate(self, eq_t):
        from .lib import get_lib, current_stream
        from .solvers import Timed
        if self.trivial:
            eq_t.zero_()
            return
        basis, solver, dist = self.basis, self.solver, self.dist
        prof = solver.prof
        Nc0, Nc1 = self.Nc0, basis.coeff_shape[1]
        Ngp, tb = self.gshape
        Ngt, rowsA = self.Ngt_full, self.rowsA
        multi = dist.size > 1
        npair_c, npair_a = Nc0 // 2, rowsA // 2
        src = solver.state_t
        if self.extra_sources:                 # fields that are not problem variables: appended behind (or instead of) the state arena
            import torch
            for f in self.extra_sources:
                f.change_layout('c')
            parts = ([solver.state_t] if self.use_state else []) + [f.device_data().reshape(-1) for f in self.extra_sources]
            src = torch.cat(parts)
        with Timed(prof, "sphere_symbols", 8 * Nc0 * Nc1 * (self.n_g + len(src) // (Nc0 * Nc1))):
            self.pre.apply(src, self.c_pre, npair_c, Nc1)
        for s, c0, c1 in self._groups(self.pre_spins):
            plan = basis.colatitude_plan(Ngt, s, dist)
            with Timed(prof, "swsh_backward", plan.matrix_bytes() + 8 * (c1 - c0) * (Nc0 * Nc1 + rowsA * Ngt)):
                plan.backward(self.c_pre[c0:c1], self.cg_a[c0:c1], 2)
        with Timed(prof, "spin_recombine", 16 * self.cg_a.numel()):
            self.rec_b.apply(self.cg_a, self.cg_b, npair_a, Ngt)
        cgB = self.cg_b
        if multi:
            with Timed(prof, "sphere_transpose", 16 * self.cg_b.numel()):
                cgB = basis.hop(dist).to_grid_side(self.cg_b.unsqueeze(-1)).squeeze(-1).contiguous()
        with Timed(prof, "azimuth_backward", 8 * (cgB.numel() + self.g_in.numel())):
            basis.azimuth_plan(Ngp).backward(cgB, self.g_in[:self.n_t], 1)
        with Timed(prof, "pointwise", 8 * self.npoints * (self.n_g + self.n_p)):
            if self.pairs is not None and self.g_in.data_ptr() % 16 == 0 and self.g_out.data_ptr() % 16 == 0:
                get_lib().call("db_pointwise_pairs", self.g_in.data_ptr(), self.g_out.data_ptr(), self.npoints, self.n_g, self.n_p,
                               self.term_ptr.data_ptr(), self.pairs.data_ptr(), current_stream())
            else:
                get_lib().call("db_pointwise", self.g_in.data_ptr(), self.g_out.data_ptr(), self.npoints, self.n_g, self.n_p,
                               self.term_ptr.data_ptr(), self.coef.data_ptr(), self.fac_ptr.data_ptr(), self.fac.data_ptr(), self.nfac, current_stream())
        with Timed(prof, "azimuth_forward", 8 * (self.g_out.numel() + self.pg_a.numel())):
            basis.azimuth_plan(Ngp).forward(self.g_out, self.pg_a, 1)
        pgA = self.pg_a
        if multi:
            with Timed(prof, "sphere_transpose", 16 * self.pg_a.numel()):
                pgA = basis.hop(dist).to_coeff_side(self.pg_a.unsqueeze(-1)).squeeze(-1).contiguous()
        with Timed(prof, "spin_recombine", 16 * pgA.numel()):
            self.rec_f.apply(pgA, self.pg_b, npair_a, Ngt)
        for s, c0, c1 in self._groups(self.post_spins):
            plan = basis.colatitude_plan(Ngt, s, dist)
            with Timed(prof, "swsh_forward", plan.matrix_bytes() + 8 * (c1 - c0) * (Nc0 * Nc1 + rowsA * Ngt)):
                plan.forward(self.pg_b[c0:c1], self.c_post[c0:c1], 2)
        n_eq = len(self.post_rows)
        with Timed(prof, "sphere_symbols", 8 * Nc0 * Nc1 * (self.n_p + n_eq)):
            self.post.apply(self.c_post, eq_t, npair_c, Nc1)


def _has(e, types):
    from . import operators as ops
    if isinstance(e, types):
        return True
    return any(_has(a, types) for a in getattr(e, 'args', []) if isinstance(a, ops.Operand))


def evaluate_linear_expression(expr):
    """Evaluate an expression built from separable sphere operators (gradient, divergence, Laplacian, skew, sums, numeric
    factors) of fields into a new Field in coefficient space: one db_pair_lincomb launch (analysis tasks such as the vorticity
    -div(skew(u)) of the stock shallow-water script; reference: Future.evaluate, core/future.py:149-206)."""
    import torch
    from .field import Field
    basis = sphere_basis_of(expr)
    dist = expr.dist
    is_field = lambda e: isinstance(e, Field)
    rows = diag_linear(expr, basis, is_field)
    leaves, comp0 = [], {}
    for terms in rows:
        for leaf, c, coef, sym in terms:
            if id(leaf) not in comp0:
                comp0[id(leaf)] = sum(max(l.ncomp, 1) for l in leaves)
                leaves.append(leaf)
    j0, j1 = basis.local_pairs(dist)
    Nc0, Nc1 = 2 * (j1 - j0), basis.coeff_shape[1]
    for leaf in leaves:
        leaf.change_layout('c')
    dev = leaves[0].device_data().device
    src = torch.cat([l.device_data().reshape(max(l.ncomp, 1), Nc0, Nc1) for l in leaves], dim=0).contiguous()
    _, ell_map = basis.elements_to_groups()
    ell_pairs = ell_map[0::2][j0:j1]
    in_range = ell_pairs <= basis.Lmax
    sym_arrays, sym_index = [], {}

    def sym_off(sym):
        if np.all(sym == 1):
            return -1
        key = sym.tobytes()
        if key not in sym_index:
            sym_index[key] = len(sym_arrays) * ell_pairs.size
            sym_arrays.append(np.where(in_range, sym[np.minimum(ell_pairs, basis.Lmax)], 0.0).ravel())
        return sym_index[key]
    prog_rows = [[(comp0[id(leaf)] + c, coef, sym_off(sym)) for leaf, c, coef, sym in terms] for terms in rows]
    syms = torch.from_numpy(np.concatenate(sym_arrays) if sym_arrays else np.zeros(1)).to(dev)
    out = torch.empty((len(rows), Nc0, Nc1), dtype=torch.float64, device=dev)
    PairProgram(prog_rows, dev, syms).apply(src, out, Nc0 // 2, Nc1)
    result = Field(dist, bases=(basis,), tensorsig=expr.tensorsig, dtype=expr.dtype)
    dist._fields.pop()
    result.set_device_data(out.reshape(result.tshape + (Nc0, Nc1)), 'c')
    return result
