"""Shared bodies of the kernel-level tests of the spectral transforms: the real and complex Fourier and the Chebyshev transforms of
csrc/fft.cu (the generic shared-memory kernel k_fft) and csrc/rfft_regs.cu (the register-resident kernels, the blocked and peer
entries, and the fused x pass k_rfft_x_products), through the CPU emulation of the kernels (tests/test_emu_transform_kernels.py) and
on the GPU (tests/test_gpu_1e_transform_kernels.py).

The references are restated from the contract in include/dedalus_b200.h in np.longdouble, not from the kernels: transform matrices
built with exact integer angle reduction, 2 pi ((j k) mod n) / n.  Every output is compared componentwise against a bound propagated
stage by stage with absolute values,
    |got - ref| <= C_BOUND * (ceil(log2 n) + banded stages) * eps * (|F_s| ... |F_1| |x|),
where the factors of a fast transform all have entries of modulus <= 1, so that their product carries the input's 1-norm to every
output of the line (times the transform's scaling and derivative factors).  The register kernels transform two real lines as one
complex line, so a line's bound includes its partner's 1-norm (lines 2m and 2m + 1).  One constant C_BOUND serves the whole file;
the largest observed error / bound of every path is kept in RATIOS (printed by the test modules at the end of the session).
Entries whose reference is exactly zero (the sin(0) slot, modes past the truncation) must be exactly zero.

Besides random data, an impulse sweep per path puts a single unit coefficient (backward) or grid value (forward) in each line, so
that every mode's twiddle and derivative factor is checked on its own.  Outputs start as NaN, every gap the contract does not read
or write is NaN (padding between strided arrays, rows past the layout, the 8 bytes in front of a misaligned buffer), and afterwards
the gaps must still be NaN and the outputs finite.  Every case asserts which kernel served it (db_rfft_regs_launches)."""
import ctypes as C
import math
import os
import numpy as np
import pytest

EPS = np.finfo(np.float64).eps
LD = np.longdouble
PI = np.arccos(LD(-1))
C_BOUND = 2.0
RR_LINES = 16                       # csrc/rfft_regs.cu: lines per register tile (two per complex line, P = 8 pairs)
REG_N = (24, 48, 96, 192, 384, 768)  # register real-Fourier lengths (x products and Chebyshev: all but 768)
RATIOS = {}


def _note(path, ratio):
    RATIOS[path] = max(RATIOS.get(path, 0.0), float(ratio))


def report():
    return "\n".join(f"  {k:<44s} {v:.3g}" for k, v in sorted(RATIOS.items()))


def _lg(n):
    return max(1, math.ceil(math.log2(n)))


def _cs(num, den):
    """cos, sin of 2 pi num / den in long double, num reduced exactly modulo den first (integers)."""
    a = 2 * PI * LD(1) * (np.asarray(num, dtype=np.int64) % den).astype(LD) / LD(den)
    return np.cos(a), np.sin(a)


def _pair_sum(s):
    """s (..., lines): add the partner line's value (line l ^ 1 of the last axis; an unpaired last line keeps its own)."""
    s = np.asarray(s)
    out = s.copy()
    L = s.shape[-1]
    idx = np.arange(L) ^ 1
    ok = idx < L
    out[..., ok] += s[..., idx[ok]]
    return out


def _lines_last(x, layout):
    """(outer, rows, inner) -> (rows, lines) with line l = o * inner + i."""
    o, r, i = x.shape
    return np.moveaxis(x, 1, 0).reshape(r, o * i)


def _lines_back(y, outer, inner):
    return np.moveaxis(y.reshape(y.shape[0], outer, inner), 0, 1)


def check_bound(path, got, ref, bound, exact_zero=None):
    """got (float64), ref and bound (long double), same shape.  Records the largest error / bound under `path`."""
    got = np.asarray(got)
    assert np.isfinite(got).all(), (path, "non-finite output", np.argwhere(~np.isfinite(got))[:4])
    err = np.abs(got.astype(LD) - ref)
    zero = bound == 0
    if exact_zero is not None:
        zero = zero | exact_zero
    assert not np.any(got[zero] != 0), (path, "entries that must be exactly 0", np.argwhere(zero & (got != 0))[:6])
    nz = ~zero
    ratio = float((err[nz] / bound[nz]).max()) if nz.any() else 0.0
    _note(path, ratio)
    bad = np.argwhere(nz & (err > bound))
    assert ratio <= 1.0, (path, "error / bound", ratio, bad[:6])
    return ratio


# ------------------------------------------------------------------------------------------------------------------------------
# padded device buffers
# ------------------------------------------------------------------------------------------------------------------------------
class Padded:
    """A device buffer holding `data` (float64) with NaN gaps in front (`front` doubles: 2 keeps the data 16-byte aligned, 1 puts it
    8 bytes past a boundary) and behind (`tail` doubles).  .p = pointer to the data, .read() = (data, front gap, tail gap)."""

    def __init__(self, B, data, front=2, tail=37):
        self.B = B
        data = np.ascontiguousarray(data, dtype=np.float64)
        self.shape, self.front, self.tail = data.shape, front, tail
        h = np.full(front + data.size + tail, np.nan)
        h[front:front + data.size] = data.reshape(-1)
        self.d = B.dev_at(h, False)
        self.p = C.c_void_p(B.ptr(self.d).value + 8 * front)

    def read(self):
        h = self.B.host(self.d)
        n = int(np.prod(self.shape))
        return h[self.front:self.front + n].reshape(self.shape).copy(), h[:self.front], h[self.front + n:]

    def result(self, what):
        out, f, t = self.read()
        assert np.isnan(f).all() and np.isnan(t).all(), (what, "wrote outside the output")
        return out


def nan_output(B, shape, front=2):
    return Padded(B, np.full(shape, np.nan), front=front)


def regs_delta(B, fn):
    before = B.lib.rfft_regs_launches()
    fn()
    return B.lib.rfft_regs_launches() - before


def _set_env(name, value):
    old = os.environ.get(name)
    if value is None:
        os.environ.pop(name, None)
    else:
        os.environ[name] = str(value)
    return old


class env:
    """Context manager: environment variables set (value None: removed) for the duration."""

    def __init__(self, **kv):
        self.kv = kv

    def __enter__(self):
        self.old = {k: _set_env(k, v) for k, v in self.kv.items()}

    def __exit__(self, *a):
        for k, v in self.old.items():
            _set_env(k, v)


# ------------------------------------------------------------------------------------------------------------------------------
# real Fourier: cos / -sin interleaved, unit amplitude, Nyquist dropped
# ------------------------------------------------------------------------------------------------------------------------------
def rf_kmax(n, M):
    return min((n - 1) // 2, (M - 1) // 2)


def rf_backward_matrix(n, M, deriv=0, kscale=1.0):
    """(F, W): g = F c for one line, F (n, M) long double; W (M,) the magnitude each coefficient carries through the stages
    (|i k kscale|^deriv).  The sin(0) slot (column 1) and modes past Kmax are not read."""
    F = np.zeros((n, M), dtype=LD)
    W = np.zeros(M, dtype=LD)
    j = np.arange(n, dtype=np.int64)
    if deriv == 0:
        F[:, 0] = 1
        W[0] = 1
    for k in range(1, rf_kmax(n, M) + 1):
        f = (LD(k) * LD(kscale)) ** deriv
        # Re((a + i b) (i k)^d e^{i theta}) = a cos(theta + d pi / 2) - b sin(theta + d pi / 2)
        c, s = _cs(4 * j * k + deriv * n, 4 * n)
        F[:, 2 * k], W[2 * k] = f * c, f
        if 2 * k + 1 < M:                            # odd M: the last mode has no sin slot
            F[:, 2 * k + 1], W[2 * k + 1] = -f * s, f
    return F, W


def rf_forward_matrix(n, M):
    """(F, W): c = F g, F (M, n); W (M,) the scaling of each row (2/n, 1/n at k = 0; 0 for the sin(0) slot and past Kmax)."""
    F = np.zeros((M, n), dtype=LD)
    W = np.zeros(M, dtype=LD)
    j = np.arange(n, dtype=np.int64)
    F[0] = LD(1) / n
    W[0] = LD(1) / n
    for k in range(1, rf_kmax(n, M) + 1):
        c, s = _cs(j * k, n)
        F[2 * k] = 2 * c / n
        if 2 * k + 1 < M:
            F[2 * k + 1] = -2 * s / n
            W[2 * k + 1] = LD(2) / n
        W[2 * k] = LD(2) / n
    return F, W


def rf_backward_ref(c, n, deriv=0, kscale=1.0):
    """c (outer, M, inner) -> (ref (outer, n, inner), bound)."""
    outer, M, inner = c.shape
    F, W = rf_backward_matrix(n, M, deriv, kscale)
    x = _lines_last(c.astype(LD), None)
    ref = F @ x
    s = _pair_sum(W @ np.abs(x))                                   # (lines,)
    bound = C_BOUND * _lg(n) * EPS * np.broadcast_to(s, ref.shape)
    return _lines_back(ref, outer, inner), _lines_back(np.array(bound), outer, inner)


def rf_forward_ref(g, M):
    outer, n, inner = g.shape
    F, W = rf_forward_matrix(n, M)
    x = _lines_last(g.astype(LD), None)
    ref = F @ x
    s = _pair_sum(np.abs(x).sum(axis=0))
    bound = C_BOUND * _lg(n) * EPS * W[:, None] * s[None, :]
    return _lines_back(ref, outer, inner), _lines_back(bound, outer, inner)


def impulse_coeffs(M, outer, inner, sin0=None):
    """Line l = o * inner + i carries a unit coefficient at mode slot l % M (slot 1, the sin(0) slot, carries `sin0` if given)."""
    c = np.zeros((M, outer * inner))
    lines = np.arange(outer * inner)
    c[lines % M, lines] = 1.0
    if sin0 is not None:
        c[1, lines % M == 1] = sin0
    return np.ascontiguousarray(_lines_back(c, outer, inner))


def impulse_grid(n, outer, inner):
    g = np.zeros((n, outer * inner))
    lines = np.arange(outer * inner)
    g[lines % n, lines] = 1.0
    return np.ascontiguousarray(_lines_back(g, outer, inner))


def random_coeffs(rng, outer, M, inner, sin0=True):
    """O(1) coefficients; the sin(0) slot holds large values, which the backward transform must not read (as the reference's
    repack, core/transforms.py RealFFT.repack_rescale, copies only the cos(0) slot)."""
    c = rng.standard_normal((outer, M, inner))
    if sin0 and M > 1:
        c[:, 1, :] = 1e3 * rng.standard_normal((outer, inner))
    return c


def rfft_backward(B, n, c, deriv=0, kscale=1.0, misalign=(False, False)):
    """db_rfft_backward on padded buffers; returns (grid, register launches)."""
    outer, M, inner = c.shape
    plan = B.plan(n, 'real')
    cin = Padded(B, c, front=1 if misalign[0] else 2)
    g = nan_output(B, (outer, n, inner), front=1 if misalign[1] else 2)
    d = regs_delta(B, lambda: B.lib.call("db_rfft_backward", plan.ref(), cin.p, g.p, outer, M, inner, deriv, float(kscale), B.stream))
    return g.result("rfft_backward"), d


def rfft_forward(B, n, g, M, misalign=(False, False)):
    outer, _, inner = g.shape
    plan = B.plan(n, 'real')
    gin = Padded(B, g, front=1 if misalign[0] else 2)
    c = nan_output(B, (outer, M, inner), front=1 if misalign[1] else 2)
    d = regs_delta(B, lambda: B.lib.call("db_rfft_forward", plan.ref(), gin.p, c.p, outer, M, inner, B.stream))
    return c.result("rfft_forward"), d


def register_rfft_covers(n, M, inner, deriv=0, aligned=True):
    """The coverage rule of the register real-Fourier kernels (db_rfft_regs_try), restated."""
    return (n in REG_N and inner >= RR_LINES and inner % RR_LINES == 0 and deriv <= 4 and M % 2 == 0 and M >= 2
            and 3 * M <= 2 * n and aligned)


def check_rfft(B, n, M, outer, inner, derivs=(0,), kscale=1.3, seed=0, misalign=(False, False), path=None, impulse=True,
               forward=True):
    """Backward (each deriv) and forward of random data and, with `impulse`, of the impulse sweeps; asserts the kernel that served."""
    rng = np.random.default_rng(seed + 7 * n + M)
    regs = register_rfft_covers(n, M, inner, max(derivs), not any(misalign))
    path = path or ("regs" if regs else "k_fft")
    for deriv in derivs:
        datas = [random_coeffs(rng, outer, M, inner)]
        if impulse:
            datas.append(impulse_coeffs(M, outer, inner, sin0=-5.0))
        for c in datas:
            g, d = rfft_backward(B, n, c, deriv, kscale, misalign)
            assert d == (1 if regs else 0), ("served by", path, d)
            ref, bound = rf_backward_ref(c, n, deriv, kscale)
            check_bound(f"rfft_backward {path} d={deriv}", g, ref, bound)
    if forward:
        for g in [rng.standard_normal((outer, n, inner))] + ([impulse_grid(n, outer, inner)] if impulse else []):
            c, d = rfft_forward(B, n, g, M, misalign)
            assert d == (1 if regs else 0), ("served by", path, d)
            ref, bound = rf_forward_ref(g, M)
            if M > 1:
                assert (c[:, 1, :] == 0).all(), "the forward transform writes exactly 0 to the sin(0) slot"
            check_bound(f"rfft_forward {path}", c, ref, bound)
    return regs


def register_rfft_shapes(full=False):
    """(n, M, outer, inner): M in {2, 2n/3 - 2, 2n/3}; inner 16 (one tile), 48 (3 tiles per outer: ragged walks over the persistent
    CTAs) and, with `full`, more."""
    out = []
    for n in REG_N:
        Ms = (2, 2 * n // 3 - 2, 2 * n // 3)
        for k, M in enumerate(Ms):
            inner, outer = ((16, 5), (48, 1), (16, 1))[k] if n >= 384 and not full else ((16, 1), (48, 5), (16, 5))[k]
            out.append((n, M, outer, inner))
    return out


# ---- the fall-back to k_fft from the register kernels' coverage edges
def check_rfft_fallbacks(B):
    """Each case sits just outside the register kernels' coverage, which the kernel counter must show: inner 1, 8, 24; odd M;
    the first even M past 2 n / 3; deriv 5; a pointer 8 bytes off a 16-byte boundary (input, output)."""
    n = 96
    cases = [dict(M=64, inner=1, outer=19), dict(M=64, inner=8, outer=3), dict(M=64, inner=24, outer=2),
             dict(M=63, inner=16, outer=2), dict(M=66, inner=16, outer=2)]
    assert 3 * 66 == 2 * n + 6 and 3 * 64 == 2 * n
    for k, cs in enumerate(cases):
        assert not register_rfft_covers(n, cs["M"], cs["inner"])
        check_rfft(B, n, cs["M"], cs["outer"], cs["inner"], derivs=(0, 2), seed=k)
    # 3 M = 2 n + 2 needs n = 2 mod 3, which no register length is: the edge is the first even M past 2 n / 3 (3 M = 2 n + 6)
    for n in (24, 48):
        M = 2 * n // 3 + 2
        assert M % 2 == 0 and 3 * M > 2 * n
        check_rfft(B, n, M, 2, 16, derivs=(0, 1), seed=n)
    assert not register_rfft_covers(96, 64, 16, deriv=5)
    check_rfft(B, 96, 64, 2, 16, derivs=(5,), seed=5, forward=False)
    for mis in ((True, False), (False, True)):
        assert not register_rfft_covers(96, 64, 16, aligned=False)
        check_rfft(B, 96, 64, 2, 16, derivs=(0, 3), seed=11, misalign=mis)


def check_rfft_generic_lengths(B):
    """k_fft at lengths the register kernels do not have: radix 5 (n = 10, 20), the run-time 7 / 11 / 13 passes (n = 14, 22, 26),
    odd n (no half-length trick: half = 0), the static passes at nc = 48, 96, 192 reached with inner = 1, a ragged last tile (inner =
    21, outer lines 35), and a length long enough that the tile width drops below 16 (n = 3000)."""
    from dedalus_b200.fftplan import HostPlan
    for n, M, outer, inner in [(10, 6, 3, 5), (20, 12, 2, 3), (14, 10, 2, 21), (22, 14, 35, 1), (26, 16, 4, 5), (15, 10, 3, 7),
                               (21, 14, 35, 1), (9, 9, 2, 3), (96, 64, 35, 1), (192, 128, 9, 1), (384, 256, 3, 1)]:
        hp = HostPlan(n, 'real')
        if n % 2:
            assert hp.half == 0
        check_rfft(B, n, M, outer, inner, derivs=(0, 1, 2), seed=n, path="k_fft")
    assert 7 in HostPlan(14, 'real').radices and 11 in HostPlan(22, 'real').radices and 13 in HostPlan(26, 'real').radices
    assert 5 in HostPlan(10, 'real').radices


def check_rfft_narrow_tile(B):
    """n = 3000: 2 * 1500 + 3000 doubles per line; the tile width shrinks below 16 lines (110 KB budget) and the transform still covers
    every line, including a partial last tile."""
    n, M = 3000, 1000
    buf_rows = 2 * (n // 2)
    T = 16
    while T > 1 and (buf_rows * (T + 1)) * 8 > 110 * 1024:
        T //= 2
    assert T < 16
    check_rfft(B, n, M, 1, T + 3, derivs=(0,), seed=3, impulse=False)


# ------------------------------------------------------------------------------------------------------------------------------
# complex Fourier: ordering [0..KM, (Nyq), -KM..-1], forward 1/N
# ------------------------------------------------------------------------------------------------------------------------------
def cf_wavenumbers(M):
    KM = (M - 1) // 2
    return (np.arange(M) + KM) % M - KM


def cf_backward_ref(c, n, deriv, kscale):
    """c (outer, M, inner, 2) -> ref (outer, n, inner, 2), bound."""
    outer, M, inner, _ = c.shape
    Kmax = min((M - 1) // 2, (n - 1) // 2)
    ks = cf_wavenumbers(M)
    j = np.arange(n, dtype=np.int64)
    Fr = np.zeros((n, M), dtype=LD)
    Fi = np.zeros((n, M), dtype=LD)
    W = np.zeros(M, dtype=LD)
    for col, k in enumerate(ks):
        if abs(k) > Kmax:
            continue
        f = (LD(abs(k)) * LD(kscale)) ** deriv if deriv else LD(1)
        cc, ss = _cs(4 * j * k + deriv * n * int(np.sign(k)), 4 * n)
        Fr[:, col], Fi[:, col], W[col] = f * cc, f * ss, f
    zr, zi = _lines_last(c[..., 0].astype(LD), None), _lines_last(c[..., 1].astype(LD), None)
    gr, gi = Fr @ zr - Fi @ zi, Fr @ zi + Fi @ zr
    s = W @ (np.abs(zr) + np.abs(zi))
    bound = C_BOUND * _lg(n) * EPS * np.broadcast_to(s, gr.shape)
    ref = np.stack([_lines_back(gr, outer, inner), _lines_back(gi, outer, inner)], -1)
    b = _lines_back(np.array(bound), outer, inner)
    return ref, np.stack([b, b], -1)


def cf_forward_ref(g, M):
    outer, n, inner, _ = g.shape
    Kmax = min((M - 1) // 2, (n - 1) // 2)
    ks = cf_wavenumbers(M)
    j = np.arange(n, dtype=np.int64)
    Fr = np.zeros((M, n), dtype=LD)
    Fi = np.zeros((M, n), dtype=LD)
    W = np.zeros(M, dtype=LD)
    for row, k in enumerate(ks):
        if abs(k) > Kmax:
            continue
        cc, ss = _cs(j * k, n)
        Fr[row], Fi[row], W[row] = cc / n, -ss / n, LD(1) / n
    xr, xi = _lines_last(g[..., 0].astype(LD), None), _lines_last(g[..., 1].astype(LD), None)
    cr, ci = Fr @ xr - Fi @ xi, Fr @ xi + Fi @ xr
    s = (np.abs(xr) + np.abs(xi)).sum(axis=0)
    bound = C_BOUND * _lg(n) * EPS * W[:, None] * s[None, :]
    ref = np.stack([_lines_back(cr, outer, inner), _lines_back(ci, outer, inner)], -1)
    b = _lines_back(bound, outer, inner)
    return ref, np.stack([b, b], -1)


def check_cfft(B, n, M, outer, inner, derivs=(0, 1, 2, 3), kscale=0.7, seed=0):
    rng = np.random.default_rng(seed + n * 31 + M)
    plan = B.plan(n, 'complex')
    lines = outer * inner
    imp = np.zeros((M, lines, 2))
    imp[np.arange(lines) % M, np.arange(lines), (np.arange(lines) // M) % 2] = 1.0      # real, then imaginary unit per slot
    imp = np.ascontiguousarray(np.moveaxis(imp.reshape(M, outer, inner, 2), 0, 1))
    for deriv in derivs:
        for c in (rng.standard_normal((outer, M, inner, 2)), imp):
            cin = Padded(B, c)
            g = nan_output(B, (outer, n, inner, 2))
            d = regs_delta(B, lambda: B.lib.call("db_cfft_backward", plan.ref(), cin.p, g.p, outer, M, inner, deriv, kscale, B.stream))
            assert d == 0
            ref, bound = cf_backward_ref(c, n, deriv, kscale)
            check_bound(f"cfft_backward d={deriv}", g.result("cfft_backward"), ref, bound)
    gimp = np.zeros((n, lines, 2))
    gimp[np.arange(lines) % n, np.arange(lines), (np.arange(lines) // n) % 2] = 1.0
    gimp = np.ascontiguousarray(np.moveaxis(gimp.reshape(n, outer, inner, 2), 0, 1))
    for g in (rng.standard_normal((outer, n, inner, 2)), gimp):
        gin = Padded(B, g)
        c = nan_output(B, (outer, M, inner, 2))
        B.lib.call("db_cfft_forward", plan.ref(), gin.p, c.p, outer, M, inner, B.stream)
        ref, bound = cf_forward_ref(g, M)
        out = c.result("cfft_forward")
        if M % 2 == 0:
            assert (out[:, M // 2] == 0).all(), "the Nyquist slot is written as 0"
        check_bound("cfft_forward", out, ref, bound)


# ------------------------------------------------------------------------------------------------------------------------------
# Chebyshev: DCT-II / DCT-III, unit-weight normalisation, odd modes negated, banded conversions
# ------------------------------------------------------------------------------------------------------------------------------
def cheb_weights(K):
    w = np.full(K, np.sqrt(LD(2) / PI), dtype=LD)
    w[0] = 1 / np.sqrt(PI)
    return w


def cheb_backward_matrix(n, K):
    """g = T y over the first K = min(M, n) modes; T (n, K)."""
    j = np.arange(n, dtype=np.int64)[:, None]
    k = np.arange(K, dtype=np.int64)[None, :]
    c, _ = _cs(k * (2 * j + 1), 4 * n)
    return c * cheb_weights(K)[None, :] * np.where(k % 2 == 1, -1, 1).astype(LD)


def cheb_forward_matrix(n, K):
    j = np.arange(n, dtype=np.int64)[None, :]
    k = np.arange(K, dtype=np.int64)[:, None]
    c, _ = _cs(k * (2 * j + 1), 4 * n)
    s = np.full(K, np.sqrt(2 * PI) / n, dtype=LD)
    s[0] = np.sqrt(PI) / n
    return c * (s * np.where(np.arange(K) % 2 == 1, -1, 1).astype(LD))[:, None], s


def banded_apply(diags, x, xa):
    """diags (nd, M): y_i = sum_{d, i + d < M} diags[d][i] x_{i+d}; x (M, lines), long double; and the same on the magnitudes xa."""
    M = x.shape[0]
    y = np.zeros_like(x)
    ya = np.zeros_like(x)
    for d in range(diags.shape[0]):
        D = diags[d, :M - d].astype(LD)[:, None]
        y[:M - d] += D * x[d:]
        ya[:M - d] += np.abs(D) * xa[d:]
    return y, ya


def banded_solve(sol, t, ta, stride=1):
    """Upper back-substitution with row 0 = reciprocal diagonal, row r = super-diagonal r * stride: x_i = (t_i - sum u x) * r_i.
    Returns x and the stage-by-stage magnitude xa (the same recurrence on |.|, started from ta)."""
    M = t.shape[0]
    x = np.zeros_like(t)
    xa = np.zeros_like(t)
    for i in range(M - 1, -1, -1):
        acc, acca = t[i].copy(), ta[i].copy()
        for r in range(1, sol.shape[0]):
            d = r * stride
            if i + d < M:
                u = LD(sol[r, i])
                acc -= u * x[i + d]
                acca += abs(u) * xa[i + d]
        r0 = LD(sol[0, i])
        x[i], xa[i] = acc * r0, acca * abs(r0)
    return x, xa


def cheb_backward_ref(c, n, pre=None, sol=None, stride=1):
    """c (outer, M, inner): g = DCT-III(scale(solve(apply(pre, c)))), modes >= n dropped; returns ref, bound."""
    outer, M, inner = c.shape
    x = _lines_last(c.astype(LD), None)
    if M > n:
        x = x.copy()
        x[n:] = 0
    xa = np.abs(x)
    stages = 0
    if pre is not None and pre.shape[0] > 0:
        x, xa = banded_apply(pre, x, xa)
        stages += pre.shape[0]
    if sol is not None and sol.shape[0] > 0:
        x, xa = banded_solve(sol, x, xa, stride)
        stages += sol.shape[0]
    K = min(M, n)
    T = cheb_backward_matrix(n, K)
    ref = T @ x[:K]
    s = _pair_sum(cheb_weights(K) @ xa[:K])
    bound = C_BOUND * (_lg(n) + stages) * EPS * np.broadcast_to(s, ref.shape)
    return _lines_back(ref, outer, inner), _lines_back(np.array(bound), outer, inner)


def cheb_forward_ref(g, M, conv=None):
    outer, n, inner = g.shape
    K = min(M, n)
    F, s = cheb_forward_matrix(n, K)
    x = _lines_last(g.astype(LD), None)
    y = np.zeros((M, x.shape[1]), dtype=LD)
    ya = np.zeros_like(y)
    y[:K] = F @ x
    ya[:K] = s[:, None] * _pair_sum(np.abs(x).sum(axis=0))[None, :]
    stages = 0
    if conv is not None and conv.shape[0] > 0:
        cv = conv.copy()
        for d in range(cv.shape[0]):            # the conversion reads modes < K only (the truncation comes first)
            cv[d, max(K - d, 0):] = 0
        y, ya = banded_apply(cv, y, ya)
        y[K:], ya[K:] = 0, 0
        stages = conv.shape[0]
    bound = C_BOUND * (_lg(n) + stages) * EPS * ya
    zero = np.zeros_like(ya, dtype=bool)
    zero[K:] = True
    return _lines_back(y, outer, inner), _lines_back(bound, outer, inner), _lines_back(zero, outer, inner)


def conversion_diags(M, n, alpha):
    """Upper diagonals (2 alpha + 1 of them, row length M) of the (-1/2, -1/2) -> (alpha - 1/2, alpha - 1/2) conversion."""
    from dedalus_b200 import jacobi
    from dedalus_b200.transforms import banded_upper_diags
    a = alpha - 0.5
    return np.ascontiguousarray(banded_upper_diags(jacobi.conversion_matrix(max(M, n), -0.5, -0.5, a, a), M, 2 * alpha + 1))


def solve_diags(M, alpha):
    """Back-conversion diagonals in the solve storage: row 0 reciprocal diagonal, every diagonal (stride 1)."""
    from dedalus_b200 import jacobi
    a = alpha - 0.5
    Cm = jacobi.conversion_matrix(M, -0.5, -0.5, a, a).toarray()
    nd = 2 * alpha + 1
    s = np.zeros((nd, M))
    for d in range(nd):
        s[d, :M - d] = np.diag(Cm, d)
    s[0] = 1.0 / s[0]
    return s


def pre_diags(rng, M, npre):
    p = np.zeros((max(npre, 1), M))
    for d in range(npre):
        p[d, :M - d] = rng.uniform(0.5, 2.0, M - d) * (1 + np.arange(M - d)) ** 0.5 * rng.choice([-1, 1], M - d)
    return p


def cheb_call(B, fwd, n, x, M, inner, conv=None, pre=None, sol=None, misalign=(False, False)):
    lines_outer = x.shape[0]
    plan = B.plan(n, 'real')
    xin = Padded(B, x, front=1 if misalign[0] else 2)
    out = nan_output(B, (lines_outer, M if fwd else n, inner), front=1 if misalign[1] else 2)
    keep = []

    def dp(a):
        if a is None or a.shape[0] == 0:
            return None, 0
        t = B.dev(np.ascontiguousarray(a))
        keep.append(t)
        return B.ptr(t), a.shape[0]
    if fwd:
        cp, cn = dp(conv)
        d = regs_delta(B, lambda: B.lib.call("db_cheb_forward", plan.ref(), xin.p, out.p, lines_outer, M, inner, cp, cn, B.stream))
    else:
        pp, pn = dp(pre)
        sp, sn = dp(sol)
        d = regs_delta(B, lambda: B.lib.call("db_cheb_backward", plan.ref(), xin.p, out.p, lines_outer, M, inner, pp, pn, sp, sn,
                                             B.stream))
    return out.result("cheb"), d


def register_cheb_covers(n, M, inner, fwd, has_banded=False, aligned=True):
    return (n in REG_N[:-1] and inner == 1 and M % 2 == 0 and 2 <= M <= n and aligned and (fwd or not has_banded))


def check_cheb(B, n, M, outer, inner, nds=(0,), seed=0, misalign=(False, False), pre_sol=(), impulse=True, path=None):
    """Forward with conversions of nd diagonals (nd = 2 alpha + 1), backward plain and with (npre, alpha) pre-apply / solve."""
    rng = np.random.default_rng(seed + 13 * n + M)
    aligned = not any(misalign)
    for nd in nds:
        conv = conversion_diags(M, n, (nd - 1) // 2) if nd else None
        regs = register_cheb_covers(n, M, inner, True, aligned=aligned)
        p = path or ("regs" if regs else "k_fft")
        gs = [rng.standard_normal((outer, n, inner))] + ([impulse_grid(n, outer, inner)] if impulse else [])
        for g in gs:
            c, d = cheb_call(B, True, n, g, M, inner, conv=conv, misalign=misalign)
            assert d == (1 if regs else 0), ("served by", p, d)
            ref, bound, zero = cheb_forward_ref(g, M, conv)
            check_bound(f"cheb_forward {p} nd={nd}", c, ref, bound, exact_zero=zero)
    for npre, alpha in ((0, 0),) + tuple(pre_sol):
        pre = pre_diags(rng, M, npre) if npre else None
        sol = solve_diags(M, alpha) if alpha else None
        regs = register_cheb_covers(n, M, inner, False, has_banded=bool(npre or alpha), aligned=aligned)
        p = path or ("regs" if regs else "k_fft")
        cs = [rng.standard_normal((outer, M, inner))] + ([impulse_coeffs(M, outer, inner)] if impulse else [])
        for c in cs:
            g, d = cheb_call(B, False, n, c, M, inner, pre=pre, sol=sol, misalign=misalign)
            assert d == (1 if regs else 0), ("served by", p, d)
            ref, bound = cheb_backward_ref(c, n, pre, sol)
            check_bound(f"cheb_backward {p} pre={npre} solve={2 * alpha + 1 if alpha else 0}", g, ref, bound)


def register_cheb_shapes():
    """(n, M, lines): M in {2, n/2, n}; lines 1, 15, 16, 17, 33 spread over the sizes (partial tiles, one line of a pair)."""
    lines = (1, 15, 16, 17, 33)
    out = []
    for i, n in enumerate(REG_N[:-1]):
        for k, M in enumerate((2, n // 2, n)):
            out.append((n, M, lines[(i + k) % len(lines)]))
    return out


def check_cheb_scan(B, n, M, lines, npre, seed=0):
    """db_cheb_backward_scan (fused pre-apply and two-diagonal back-conversion, register DCT) against the long-double chain."""
    from dedalus_b200 import jacobi
    rng = np.random.default_rng(seed + n + npre)
    Cm = jacobi.conversion_matrix(M, -0.5, -0.5, 0.5, 0.5).toarray()
    sol2 = np.zeros((2, M))
    sol2[0], sol2[1, :M - 2] = 1.0 / np.diag(Cm), np.diag(Cm, 2)
    pre = pre_diags(rng, M, npre) if npre else None
    plan = B.plan(n, 'real')
    for c in (rng.standard_normal((lines, M, 1)), impulse_coeffs(M, lines, 1)):
        cin = Padded(B, c)
        g = nan_output(B, (lines, n, 1))
        pd = B.dev(pre) if pre is not None else None
        sd = B.dev(sol2)
        rc = []
        d = regs_delta(B, lambda: rc.append(B.lib.call_optional("db_cheb_backward_scan", plan.ref(), cin.p, g.p, lines, M,
                                                                 B.ptr(pd) if pd is not None else None, npre, B.ptr(sd), B.stream)))
        assert rc == [True] and d == 1
        ref, bound = cheb_backward_ref(c, n, pre, sol2, stride=2)
        check_bound(f"cheb_backward_scan pre={npre}", g.result("cheb_backward_scan"), ref, bound)


def check_cheb_scan_declines(B):
    """Returns 2 and records no error where the fused kernel does not apply: n = 20, odd M, a misaligned input or output."""
    M = 12
    sol2 = B.dev(np.ones((2, 14)))
    err0 = B.lib._raw_db_last_error()
    for n, M, mis in ((20, 12, (False, False)), (48, 13, (False, False)), (48, 12, (True, False)), (48, 12, (False, True))):
        plan = B.plan(n, 'real')
        cin = Padded(B, np.ones((3, M, 1)), front=1 if mis[0] else 2)
        g = nan_output(B, (3, n, 1), front=1 if mis[1] else 2)
        d = regs_delta(B, lambda: (assert_false(B.lib.call_optional("db_cheb_backward_scan", plan.ref(), cin.p, g.p, 3, M, None, 0,
                                                                     B.ptr(sol2), B.stream))))
        assert d == 0
        assert np.isnan(g.read()[0]).all(), "nothing written"
    assert B.lib._raw_db_last_error() == err0


def assert_false(v):
    assert v is False


def check_band_lines(B, n, lines, npre, stride, seed=0):
    """db_band_lines: stride 1 (every diagonal, one thread per line) and 2 (main and second super-diagonal, warp scan)."""
    rng = np.random.default_rng(seed + n * 3 + npre + stride)
    if stride == 1:
        sol = solve_diags(n, 1)
    else:
        from dedalus_b200 import jacobi
        Cm = jacobi.conversion_matrix(n, -0.5, -0.5, 0.5, 0.5).toarray()
        sol = np.zeros((2, n))
        sol[0], sol[1, :n - 2] = 1.0 / np.diag(Cm), np.diag(Cm, 2)
    pre = pre_diags(rng, n, npre) if npre else None
    for c in (rng.standard_normal((lines, n)), impulse_coeffs(n, lines, 1)[:, :, 0]):
        cin = Padded(B, c)
        out = nan_output(B, (lines, n))
        pd = B.dev(pre) if pre is not None else None
        sd = B.dev(sol)
        B.lib.call("db_band_lines", cin.p, out.p, lines, n, B.ptr(pd) if pd is not None else None, npre, B.ptr(sd), sol.shape[0], stride,
                   B.stream)
        x = c.T.astype(LD)
        xa = np.abs(x)
        if pre is not None:
            x, xa = banded_apply(pre, x, xa)
        x, xa = banded_solve(sol, x, xa, stride)
        bound = C_BOUND * (_lg(n) + npre + sol.shape[0]) * EPS * xa
        check_bound(f"band_lines stride={stride}", out.result("band_lines"), x.T, bound.T)


# ------------------------------------------------------------------------------------------------------------------------------
# blocked and peer entries
# ------------------------------------------------------------------------------------------------------------------------------
def blocked_layout(a, rpb):
    """(outer, rows, inner) -> blocks (rows // rpb, outer, rpb, inner): the blocked row addressing with blk_stride = outer rpb inner."""
    outer, rows, inner = a.shape
    return np.ascontiguousarray(a.reshape(outer, rows // rpb, rpb, inner).transpose(1, 0, 2, 3))


def check_blocked_and_peer(B, n, M, outer, inner, n_peers, in_blocked, deriv=1, kscale=0.9, seed=0):
    """Backward and forward through the blocked entry (blocks in one buffer, NaN gaps between them) and through the peer entry
    (each block its own allocation): bitwise equal to each other, both within the bound of the long-double reference."""
    rng = np.random.default_rng(seed + n + n_peers)
    plan = B.plan(n, 'real')
    for fwd in (False, True):
        rows_in, rows_out = (n, M) if fwd else (M, n)
        assert rows_out % n_peers == 0 and (not in_blocked or rows_in % n_peers == 0)
        orpb = rows_out // n_peers
        irpb = rows_in // n_peers if in_blocked else 0
        x = rng.standard_normal((outer, rows_in, inner)) if fwd else random_coeffs(rng, outer, M, inner)
        gap = 6                                        # doubles of NaN between blocks (even: every block stays 16-byte aligned)
        if irpb:
            blk_in = blocked_layout(x, irpb)
            in_stride = outer * irpb * inner + gap
            hin = np.full((n_peers, in_stride), np.nan)
            hin[:, :outer * irpb * inner] = blk_in.reshape(n_peers, -1)
            xin = Padded(B, hin)
        else:
            in_stride = 0
            xin = Padded(B, x)
        out_stride = outer * orpb * inner + gap
        blk = Padded(B, np.full((n_peers, out_stride), np.nan))
        args_in = (xin.p, blk.p, outer, M, inner) if fwd else (xin.p, blk.p, outer, M, inner, deriv, kscale)
        name = "db_rfft_forward_blocked" if fwd else "db_rfft_backward_blocked"
        d = regs_delta(B, lambda: assert_true(B.lib.call_optional(name, plan.ref(), *args_in, irpb, in_stride, orpb, out_stride,
                                                                  B.stream)))
        assert d == 1
        hb = blk.result("blocked").reshape(n_peers, out_stride)
        assert np.isnan(hb[:, outer * orpb * inner:]).all(), "wrote into the gap between blocks"
        got = hb[:, :outer * orpb * inner].reshape(n_peers, outer, orpb, inner).transpose(1, 0, 2, 3).reshape(outer, rows_out, inner)
        ref, bound = rf_forward_ref(x, M) if fwd else rf_backward_ref(x, n, deriv, kscale)
        check_bound(f"rfft_{'forward' if fwd else 'backward'}_blocked", got, ref, bound)
        # peer: separate allocations, each the layout (outer, rpb, inner) of one block; local_out = an aligned origin
        peers = [Padded(B, np.full((outer, orpb, inner), np.nan), tail=8) for _ in range(n_peers)]
        local = B.dev(np.zeros(2))
        ptrs = (C.c_void_p * n_peers)(*[p.p.value for p in peers])
        args_in = (xin.p, B.ptr(local), outer, M, inner) if fwd else (xin.p, B.ptr(local), outer, M, inner, deriv, kscale)
        d = regs_delta(B, lambda: assert_true(B.lib.call_optional("db_rfft_forward_peer" if fwd else "db_rfft_backward_peer",
                                                                  plan.ref(), *args_in, irpb, in_stride, orpb, n_peers, ptrs, B.stream)))
        assert d == 1
        for b, p in enumerate(peers):
            got_b = p.result("peer")
            assert np.array_equal(got_b, hb[b, :outer * orpb * inner].reshape(outer, orpb, inner)), ("peer != blocked", b)


def assert_true(v):
    assert v is True


def check_blocked_declines(B):
    """Return code 2 (not covered): 9 peers, a peer block 8 bytes off a 16-byte boundary, an odd block stride."""
    n, M, outer, inner = 48, 32, 1, 16
    plan = B.plan(n, 'real')
    g = Padded(B, np.ones((outer, n, inner)))
    local = B.dev(np.zeros(2))
    blocks = [Padded(B, np.full((outer, 4, inner), np.nan)) for _ in range(9)]
    for k, ptrs in ((9, [b.p.value for b in blocks]), (4, [b.p.value for b in blocks[:3]] + [blocks[3].p.value + 8])):
        arr = (C.c_void_p * k)(*ptrs)
        d = regs_delta(B, lambda: assert_false(B.lib.call_optional("db_rfft_forward_peer", plan.ref(), g.p, B.ptr(local), outer, M, inner,
                                                                   0, 0, M // k if M % k == 0 else 4, k, arr, B.stream)))
        assert d == 0
    out = Padded(B, np.full(4 * 200, np.nan))
    for in_rpb, in_st, out_rpb, out_st in ((0, 0, 8, 129), (8, 129, 8, 130)):
        d = regs_delta(B, lambda: assert_false(B.lib.call_optional("db_rfft_forward_blocked", plan.ref(), g.p, out.p, outer, M, inner,
                                                                   in_rpb, in_st, out_rpb, out_st, B.stream)))
        assert d == 0
    for b in blocks:
        assert np.isnan(b.read()[0]).all()


# ------------------------------------------------------------------------------------------------------------------------------
# the fused x pass: db_rfft_x_products
# ------------------------------------------------------------------------------------------------------------------------------
XPROD_DTYPE = np.dtype([('coef', '<f8'), ('src', '<i4'), ('deriv', '<i4'), ('a', '<i4'), ('b', '<i4'), ('out', '<i4'), ('flags', '<i4')])
HELD, LAST = 1, 2


def xprod_items(rec):
    return np.array([tuple(r) for r in rec], dtype=XPROD_DTYPE)


def xprod_schedules():
    """name -> (n_in, n_out, items as (coef, src, deriv, a, b, out, flags)).  Factor codes: 0..2 held, 3 the input streamed by the
    item, -1 none."""
    S = {}
    # linear terms only, no held factors; outputs in non-ascending order; one single-term output
    S["linear_no_held"] = (3, 3, [(1.5, 0, 1, 3, -1, 2, 0), (-0.25, 1, 0, 3, -1, 2, LAST),
                                  (2.0, 2, 2, 3, -1, 0, LAST), (-1e-3, 0, 0, 3, -1, 1, LAST)])
    # one held factor times streamed inputs; a streamed input loaded twice with different derivative orders
    S["one_held"] = (3, 2, [(0, 0, 0, 0, -1, -1, HELD),
                            (1.0, 1, 1, 0, 3, 1, 0), (-2.0, 1, 3, 3, 0, 1, LAST),
                            (0.5, 2, 4, 3, 0, 0, 0), (3.0, 2, 0, 0, 3, 0, LAST)])
    # two held factors, a product of two held factors (src < 0), held slot 0 overwritten mid-schedule (with another deriv)
    S["held_reuse"] = (3, 3, [(0, 0, 0, 0, -1, -1, HELD), (0, 1, 1, 1, -1, -1, HELD),
                              (1.0, -1, 0, 0, 1, 2, 0), (-0.75, 2, 2, 3, 1, 2, LAST),
                              (0, 0, 2, 0, -1, -1, HELD),
                              (1e-6, -1, 0, 0, 0, 0, 0), (-4.0, -1, 0, 1, -1, 0, LAST),
                              (2.5, 2, 0, 0, 3, 1, LAST)])
    # three held factors: a u . grad(u)-like schedule with linear terms mixed in, outputs 1, 0, 2 in that order
    S["three_held"] = (4, 3, [(0, 0, 0, 0, -1, -1, HELD), (0, 1, 0, 1, -1, -1, HELD), (0, 2, 0, 2, -1, -1, HELD),
                              (-1.0, 3, 1, 0, 3, 1, 0), (-1.0, 3, 2, 1, 3, 1, 0), (0.5, 3, 0, 3, -1, 1, LAST),
                              (-1.0, 0, 1, 0, 3, 0, 0), (-1.0, -1, 0, 1, 2, 0, 0), (1e-2, -1, 0, 2, -1, 0, LAST),
                              (-3.0, -1, 0, 2, 2, 2, LAST)])
    return S


def xprod_ref(cin, n, items, kscale, n_out):
    """cin (n_in, M, inner) -> (ref (n_out, M, inner), bound, written outputs).  Every factor: the long-double backward transform with
    its derivative; its error bound e = C L eps (pair-summed stage magnitude).  A term's error |coef| (|a| e_b + |b| e_a) plus
    rounding; the output's error through the forward transform, plus the forward's own rounding of the accumulated grid values."""
    n_in, M, inner = cin.shape
    L = _lg(n)
    Ff, Wf = rf_forward_matrix(n, M)
    grids = {}

    def factor(src, deriv):
        key = (src, deriv)
        if key not in grids:
            F, W = rf_backward_matrix(n, M, deriv, kscale)
            x = cin[src].astype(LD)
            g = F @ x
            e = C_BOUND * L * EPS * _pair_sum(W @ np.abs(x))
            grids[key] = (g, np.broadcast_to(e, g.shape))
        return grids[key]
    held = {}
    acc = {}
    out_ref = {}
    for it in items:
        coef, src, deriv, a, b, o, flags = (it[k] for k in XPROD_DTYPE.names)
        stream = factor(src, deriv) if src >= 0 else None
        if flags & HELD:
            held[a] = stream
            continue
        fa = stream if a == 3 else held[a]
        fb = None if b < 0 else (stream if b == 3 else held[b])
        g, e, m = acc.get(o, (0, 0, 0))
        c = LD(coef)
        if fb is None:
            g = g + c * fa[0]
            e = e + abs(c) * fa[1]
            m = m + abs(c) * np.abs(fa[0])
        else:
            g = g + c * fa[0] * fb[0]
            e = e + abs(c) * (np.abs(fa[0]) * fb[1] + np.abs(fb[0]) * fa[1] + fa[1] * fb[1])
            m = m + abs(c) * np.abs(fa[0] * fb[0])
        acc[o] = (g, e, m)
        if flags & LAST:
            g, e, m = acc.pop(o)
            e = e + C_BOUND * 4 * EPS * m                                 # products and the accumulation
            ref = Ff @ g
            bound = Wf[:, None] * (_pair_sum(e.sum(axis=0)) + C_BOUND * L * EPS * _pair_sum(m.sum(axis=0)))[None, :]
            out_ref[o] = (ref, bound)
    return out_ref


def x_products(B, n, cin, items, n_out, kscale, n_held, in_pad=0, out_pad=0, expect_rc=0):
    """db_rfft_x_products with the inputs / outputs `in_pad` / `out_pad` doubles apart (NaN between them).  Returns (outputs, the
    stride gaps, register launches)."""
    n_in, M, inner = cin.shape
    in_stride, out_stride = M * inner + in_pad, M * inner + out_pad
    hin = np.full((n_in, in_stride), np.nan)
    hin[:, :M * inner] = cin.reshape(n_in, -1)
    xin = Padded(B, hin)
    out = Padded(B, np.full((n_out, out_stride), np.nan))
    it = B.dev(np.frombuffer(items.tobytes(), dtype=np.uint8).copy())
    loads = np.ascontiguousarray(items['src'][items['src'] >= 0].astype(np.int32))
    ld = B.dev(loads)
    plan = B.plan(n, 'real')
    rc = []
    d = regs_delta(B, lambda: rc.append(B.lib._raw_db_rfft_x_products(plan.ref(), xin.p, in_stride, out.p, out_stride, M, inner,
                                                                      float(kscale), B.ptr(it), len(items), B.ptr(ld), len(loads),
                                                                      n_held, B.stream)))
    if expect_rc:
        assert rc[0] != 0, "expected a rejection"
        return None, None, d
    assert rc[0] == 0, B.lib._raw_db_last_error()
    h = out.result("x_products").reshape(n_out, out_stride)
    return h[:, :M * inner].reshape(n_out, M, inner), h[:, M * inner:], d


def check_x_products(B, n, M, inner, sched, in_pad=0, out_pad=0, impulse=False, seed=0, kscale=1.1):
    n_in, n_out, rec = xprod_schedules()[sched]
    items = xprod_items(rec)
    n_held = len({r[3] for r in rec if r[6] & HELD})
    rng = np.random.default_rng(seed + n + M + inner)
    if impulse:
        lines = np.arange(inner)
        cin = np.zeros((n_in, M, inner))
        for s in range(n_in):
            cin[s, (lines + 5 * s) % M, lines] = 1.0
            cin[s, 0, :] += 0.5                              # a mean, so that products of impulses are not all zero
    else:
        cin = rng.standard_normal((n_in, M, inner))
    cin[:, 1, :] = 1e3                                    # the sin(0) slot is not read
    got, gaps, d = x_products(B, n, cin, items, n_out, kscale, n_held, in_pad, out_pad)
    assert d == 1
    assert np.isnan(gaps).all(), "wrote into the padding between outputs"
    refs = xprod_ref(cin, n, items, kscale, n_out)
    assert sorted(refs) == sorted(set(items['out'][items['out'] >= 0]))
    for o, (ref, bound) in refs.items():
        check_bound(f"x_products {'impulse' if impulse else 'random'}", got[o], ref, bound)
    return n_held


def xprod_shapes():
    """(n, M): M in {2, 2n/3 - 2, 2n/3}."""
    return [(n, M) for n in REG_N[:-1] for M in (2, 2 * n // 3 - 2, 2 * n // 3)]


def check_x_products_rejections(B):
    """The error return and its message: n = 768 (no kernel), inner = 8, n_held = 4, odd M."""
    n_in, n_out, rec = xprod_schedules()["one_held"]
    items = xprod_items(rec)
    for n, M, inner, n_held, msg in ((768, 64, 16, 1, "no kernel for n = 768"),
                                     (96, 64, 8, 1, "case not covered (n = 96, M = 64, inner = 8, 1 held factors)"),
                                     (96, 64, 16, 4, "case not covered (n = 96, M = 64, inner = 16, 4 held factors)"),
                                     (96, 63, 16, 1, "case not covered (n = 96, M = 63, inner = 16, 1 held factors)")):
        cin = np.ones((n_in, M, inner))
        _, _, d = x_products(B, n, cin, items, n_out, 1.0, n_held, expect_rc=1)
        assert d == 0
        err = B.lib._raw_db_last_error().decode()
        assert msg in err, (msg, err)


def check_x_products_supported_agrees(B):
    """RealFourierTransform.x_products_supported against the C entry point (rejection or launch) over (n, M, inner, n_held)."""
    from dedalus_b200.transforms import RealFourierTransform
    _, _, rec = xprod_schedules()["linear_no_held"]
    items = xprod_items(rec)
    seen = set()
    for n in (24, 48, 96, 192, 384, 768, 72):
        for M in (2, 2 * n // 3 - 1, 2 * n // 3, 2 * n // 3 + 2):
            for inner in (8, 16, 24, 32):
                for n_held in (0, 3, 4):
                    ok = RealFourierTransform(n, M).x_products_supported(inner, n_held)
                    _, _, d = x_products(B, n, np.zeros((3, M, inner)), items, 3, 1.0, n_held, expect_rc=0 if ok else 1)
                    assert d == (1 if ok else 0)
                    seen.add(ok)
    assert seen == {True, False}


def check_x_products_large(B, n, M, inner, sched, sample=64, seed=0, kscale=1.0):
    """The fused x pass over `inner` lines; the reference on `sample` random line pairs (the bound pairs lines 2m, 2m + 1)."""
    n_in, n_out, rec = xprod_schedules()[sched]
    items = xprod_items(rec)
    n_held = len({r[3] for r in rec if r[6] & HELD})
    rng = np.random.default_rng(seed + n + inner)
    cin = rng.standard_normal((n_in, M, inner))
    got, gaps, d = x_products(B, n, cin, items, n_out, kscale, n_held)
    assert d == 1
    pairs = np.sort(rng.choice(inner // 2, sample, replace=False))
    cols = np.stack([2 * pairs, 2 * pairs + 1], 1).reshape(-1)
    cols[-2:] = inner - 2, inner - 1                              # the last tile's last pair
    for o, (ref, bound) in xprod_ref(np.ascontiguousarray(cin[:, :, cols]), n, items, kscale, n_out).items():
        check_bound("x_products benchmark shape", got[o][:, cols], ref, bound)


def check_rfft_backward_odd_M_reads_no_row_past_the_line(B):
    """Regression: with odd M the last mode k = (M - 1) / 2 has its cos slot only.  k_fft's backward read a -sin value for it from
    row M -- the next outer slab's row 0 on a strided axis (a wrong mode), past the array for the last slab (NaN here), and past the
    staged coefficients in shared memory on a contiguous one.  Both layouts, with a NaN gap behind the input."""
    for n, M, outer, inner in ((96, 63, 3, 16), (48, 31, 2, 8), (96, 63, 21, 1), (22, 13, 2, 3)):
        assert M % 2 == 1 and not register_rfft_covers(n, M, inner)
        rng = np.random.default_rng(M + inner)
        for c in (rng.standard_normal((outer, M, inner)), impulse_coeffs(M, outer, inner)):
            for deriv in (0, 1):
                g, d = rfft_backward(B, n, c, deriv, 0.8)
                assert d == 0
                ref, bound = rf_backward_ref(c, n, deriv, 0.8)
                check_bound(f"rfft_backward k_fft d={deriv}", g, ref, bound)
