"""Shared bodies of the kernel-level tests of the grid products and the transposes in csrc/pointwise.cu: db_pointwise (k_pointwise,
k_pointwise_v3), db_pointwise_pairs (k_pointwise_pairs) and the four db_transpose_* entries (k_tr_chunks), through the CPU emulation of
the kernels (tests/test_emu_pointwise_kernels.py) and on the GPU (tests/test_gpu_1f_pointwise_kernels.py).

The product references are restated from include/dedalus_b200.h in np.longdouble: out[o, p] = sum_t coef_t prod_f in[f, p], compared
componentwise against
    C_BOUND * (T_o + F_max) * eps * sum_t |coef_t| prod_f |in[f, p]|,
with T_o the number of terms of output o and F_max the largest factor count of the program (a product of F factors rounds F times, a
sum of T terms T - 1 times; the pairs kernel's fma(coef * a, b, acc) rounds no more often).  One constant C_BOUND serves the file; the
largest observed error / bound per kernel is kept in RATIOS.  Outputs without terms must be exactly +0.0.  The transposes are checked
bitwise against the layouts of the header, restated as numpy index arithmetic.  Every output buffer starts as NaN with NaN gaps before
and after it, which must survive, and every case asserts which kernel ran (db_pointwise_launches)."""
import ctypes as C
import numpy as np
from transform_kernel_cases import Padded, nan_output, env

EPS = np.finfo(np.float64).eps
LD = np.longdouble
C_BOUND = 2.0
PW_TILE, PW3_T = 256, 128                         # csrc/pointwise.cu: points per CTA of k_pointwise, point pairs per CTA of v3 / pairs
MAX_SMEM = 227 * 1024
MAX_IN = MAX_SMEM // (PW_TILE * 8)                # k_pointwise: one tile of every input
MAX_IN_V3 = MAX_SMEM // (2 * PW3_T * 16)          # v3 and pairs: two tiles of point pairs
assert (MAX_IN, MAX_IN_V3) == (113, 56)
K_PW, K_V3, K_PAIRS, K_TR16, K_TR8 = range(5)     # db_pointwise_launches kinds
NAMES = {K_PW: "k_pointwise", K_V3: "k_pointwise_v3", K_PAIRS: "k_pointwise_pairs", K_TR16: "transpose 16-byte", K_TR8: "transpose 8-byte"}
PAIR_DTYPE = np.dtype([('coef', '<f8'), ('a', '<i4'), ('b', '<i4')])      # db_pair_term
RATIOS = {}


def report():
    return "\n".join(f"  {k:<24s} {v:.3g}" for k, v in sorted(RATIOS.items()))


def launches(B):
    return np.array([B.lib._raw_db_pointwise_launches(k) for k in range(5)])


def ran(B, fn):
    """(return value of fn, the kernel kinds it launched as a count per kind)."""
    before = launches(B)
    rc = fn()
    return rc, launches(B) - before


def one(kind):
    d = np.zeros(5, dtype=np.int64)
    d[kind] = 1
    return d


# ------------------------------------------------------------------------------------------------------------------------------
# programs
# ------------------------------------------------------------------------------------------------------------------------------
class Program:
    """outputs: list (one per output) of lists of (coef, [factor inputs])."""

    def __init__(self, n_in, outputs):
        self.n_in, self.outputs = n_in, outputs
        self.n_out = len(outputs)
        self.term_ptr = np.cumsum([0] + [len(o) for o in outputs]).astype(np.int32)
        terms = [t for o in outputs for t in o]
        self.coef = np.array([c for c, _ in terms] or [0.0], dtype=np.float64)
        self.fac_ptr = np.cumsum([0] + [len(f) for _, f in terms]).astype(np.int32)
        self.fac = np.array([i for _, f in terms for i in f] or [0], dtype=np.int32)
        self.nfac = int(self.fac_ptr[-1])
        self.nterms = len(terms)
        self.fmax = max([len(f) for _, f in terms] or [0])
        assert all(0 <= i < n_in for _, f in terms for i in f)

    @property
    def is_pairs(self):
        return all(1 <= len(f) <= 2 for o in self.outputs for _, f in o)

    def records(self):
        """The db_pair_term records, as evaluator.RHSPlan and sphere.SphereRHSPlan encode them."""
        rec = np.zeros(max(self.nterms, 1), dtype=PAIR_DTYPE)
        terms = [t for o in self.outputs for t in o]
        for k, (c, f) in enumerate(terms):
            rec[k] = (c, f[0], f[1] if len(f) == 2 else -1)
        return rec

    @classmethod
    def from_arrays(cls, n_in, term_ptr, coef, fac_ptr, fac):
        term_ptr, fac_ptr = np.asarray(term_ptr), np.asarray(fac_ptr)
        outs = []
        for o in range(len(term_ptr) - 1):
            outs.append([(float(coef[t]), [int(i) for i in fac[fac_ptr[t]:fac_ptr[t + 1]]]) for t in range(term_ptr[o], term_ptr[o + 1])])
        return cls(n_in, outs)


def random_program(rng, n_in, n_out, terms=(1, 12), factors=(1, 2), empty=(), pairs_edges=True):
    """Random program; outputs in `empty` have no terms.  With pairs_edges (and at least one factor allowed) the first output also
    holds the pair-record edges: input 0 as the second factor (b == 0), input n_in - 1 first and second, a repeated factor, and a
    single-factor term (b = -1)."""
    outs = []
    for o in range(n_out):
        if o in empty:
            outs.append([])
            continue
        nt = int(rng.integers(terms[0], terms[1] + 1))
        out = []
        for _ in range(nt):
            nf = int(rng.integers(factors[0], factors[1] + 1)) if n_in else 0
            out.append((float(rng.uniform(0.5, 2.0) * rng.choice([-1, 1])), [int(i) for i in rng.integers(0, n_in, nf)]))
        outs.append(out)
    if pairs_edges and n_in and factors[1] >= 1:
        o = next(k for k in range(n_out) if k not in empty)
        last = n_in - 1
        edges = [[last, 0], [0, last], [last, last], [last], [0]]
        if factors[1] >= 2:
            outs[o] += [(float(rng.uniform(0.5, 2.0)), e) for e in edges]
        else:
            outs[o] += [(-1.5, [last]), (0.75, [0])]
    return Program(n_in, outs)


# ------------------------------------------------------------------------------------------------------------------------------
# data and reference
# ------------------------------------------------------------------------------------------------------------------------------
def data(rng, kind, n_in, npoints, fmax=2):
    if kind == "random":
        return rng.standard_normal((n_in, npoints))
    if kind == "impulse":
        # every input 1 but for one point, a distinct value at a distinct point per input
        x = np.ones((n_in, npoints))
        for i in range(n_in):
            x[i, (37 * i + 5) % npoints] = 2.0 + i
        return x
    if kind == "wide":
        # exponents up to about 2^+-200, limited so that no product of fmax factors leaves the normal range
        E = min(200, 900 // max(fmax, 1))
        e = rng.integers(-E, E + 1, (n_in, npoints))
        return rng.uniform(1.0, 2.0, (n_in, npoints)) * rng.choice([-1.0, 1.0], (n_in, npoints)) * np.exp2(e.astype(np.float64))
    raise ValueError(kind)


def reference(prog, x):
    """(ref, bound, reads) over (n_out, npoints): ref and bound in long double; reads[o] = the inputs the terms of output o read."""
    npoints = x.shape[1]
    xl = x.astype(LD)
    ax = np.abs(xl)
    ref = np.zeros((prog.n_out, npoints), dtype=LD)
    mag = np.zeros_like(ref)
    reads = []
    for o, terms in enumerate(prog.outputs):
        r = set()
        for c, f in terms:
            p = np.full(npoints, LD(c))
            m = np.full(npoints, abs(LD(c)))
            for i in f:
                p = p * xl[i]
                m = m * ax[i]
                r.add(i)
            ref[o] += p
            mag[o] += m
        reads.append(r)
    T = np.array([len(t) for t in prog.outputs], dtype=LD)[:, None]
    bound = C_BOUND * (T + prog.fmax) * LD(EPS) * mag
    return ref, bound, reads


def check_products(path, prog, x, got):
    """got (n_out, npoints) against the reference.  Non-finite inputs: exactly the (output, point) entries whose terms read one are
    non-finite, every other entry within the bound."""
    with np.errstate(invalid="ignore", over="ignore"):
        ref, bound, reads = reference(prog, x)
    bad_in = ~np.isfinite(x)
    nonfin = np.zeros(got.shape, dtype=bool)
    for o, r in enumerate(reads):
        for i in r:
            nonfin[o] |= bad_in[i]
    assert np.isfinite(got[~nonfin]).all(), (path, "non-finite outputs", np.argwhere(~nonfin & ~np.isfinite(got))[:6])
    assert not np.isfinite(got[nonfin]).any(), (path, "finite where a non-finite input is read", np.argwhere(nonfin & np.isfinite(got))[:6])
    for o, terms in enumerate(prog.outputs):
        if not terms:
            assert np.all(got[o] == 0) and not np.signbit(got[o]).any(), (path, "an output without terms must be +0.0", o)
    ok = ~nonfin
    err = np.abs(got[ok].astype(LD) - ref[ok])
    b = bound[ok]
    zero = b == 0
    assert np.all(got[ok][zero] == 0), (path, "entries whose products are all exactly 0")
    ratio = float((err[~zero] / b[~zero]).max()) if (~zero).any() else 0.0
    RATIOS[path] = max(RATIOS.get(path, 0.0), ratio)
    assert ratio <= 1.0, (path, "error / bound", ratio)
    return ratio


# ------------------------------------------------------------------------------------------------------------------------------
# calls
# ------------------------------------------------------------------------------------------------------------------------------
def expected_kernel(prog, npoints, aligned=True):
    return K_V3 if npoints % 2 == 0 and aligned and prog.n_in <= MAX_IN_V3 else K_PW


def run_general(B, prog, x, misalign=(False, False), expect_rc=0):
    """db_pointwise on padded buffers.  Returns (outputs or None, kernel counts, the return code)."""
    n_in, npoints = prog.n_in, x.shape[1]
    xin = Padded(B, x, front=1 if misalign[0] else 2)
    out = nan_output(B, (prog.n_out, npoints), front=1 if misalign[1] else 2)
    arrs = [B.dev(a) for a in (prog.term_ptr, prog.coef, prog.fac_ptr, prog.fac)]
    rc, d = ran(B, lambda: B.lib._raw_db_pointwise(xin.p, out.p, npoints, n_in, prog.n_out, *[B.ptr(a) for a in arrs], prog.nfac, B.stream))
    assert rc == expect_rc, (rc, B.lib._raw_db_last_error())
    return out.result("pointwise"), d, rc


def run_pairs(B, prog, x, misalign=(False, False, False), expect_rc=0, records=None):
    """db_pointwise_pairs; misalign = (in, out, terms) 8 bytes past a 16-byte boundary."""
    n_in, npoints = prog.n_in, x.shape[1]
    xin = Padded(B, x, front=1 if misalign[0] else 2)
    out = nan_output(B, (prog.n_out, npoints), front=1 if misalign[1] else 2)
    rec = prog.records() if records is None else records
    tp = B.dev(prog.term_ptr)
    tr = B.dev_at(np.frombuffer(rec.tobytes(), dtype=np.uint8).copy(), misalign[2])
    rc, d = ran(B, lambda: B.lib._raw_db_pointwise_pairs(xin.p, out.p, npoints, n_in, prog.n_out, B.ptr(tp), B.ptr(tr), B.stream))
    assert rc == expect_rc, (rc, B.lib._raw_db_last_error())
    return out.result("pointwise_pairs"), d, rc


def check_program(B, prog, x, entries=("general", "pairs")):
    """Runs the program through the given entries on x; asserts the kernel and the bound.  Returns the outputs by entry."""
    got = {}
    npoints = x.shape[1]
    if "general" in entries:
        g, d, _ = run_general(B, prog, x)
        k = expected_kernel(prog, npoints)
        assert (d == one(k)).all(), ("expected", NAMES[k], d)
        check_products(NAMES[k], prog, x, g)
        got["general"] = g
    if "pairs" in entries:
        assert prog.is_pairs
        g, d, _ = run_pairs(B, prog, x)
        assert (d == one(K_PAIRS)).all(), d
        check_products(NAMES[K_PAIRS], prog, x, g)
        got["pairs"] = g
    return got


def last_error(B):
    return B.lib._raw_db_last_error().decode()


# ------------------------------------------------------------------------------------------------------------------------------
# hand-built programs
# ------------------------------------------------------------------------------------------------------------------------------
def check_inputs_count(B, n_in, npoints, seed=0):
    """A pair program and a general program (0 .. 6 factors) with n_in inputs, about 40 outputs with empty ones first, in the middle
    and last; random, impulse and wide-exponent data."""
    rng = np.random.default_rng(seed + 1000 * n_in + npoints)
    n_out = 40 if n_in >= 7 else 9
    empty = (0, n_out // 2, n_out - 1)
    progs = []
    if n_in == 0:
        progs.append((random_program(rng, 0, 5, terms=(1, 4), factors=(0, 0), empty=(2,)), ("general",)))
    else:
        pp = random_program(rng, n_in, n_out, terms=(1, 12), factors=(1, 2), empty=empty)
        pp.outputs[1] = pp.outputs[1] + [(float(rng.standard_normal()), [int(rng.integers(n_in))]) for _ in range(200 - len(pp.outputs[1]))]
        pp = Program(n_in, pp.outputs)                    # one output with 200 terms
        progs.append((pp, ("general", "pairs") if n_in <= MAX_IN_V3 and npoints % 2 == 0 else ("general",)))
        progs.append((random_program(rng, n_in, n_out // 2, terms=(1, 8), factors=(0, 6), empty=(0, n_out // 4, n_out // 2 - 1)),
                      ("general",)))
    for prog, entries in progs:
        for kind in ("random", "impulse", "wide"):
            check_program(B, prog, data(rng, kind, n_in, npoints, prog.fmax), entries)


def check_too_many_inputs(B):
    """114 inputs: db_pointwise returns 1 with the limit in its message, at odd and even npoints; nothing is written.  The pairs entry
    refuses 57 inputs."""
    rng = np.random.default_rng(114)
    prog = random_program(rng, MAX_IN + 1, 3, terms=(1, 3))
    for npoints in (255, 256):
        got, d, _ = run_general(B, prog, np.ones((MAX_IN + 1, npoints)), expect_rc=1)
        assert (d == 0).all() and np.isnan(got).all()
        assert "pointwise: too many inputs (114, at most 113)" in last_error(B), last_error(B)
    prog = random_program(rng, MAX_IN_V3 + 1, 3, terms=(1, 3))
    got, d, _ = run_pairs(B, prog, np.ones((MAX_IN_V3 + 1, 256)), expect_rc=1)
    assert (d == 0).all() and np.isnan(got).all()
    assert "at most 56 inputs" in last_error(B)


def check_odd_even_limit(B, n_in):
    """Regression: the general entry accepts the same inputs at odd and even npoints (k_pointwise beyond v3's 56 inputs)."""
    rng = np.random.default_rng(n_in)
    prog = random_program(rng, n_in, 5, terms=(1, 6), factors=(1, 3))
    for npoints in (999, 1000):
        check_program(B, prog, data(rng, "random", n_in, npoints), ("general",))


def check_small_shapes(B, npoints):
    """npoints 1, 2, 3, 255, 256, 257: partial tiles and odd against even."""
    rng = np.random.default_rng(npoints)
    prog = random_program(rng, 7, 6, terms=(1, 6), factors=(1, 2), empty=(3,))
    entries = ("general", "pairs") if npoints % 2 == 0 else ("general",)
    check_program(B, prog, data(rng, "random", 7, npoints), entries)
    gen = random_program(rng, 7, 4, terms=(1, 5), factors=(0, 6))
    check_program(B, gen, data(rng, "random", 7, npoints, gen.fmax), ("general",))


def check_nonfinite(B):
    """NaN and Inf at chosen points of chosen inputs: exactly the outputs whose terms read them turn non-finite there."""
    rng = np.random.default_rng(77)
    n_in, npoints = 9, 514
    outs = [[(1.0, [0, 1])], [(2.0, [2])], [(1.0, [3, 4]), (-1.0, [5])], [(0.5, [6, 6])], [(1.0, [7, 8]), (1.0, [0])], []]
    prog = Program(n_in, outs)
    x = data(rng, "random", n_in, npoints)
    x[1, 3] = np.nan
    x[4, 100] = np.inf
    x[6, 257] = -np.inf
    x[8, 513] = np.nan
    x[2, 0] = np.inf
    check_program(B, prog, x)
    check_program(B, prog, x[:, :-1].copy(), ("general",))   # odd: k_pointwise


def check_bitwise_v3_vs_pointwise(B):
    """The same program and data through k_pointwise_v3 and, with the input 8 bytes off a 16-byte boundary (or the output), through
    k_pointwise: bitwise equal."""
    rng = np.random.default_rng(5)
    for n_in, npoints, factors in ((7, 1000, (1, 2)), (29, 514, (0, 6)), (56, 258, (1, 4))):
        prog = random_program(rng, n_in, 12, terms=(1, 30), factors=factors, empty=(4,))
        x = data(rng, "random", n_in, npoints, prog.fmax)
        a, d, _ = run_general(B, prog, x)
        assert (d == one(K_V3)).all()
        for mis in ((True, False), (False, True)):
            b, d, _ = run_general(B, prog, x, misalign=mis)
            assert (d == one(K_PW)).all()
            assert np.array_equal(a, b), ("v3 != k_pointwise", np.abs(a - b).max())


def check_return_codes(B):
    """npoints <= 0 or n_out <= 0: 0 and nothing written.  Pairs: odd npoints, misaligned in / out / terms: 1 with the message, the
    output untouched."""
    rng = np.random.default_rng(3)
    prog = random_program(rng, 4, 3, terms=(1, 4))
    x = np.ones((4, 8))
    for npoints in (0, -2):
        for name, fn in (("general", lambda: B.lib._raw_db_pointwise(xin.p, out.p, npoints, 4, 3, *[B.ptr(a) for a in arrs], prog.nfac,
                                                                   B.stream)),
                         ("pairs", lambda: B.lib._raw_db_pointwise_pairs(xin.p, out.p, npoints, 4, 3, B.ptr(arrs[0]), B.ptr(rec), B.stream))):
            xin, out = Padded(B, x), nan_output(B, (3, 8))
            arrs = [B.dev(a) for a in (prog.term_ptr, prog.coef, prog.fac_ptr, prog.fac)]
            rec = B.dev(np.frombuffer(prog.records().tobytes(), dtype=np.uint8).copy())
            rc, d = ran(B, fn)
            assert rc == 0 and (d == 0).all() and np.isnan(out.result(name)).all()
    for name, fn in (("general", lambda: B.lib._raw_db_pointwise(xin.p, out.p, 8, 4, n_out, *[B.ptr(a) for a in arrs], prog.nfac, B.stream)),
                     ("pairs", lambda: B.lib._raw_db_pointwise_pairs(xin.p, out.p, 8, 4, n_out, B.ptr(arrs[0]), B.ptr(rec), B.stream))):
        for n_out in (0, -1):
            xin, out = Padded(B, x), nan_output(B, (3, 8))
            rc, d = ran(B, fn)
            assert rc == 0 and (d == 0).all() and np.isnan(out.result(name)).all()
    for mis, npoints, msg in (((False, False, False), 7, "needs an even point count"),
                              ((True, False, False), 8, "16-byte aligned arrays"),
                              ((False, True, False), 8, "16-byte aligned arrays"),
                              ((False, False, True), 8, "the term records must be 16-byte aligned")):
        got, d, _ = run_pairs(B, prog, np.ones((4, npoints)), misalign=mis, expect_rc=1)
        assert (d == 0).all() and np.isnan(got).all()
        assert msg in last_error(B), (msg, last_error(B))


# ------------------------------------------------------------------------------------------------------------------------------
# the grid-stride loops
# ------------------------------------------------------------------------------------------------------------------------------
def v3_grid(B, n_in, npoints):
    """(CTAs, tiles of the busiest CTA) of k_pointwise_v3 / k_pointwise_pairs: per_sm from shared memory, at most 8, times the SMs."""
    smem = 2 * n_in * PW3_T * 16
    per_sm = min(8, (226 * 1024) // (smem + 1024))
    tiles = -(-(npoints // 2) // PW3_T)
    blocks = min(tiles, B.sms * per_sm)
    return blocks, -(-tiles // blocks)


def pw_grid(B, npoints):
    tiles = -(-npoints // PW_TILE)
    blocks = min(tiles, B.sms * 8)
    return blocks, -(-tiles // blocks)


def stride_npoints(B, n_in, tiles_per_cta, partial=37):
    """An even npoints at which the busiest CTA of v3 / pairs takes `tiles_per_cta` tiles, the last one partial."""
    smem = 2 * n_in * PW3_T * 16
    cap = B.sms * min(8, (226 * 1024) // (smem + 1024))
    return 2 * (PW3_T * cap * (tiles_per_cta - 1) + PW3_T * (cap // 2 if tiles_per_cta > 1 else cap - 3) + partial)


def check_grid_stride_v3(B, tiles_per_cta, n_in=29, seed=0):
    rng = np.random.default_rng(seed + tiles_per_cta)
    npoints = stride_npoints(B, n_in, tiles_per_cta)
    blocks, tiles = v3_grid(B, n_in, npoints)
    assert tiles == tiles_per_cta and (npoints // 2) % PW3_T != 0, (blocks, tiles)
    if n_in >= 29:
        assert blocks <= B.sms
    prog = random_program(rng, n_in, 3, terms=(2, 5), factors=(1, 2), empty=(1,))
    check_program(B, prog, data(rng, "random", n_in, npoints))


def check_grid_stride_pointwise(B, tiles_per_cta, n_in=3, seed=0):
    """k_pointwise (the input 8 bytes off a boundary) with 1, 2 or 3 tiles per CTA, the last one partial."""
    rng = np.random.default_rng(seed + 10 * tiles_per_cta)
    cap = B.sms * 8
    npoints = PW_TILE * cap * (tiles_per_cta - 1) + PW_TILE * (cap // 2 if tiles_per_cta > 1 else cap - 3) + 41
    blocks, tiles = pw_grid(B, npoints)
    assert tiles == tiles_per_cta
    prog = random_program(rng, n_in, 2, terms=(2, 4), factors=(0, 3))
    x = data(rng, "random", n_in, npoints)
    got, d, _ = run_general(B, prog, x, misalign=(True, False))
    assert (d == one(K_PW)).all()
    check_products(NAMES[K_PW], prog, x, got)


# ------------------------------------------------------------------------------------------------------------------------------
# programs of real plans
# ------------------------------------------------------------------------------------------------------------------------------
def _np(t):
    return t.detach().cpu().numpy() if hasattr(t, "detach") else np.asarray(t)


def plan_program(plan):
    """(Program, npoints, pair records or None) of an RHS plan: RHSPlan (n_in), ComplexRHSPlan (2 n_in planes), SphereRHSPlan and
    ShellRHSPlan (n_g)."""
    from dedalus_b200.complex_path import ComplexRHSPlan
    if isinstance(plan, ComplexRHSPlan):
        n_in = 2 * plan.n_in
    else:
        n_in = plan.n_g if hasattr(plan, "n_g") else plan.n_in
    prog = Program.from_arrays(n_in, _np(plan.term_ptr), _np(plan.coef), _np(plan.fac_ptr), _np(plan.fac))
    pairs = getattr(plan, "pairs", None)
    rec = None if pairs is None else np.frombuffer(_np(pairs).tobytes(), dtype=PAIR_DTYPE)
    return prog, plan.npoints, rec


def check_plan(B, plan, seed=0, expect_pairs=None):
    prog, npoints, rec = plan_program(plan)
    assert prog.n_out > 0 and prog.nterms > 0
    if expect_pairs is not None:
        assert (rec is not None) == expect_pairs
    if rec is not None:
        # the byte records encode exactly the (term_ptr, coef, fac_ptr, fac) program
        assert prog.is_pairs and len(rec) == prog.nterms
        assert np.array_equal(rec, prog.records()), "pair records differ from the program"
    rng = np.random.default_rng(seed)
    x = data(rng, "random", prog.n_in, npoints)
    entries = ("general", "pairs") if prog.is_pairs and npoints % 2 == 0 and prog.n_in <= MAX_IN_V3 else ("general",)
    check_program(B, prog, x, entries if rec is None else ("general", "pairs"))
    return prog, npoints


# ------------------------------------------------------------------------------------------------------------------------------
# many passive tracers: the general entry past 56 inputs on an even grid
# ------------------------------------------------------------------------------------------------------------------------------
def tracer_solver(seeds, Nx=16, Nz=32, useed=11):
    """The 2-D shear flow of rhs_fused_cases with one passive tracer per seed: dt(c_k) - D lap(c_k) = - u@grad(c_k).  u from useed."""
    import dedalus_b200 as d3
    coords = d3.CartesianCoordinates('x', 'z')
    dist = d3.Distributor(coords, dtype=np.float64)
    xb = d3.RealFourier(coords['x'], size=Nx, bounds=(0, 1), dealias=3/2)
    zb = d3.RealFourier(coords['z'], size=Nz, bounds=(-1, 1), dealias=3/2)
    p = dist.Field(name='p', bases=(xb, zb))
    u = dist.VectorField(coords, name='u', bases=(xb, zb))
    tau_p = dist.Field(name='tau_p')
    cs = [dist.Field(name=f'c{k}', bases=(xb, zb)) for k in range(len(seeds))]
    ns = dict(u=u, p=p, tau_p=tau_p, nu=2e-5, D=3e-5, **{f'c{k}': c for k, c in enumerate(cs)})
    problem = d3.IVP([u, p, tau_p] + cs, namespace=ns)
    problem.add_equation("dt(u) + grad(p) - nu*lap(u) = - u@grad(u)")
    for k in range(len(cs)):
        problem.add_equation(f"dt(c{k}) - D*lap(c{k}) = - u@grad(c{k})")
    problem.add_equation("div(u) + tau_p = 0")
    problem.add_equation("integ(p) = 0")
    solver = problem.build_solver(d3.RK222)
    u['c'] = np.random.default_rng(useed).uniform(-1, 1, np.shape(u['c']))
    for s, c in zip(seeds, cs):
        c['c'] = np.random.default_rng(s).uniform(-1, 1, np.shape(c['c']))
    solver._init_device()
    return solver


def _eq_block(solver, arena, ie):
    off = solver.eq_arena.offsets[ie]
    tsh, shp = solver.eq_arena.shapes[ie]
    return arena[off:off + int(np.prod(tsh, dtype=int)) * int(np.prod(shp, dtype=int))]


def check_many_tracers(B, K=26, compare=(0, 13, 25)):
    """Regression: K = 26 tracers give 6 + 2 K = 58 inputs (u, grad u, and c_k's gradient per tracer), past v3's 56, on a 24 x 48
    grid.  The right-hand side evaluates, and each compared tracer's block equals the one-tracer problem with the same u and c_k."""
    import rhs_fused_cases as cases
    seeds = [100 + k for k in range(K)]
    solver = tracer_solver(seeds)
    plan = solver.rhs_plan
    assert MAX_IN_V3 < plan.n_in <= MAX_IN and plan.npoints % 2 == 0, (plan.n_in, plan.npoints)
    assert plan.pairs is None and plan.xprod is None
    before = launches(B)
    big = cases.evaluate(solver, False)
    assert (launches(B) - before)[K_PW] == 1
    for k in compare:
        one_solver = tracer_solver([seeds[k]])
        small = cases.evaluate(one_solver, one_solver.rhs_plan.use_x_products)
        a, b = _eq_block(solver, big, 1 + k), _eq_block(one_solver, small, 1)
        scale = np.abs(b).max()
        assert scale > 0 and a.shape == b.shape
        assert np.abs(a - b).max() <= 1e-13 * scale, (k, np.abs(a - b).max() / scale)
    # the velocity equation too
    assert np.abs(_eq_block(solver, big, 0) - _eq_block(one_solver, small, 0)).max() <= 1e-13 * np.abs(_eq_block(one_solver, small, 0)).max()


# ------------------------------------------------------------------------------------------------------------------------------
# transposes
# ------------------------------------------------------------------------------------------------------------------------------
TR_NAMES = ("db_transpose_pack", "db_transpose_unpack", "db_transpose_pack_rev", "db_transpose_unpack_rev")


def tr_shapes(mode, B_, nA, nB, n3, P):
    """(source shape, destination shape, numpy permutation source -> destination) of the header's layouts; (nA, nB) are the
    entry's (n1loc, n2), (n1, n2loc), (n1, n2loc), (n1loc, n2) for modes 0 .. 3."""
    if mode == 0:                       # A (B, n1loc, n2, n3) -> send (P, B, n1loc, n2blk, n3)
        blk = nB // P
        return (B_, nA, nB, n3), (P, B_, nA, blk, n3), lambda a: a.reshape(B_, nA, P, blk, n3).transpose(2, 0, 1, 3, 4)
    if mode == 1:                       # recv (P, B, n1blk, n2loc, n3) -> out (B, n1, n2loc, n3)
        blk = nA // P
        return (P, B_, blk, nB, n3), (B_, nA, nB, n3), lambda r: r.transpose(1, 0, 2, 3, 4).reshape(B_, nA, nB, n3)
    if mode == 2:                       # A (B, n1, n2loc, n3) -> send (P, B, n1blk, n2loc, n3)
        blk = nA // P
        return (B_, nA, nB, n3), (P, B_, blk, nB, n3), lambda a: a.reshape(B_, P, blk, nB, n3).transpose(1, 0, 2, 3, 4)
    blk = nB // P                       # recv (P, B, n1loc, n2blk, n3) -> out (B, n1loc, n2, n3)
    return (P, B_, nA, blk, n3), (B_, nA, nB, n3), lambda r: r.transpose(1, 2, 0, 3, 4).reshape(B_, nA, nB, n3)


def tr_clen(mode, nA, nB, n3, P):
    return (nB // P) * n3 if mode in (0, 3) else nB * n3


def run_transpose(B, mode, B_, nA, nB, n3, P, src, misalign=(False, False), expect_rc=0):
    _, dshape, _ = tr_shapes(mode, B_, nA, nB, n3, P)
    s = Padded(B, src, front=1 if misalign[0] else 2)
    d = nan_output(B, dshape, front=1 if misalign[1] else 2)
    rc, k = ran(B, lambda: getattr(B.lib, "_raw_" + TR_NAMES[mode])(s.p, d.p, B_, nA, nB, n3, P, B.stream))
    assert rc == expect_rc, (rc, last_error(B))
    return d.result(TR_NAMES[mode]), k


def distinct(rng, shape):
    n = int(np.prod(shape))
    return (np.arange(n) + rng.uniform(0.1, 0.9, n)).reshape(shape)


def check_transpose(B, mode, B_, nA, nB, n3, P, misalign=(False, False), seed=0):
    """One entry alone against the header's layout, bitwise; every destination element holds its own source value."""
    rng = np.random.default_rng(seed + 17 * mode + nA + nB + n3 + P)
    sshape, dshape, perm = tr_shapes(mode, B_, nA, nB, n3, P)
    src = distinct(rng, sshape)
    got, k = run_transpose(B, mode, B_, nA, nB, n3, P, src, misalign)
    clen = tr_clen(mode, nA, nB, n3, P)
    kind = K_TR16 if clen % 2 == 0 and not any(misalign) else K_TR8
    assert (k == one(kind)).all(), ("expected", NAMES[kind], k)
    ref = np.ascontiguousarray(perm(src))
    assert got.shape == ref.shape and np.array_equal(got, ref), (TR_NAMES[mode], np.argwhere(got != ref)[:4])
    return kind


def tr_small_cases():
    """(mode, B, nA, nB, n3, P): P 1, 2, 3, 8; B 1, 3; n3 1, 2, 5; split blocks of 2 and 3 rows (odd and even clen)."""
    out = []
    for mode in range(4):
        for P in (1, 2, 3, 8):
            for B_ in (1, 3):
                for n3 in (1, 2, 5):
                    blk = 2 if (P + B_ + n3) % 2 else 3
                    other = 2 + (P % 3)
                    nA, nB = (other, P * blk) if mode in (0, 3) else (P * blk, other)
                    out.append((mode, B_, nA, nB, n3, P))
    return out


def check_transpose_return_codes(B):
    """B, n1 or n3 = 0: 0 and nothing written; the split axis not divisible by P, and P < 1: 1 with the message."""
    for mode in range(4):
        for B_, nA, nB, n3 in ((0, 2, 4, 3), (2, 0, 4, 3) if mode in (0, 3) else (2, 4, 0, 3), (2, 2, 4, 0)):
            s = Padded(B, np.ones(16))
            d = nan_output(B, (16,))
            rc, k = ran(B, lambda: getattr(B.lib, "_raw_" + TR_NAMES[mode])(s.p, d.p, B_, nA, nB, n3, 2, B.stream))
            assert rc == 0 and (k == 0).all() and np.isnan(d.result("empty")).all()
        name = TR_NAMES[mode][3:]
        split = "n2" if mode in (0, 3) else "n1"
        for P, nA, nB, msg in ((3, 4, 4, f"{name}: {split} not divisible by P"), (0, 4, 4, f"{name}: P must be at least 1 (got 0)"),
                               (-2, 4, 4, f"{name}: P must be at least 1 (got -2)")):
            s = Padded(B, np.ones(64))
            d = nan_output(B, (64,))
            rc, k = ran(B, lambda: getattr(B.lib, "_raw_" + TR_NAMES[mode])(s.p, d.p, 2, nA, nB, 2, P, B.stream))
            assert rc == 1 and (k == 0).all() and np.isnan(d.result("rejected")).all()
            assert msg in last_error(B), (msg, last_error(B))


def check_transpose_misaligned(B):
    """Even clen with a base pointer 8 bytes off a 16-byte boundary on either side: the 8-byte branch, bitwise correct."""
    for mode in range(4):
        for mis in ((True, False), (False, True), (True, True)):
            for P, B_, n3 in ((2, 3, 2), (3, 1, 4)):
                nA, nB = (3, 2 * P) if mode in (0, 3) else (2 * P, 3)
                assert tr_clen(mode, nA, nB, n3, P) % 2 == 0
                assert check_transpose(B, mode, B_, nA, nB, n3, P, misalign=mis) == K_TR8


def exchange(sends):
    """all_to_all_single over P ranks: rank r receives block r of every rank's send buffer, in rank order."""
    P = len(sends)
    return [np.stack([sends[p][r] for p in range(P)]) for r in range(P)]


def check_transpose_round_trip(B, P, B_, n1loc, n2, n3, complex_=False, seed=0):
    """pack -> exchange -> unpack gives every rank its n2 block of the global array (B, n1, n2, n3); pack_rev -> exchange ->
    unpack_rev brings back the original split.  Bitwise; with complex_ the data is complex128 seen as (..., 2 n3) doubles."""
    rng = np.random.default_rng(seed + P * 7 + n3)
    n1, n2blk = P * n1loc, n2 // P
    if complex_:
        G = (rng.standard_normal((B_, n1, n2, n3)) + 1j * rng.standard_normal((B_, n1, n2, n3))).view(np.float64)
    else:
        G = rng.standard_normal((B_, n1, n2, n3))
    m3 = G.shape[3]
    A = [np.ascontiguousarray(G[:, r * n1loc:(r + 1) * n1loc]) for r in range(P)]
    sends = [run_transpose(B, 0, B_, n1loc, n2, m3, P, A[r])[0] for r in range(P)]
    recvs = exchange(sends)
    outs = [run_transpose(B, 1, B_, n1, n2blk, m3, P, recvs[r])[0] for r in range(P)]
    for r in range(P):
        assert np.array_equal(outs[r], G[:, :, r * n2blk:(r + 1) * n2blk]), ("forward hop", r)
    sends = [run_transpose(B, 2, B_, n1, n2blk, m3, P, outs[r])[0] for r in range(P)]
    recvs = exchange(sends)
    back = [run_transpose(B, 3, B_, n1loc, n2, m3, P, recvs[r])[0] for r in range(P)]
    for r in range(P):
        assert np.array_equal(back[r], A[r]), ("reverse hop", r)
    if complex_:
        assert np.array_equal(np.concatenate(back, axis=1).view(np.complex128), G.view(np.complex128))
