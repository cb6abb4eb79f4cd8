"""Shared bodies of the fused pencil-batch kernel tests (csrc/pencil.cu db_batches_*): assemble, factor, solve in every kernel
variant (db_batches_solve_set_mode), mat-vec, residual, gather and scatter, each against a plain long-double reference built on the
host from the batch's own matrices and programs.  They run through the CPU emulation of the kernels (tests/test_emu_pencil_batches.py)
and on the GPU (tests/test_gpu_1c_pencil_batches.py), on the work vectors of a real solver's BatchSet.

Every solve variant runs the same FMA sequence per pencil and member, so their solutions must agree bit for bit with the default
kernel: a difference is a race or an indexing error, never rounding.  Each check asserts from host data that its case reaches the
edges it is there for (control-block masks, ring wraps and partial stages, unstaged mat-vec blocks, long lines), so that a later
change of shapes cannot silently drop them."""
import ctypes as C
import numpy as np
from scipy.sparse.linalg import splu
from dedalus_b200 import lib as dlib
from dedalus_b200.pencils import assembly_program, line_maps
import program_interp as pi

U = np.finfo(np.float64).eps / 2
LD = np.longdouble
CE, FSTAGE_BYTES, MAX_SMEM, MV_R, MV_RECMAX = 16, 16 * 64 * 8 + 44 * 4, 227 * 1024, 32, 768
# (kernel, stages, chunks per stage, minb, prefetch, deep members) for db_batches_solve_set_mode; -1 = the environment's choice
WS_RINGS = ((2, 1), (3, 2), (3, 3), (8, 2), (3, 8))
VARIANTS = ([("ws", (0, st, cps, -1, -1, -1)) for st, cps in WS_RINGS]
            + [("flat", (1, st, -1, mb, -1, -1)) for mb in (2, 3, 4) for st in (2, 4, 16)]
            + [("pipe", (2, -1, -1, -1, -1, -1)), ("mr2", (3, -1, -1, -1, -1, -1)), ("mr4", (4, -1, -1, -1, -1, -1))]
            + [("deep", (5, -1, -1, -1, -1, m)) for m in (1, 2, 4)])
NVECS = (0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 12, 13, 16)


class Case:
    """A solver's BatchSet with its LHS a0 M + b0 L factorised into LU slot 0, and host references per batch."""

    def __init__(self, solver, a0, b0):
        import torch
        self.torch = torch
        self.solver, self.a0, self.b0 = solver, a0, b0
        solver._init_device()
        solver._prepare_batches(a0, b0)
        self.bs = bs = solver.bset
        self.lib = solver.lib
        self.dev = solver.device
        self.desc = bs.desc
        self.nslots = bs.nslots
        assert self.nslots >= 6
        self._A = {}
        bs.factor(0, a0, b0)
        bs.check_info()

    # ---- plumbing
    def call(self, name, *args, desc=None):
        d = self.desc if desc is None else desc
        self.lib.call(name, d.data_ptr(), self.bs.nb, *args, self.solver.stream())

    def host(self, t):
        return t.detach().cpu().numpy().copy()

    def put(self, t, a):
        t.copy_(self.torch.from_numpy(np.ascontiguousarray(a)))

    def vec(self, db, slot):
        """(R_alloc, n, ld) host view of a work vector: member, row, pencil."""
        return pi.from_tiles(self.host(db.vecs[slot]), db.n, db.ld * db.R_alloc).reshape(db.n, db.R_alloc, db.ld).transpose(1, 0, 2)

    def set_vec(self, db, slot, v):
        flat = np.ascontiguousarray(v.transpose(1, 0, 2)).reshape(db.n, db.R_alloc * db.ld)
        self.put(db.vecs[slot], pi.to_tiles(flat))

    def random_vecs(self, slots, seed, padding=0.0):
        """Random values in every member and pencil of the given slots; padding lanes (s >= S) and members past R get `padding`."""
        rng = np.random.default_rng(seed)
        for db in self.bs.items:
            for slot in slots:
                v = np.full((db.R_alloc, db.n, db.ld), padding)
                v[:db.R, :, :db.S] = rng.standard_normal((db.R, db.n, db.S))
                self.set_vec(db, slot, v)

    def matrix(self, db, s):
        """(a0 M + b0 L, M, L) of pencil s in the batch's solver ordering, as scipy CSR."""
        key = (id(db), s)
        if key not in self._A:
            g = db.batch.groups[s]
            M, L = db.batch.matrix('M', g).tocsr(), db.batch.matrix('L', g).tocsr()
            self._A[key] = ((self.a0 * M + self.b0 * L).tocsr(), M, L)
        return self._A[key]

    def solve(self, x_slot, terms, lu_slot=0, desc=None, max_nrhs=None):
        sc = dlib.SlotComb()
        sc.nvec = len(terms)
        for j, (slot, coef) in enumerate(terms):
            sc.slot[j], sc.coef[j] = slot, coef
        self.call("db_batches_solve", self.bs.blocks['solve'], self.bs.max_nrhs if max_nrhs is None else max_nrhs, lu_slot, x_slot,
                  C.byref(sc), desc=desc)

    def set_mode(self, *mode):
        self.lib.call("db_batches_solve_set_mode", *mode)

    def reset_mode(self):
        self.lib.call("db_batches_solve_set_mode", -1, -1, -1, -1, -1, -1)

    def lu(self, db, slot=0):
        return pi.from_tiles(self.host(db.lu_tensor(slot)), db.prog.nE, db.ld)

    def nchunks(self, db):
        return db.prog.nE // CE


# ---------------------------------------------------------------------------------------------------------------------------------
# assemble and factor
# ---------------------------------------------------------------------------------------------------------------------------------
def assembled_reference(db, a0, b0):
    """Long-double sum_t val_t mono_t per LU entry and the bound 4 u sum_t |val_t mono_t|, (nE, S)."""
    ptr, mono, val = (np.asarray(a) for a in assembly_program(db.batch, db.prog, a0, b0))
    entry = np.repeat(np.arange(len(ptr) - 1), np.diff(ptr))
    terms = val.astype(LD)[:, None] * np.asarray(db.prog.mono_vals, dtype=LD)[mono]
    ref = np.zeros((len(ptr) - 1, db.S), dtype=LD)
    mag = np.zeros_like(ref)
    np.add.at(ref, entry, terms)
    np.add.at(mag, entry, np.abs(terms))
    return ref, 4 * U * mag


def check_assemble_factor(case):
    a0, b0, bs = case.a0, case.b0, case.bs
    for db in bs.items:
        db.set_lhs(a0, b0)
        db.info.zero_()
        case.put(db.lu_tensor(0), np.full(db.prog.nE * db.ld, np.nan))
    case.call("db_batches_assemble", bs.blocks['asm'], 0)
    assembled = [case.lu(db) for db in bs.items]
    case.call("db_batches_factor", bs.blocks['solve'], 0)
    for db, asm in zip(bs.items, assembled):
        tag = dict(n=db.n, S=db.S, R=db.R)
        ref, bound = assembled_reference(db, a0, b0)
        assert np.all(np.abs(asm[:, :db.S] - ref) <= bound), (tag, "assemble", float(np.abs(asm[:, :db.S] - ref).max()))
        assert np.isnan(asm[:, db.S:]).all(), (tag, "assemble wrote a padding lane")
        lu_ref = pi.factor(db.prog, asm[:, :db.S].astype(LD))
        lu = case.lu(db)[:, :db.S]
        scale = np.abs(lu_ref).max(axis=0)
        err = (np.abs(lu - lu_ref) / scale).max()
        # the static pivot order lets a few pencils cancel in a pivot (RB2D, S = 79: 2.6e-11); there a plain double replay of the same
        # program is as far from the long-double one, and the kernel may not be further than 4 times that
        err64 = (np.abs(pi.factor(db.prog, asm[:, :db.S].copy()) - lu_ref) / scale).max()
        assert err <= max(1e-12, 4 * err64), (tag, "factor", float(err), float(err64))
        assert int(db.info.item()) == 0, tag
    for db in bs.items:                                  # back to the solver's state: zero padding lanes
        case.put(db.lu_tensor(0), np.zeros(db.prog.nE * db.ld))
    bs.factor(0, a0, b0)


def check_factor_info(case):
    """info counts exactly the pencils that meet a zero or non-finite pivot: NaN monomials in one pencil of the first batch, a0 = b0 = 0
    in the last batch (every pencil), nothing elsewhere."""
    bs = case.bs
    assert bs.nb >= 2
    first, last = bs.items[0], bs.items[-1]
    s_bad = first.S // 2
    mono = case.host(first.t['mono'])
    saved = mono.copy()
    mono.reshape(-1, first.ld)[:, s_bad] = np.nan
    case.put(first.t['mono'], mono)
    try:
        for db in bs.items:
            db.set_lhs(case.a0, case.b0)
            db.info.zero_()
        last.set_lhs(0.0, 0.0)
        case.call("db_batches_assemble", bs.blocks['asm'], 0)
        case.call("db_batches_factor", bs.blocks['solve'], 0)
        got = [int(db.info.item()) for db in bs.items]
        want = [1 if db is first else db.S if db is last else 0 for db in bs.items]
        assert got == want, (got, want)
    finally:
        case.put(first.t['mono'], saved)
        bs.factor(0, case.a0, case.b0)
        bs.check_info()


# ---------------------------------------------------------------------------------------------------------------------------------
# solve
# ---------------------------------------------------------------------------------------------------------------------------------
def combined_rhs(case, db, terms):
    """Long-double sum_j coef_j vec[slot_j], (R_alloc, n, ld)."""
    b = np.zeros((db.R_alloc, db.n, db.ld), dtype=LD)
    cache = {}
    for slot, coef in terms:
        if slot not in cache:
            cache[slot] = case.vec(db, slot).astype(LD)
        b += LD(coef) * cache[slot]
    return b


def _ld_matvec(A, x):
    """A x in long double for scipy CSR A and x (n,) or (n, k)."""
    A = A.tocsr()
    data = A.data.astype(LD)
    rows = np.repeat(np.arange(A.shape[0]), np.diff(A.indptr))
    x = np.asarray(x, dtype=LD)
    prod = data.reshape((-1,) + (1,) * (x.ndim - 1)) * x[A.indices]
    y = np.zeros((A.shape[0],) + x.shape[1:], dtype=LD)
    np.add.at(y, rows, prod)
    return y


def refined_solve(A, b):
    """LAPACK (SuperLU) solve of A x = b, then two refinement steps with residuals in long double."""
    lu = splu(A.tocsc())
    x = lu.solve(np.asarray(b, dtype=np.float64)).astype(LD)
    for _ in range(2):
        r = np.asarray(b, dtype=LD) - _ld_matvec(A, x)
        x = x + lu.solve(r.astype(np.float64)).astype(LD)
    return x


def check_solution(case, x_slot, terms, pencils=None, forward=True, desc_nrhs=None):
    """Normwise long-double backward error <= 1e-12 per pencil and member; x within 1e-9 of a refined solve; returns the worst
    backward error.  pencils: {batch index: pencil indices} (default: all)."""
    worst = 0.0
    for i, db in enumerate(case.bs.items):
        R = db.R if desc_nrhs is None else desc_nrhs[i]
        x_all = case.vec(db, x_slot)
        b_all = combined_rhs(case, db, terms)
        for s in (range(db.S) if pencils is None else pencils[i]):
            A = case.matrix(db, s)[0]
            x, b = x_all[:R, :, s].T.astype(LD), b_all[:R, :, s].T            # (n, R)
            r = b - _ld_matvec(A, x)
            anorm = LD(np.abs(A).sum(axis=1).max())
            be = np.abs(r).max(axis=0) / (anorm * np.abs(x).max(axis=0) + np.abs(b).max(axis=0))
            be = float(np.nan_to_num(be.astype(np.float64), nan=np.inf).max())
            assert be <= 1e-12, (dict(n=db.n, S=db.S, R=R, s=s), "backward error", be)
            worst = max(worst, be)
            if forward:
                xr = refined_solve(A, b)
                err = float(np.abs(x - xr).max() / max(np.abs(xr).max(), LD(1e-300)))
                assert err <= 1e-9, (dict(n=db.n, S=db.S, s=s), "x vs refined solve", err)
    return worst


def solve_coverage(case, rings):
    """Host facts about the solve streams: control-block masks, and for each (stages, cps) ring the stage counts."""
    cov = dict(maskF=0, maskF2=0, maskR=0, maskG=0, pure=0, short=False, partial=False, wraps=0)
    for db in case.bs.items:
        ctrl = np.asarray(db.prog.ctrl)
        for name, w in (("maskF", 34), ("maskF2", 35), ("maskR", 36), ("maskG", 37)):
            cov[name] += int((ctrl[:, w] != 0).sum())
        cov["pure"] += int(((ctrl[:, 33] | ctrl[:, 34]) == 0).sum())
        nch = case.nchunks(db)
        for st, cps in rings:
            nst = -(-nch // cps)
            cov["short"] |= nst < st
            cov["partial"] |= nch % cps != 0
            cov["wraps"] = max(cov["wraps"], nst // st)
    return cov


def default_solve(case, terms, x_slot=0, padding=0.0, seed=11):
    case.random_vecs({s for s, _ in terms}, seed, padding=padding)
    case.put_nan(x_slot)
    case.reset_mode()
    case.solve(x_slot, terms)
    return [case.vec(db, x_slot) for db in case.bs.items]


def _put_nan(self, slot):
    for db in self.bs.items:
        self.put(db.vecs[slot], np.full(db.n * db.ld * db.R_alloc, np.nan))


Case.put_nan = _put_nan


def same_bits(case, a, b, R=None):
    for i, (db, xa, xb) in enumerate(zip(case.bs.items, a, b)):
        r = db.R if R is None else R[i]
        va, vb = xa[:r, :, :db.S], xb[:r, :, :db.S]
        if va.tobytes() != vb.tobytes():
            bad = np.argwhere(va.view(np.uint64) != vb.view(np.uint64))
            return dict(batch=i, n=db.n, S=db.S, R=r, first=bad[0].tolist(), count=len(bad))
    return None


TERMS = [(1, 1.0), (2, -0.37), (3, 0.5)]


def check_solve_default(case, pencils=None):
    """The default kernel against the long-double references; padding lanes stay finite and never reach valid columns.
    Returns the worst backward error."""
    x = default_solve(case, TERMS)
    worst = check_solution(case, 0, TERMS, pencils)
    x_pad = default_solve(case, TERMS, padding=3.0)
    assert same_bits(case, x, x_pad) is None, "padding lanes changed a valid column"
    for db, v in zip(case.bs.items, x_pad):
        assert np.isfinite(v[:db.R, :, db.S:]).all(), "padding lane of x not finite"
    return worst


def check_solve_variants(case, variants=VARIANTS):
    """Every kernel variant gives the default kernel's x bit for bit."""
    ref = default_solve(case, TERMS)
    failures = []
    try:
        for name, mode in variants:
            case.put_nan(0)
            case.set_mode(*mode)
            case.solve(0, TERMS)
            got = [case.vec(db, 0) for db in case.bs.items]
            diff = same_bits(case, ref, got)
            if diff:
                failures.append((name, mode, diff))
    finally:
        case.reset_mode()
    assert not failures, failures


def check_solve_mixed_nrhs(case, variants=VARIANTS):
    """One launch with a batch whose nrhs is lowered to 3 (below max_nrhs = 4) in a copy of the descriptor: members 0 .. 2 are solved
    as before, bitwise in every variant, and the fourth is left alone."""
    import torch
    bs = case.bs
    four = [i for i, db in enumerate(bs.items) if db.R == 4]
    assert four and bs.max_nrhs == 4
    assert len({db.n for db in bs.items}) > 1 and any(db.R < 4 for db in bs.items)
    arr = (dlib.Batch * bs.nb)()
    C.memmove(arr, C.addressof(bs.host_desc), C.sizeof(arr))
    arr[four[0]].nrhs = 3
    desc = torch.from_numpy(np.frombuffer(bytes(arr), dtype=np.uint8).copy()).to(case.dev)
    R = [db.R for db in bs.items]; R[four[0]] = 3
    ref = default_solve(case, TERMS)
    failures = []
    try:
        for name, mode in [("default", (-1,) * 6)] + list(variants):
            case.put_nan(0)
            case.set_mode(*mode)
            case.solve(0, TERMS, desc=desc)
            got = [case.vec(db, 0) for db in bs.items]
            diff = same_bits(case, ref, got, R)
            if diff:
                failures.append((name, mode, diff))
            if name not in ("mr2", "mr4"):          # the members-in-registers kernels solve whole groups of members
                assert np.isnan(got[four[0]][3]).all(), (name, "member past nrhs was written")
    finally:
        case.reset_mode()
    assert not failures, failures


def check_rhs_combinations(case):
    """nvec = 0 .. 16 terms (every NV template and the counts rounded up inside them), zero coefficients, a repeated slot."""
    slots = (1, 2, 3, 4)
    case.random_vecs(slots, 5)
    for nv in NVECS:
        terms = [(slots[j % 4] if j != 5 else 1, (0.0 if j % 7 == 3 else (-1) ** j * (0.25 + 0.125 * j))) for j in range(nv)]
        case.put_nan(0)
        if nv == 0:
            # the kernels pad the combination with zero-coefficient copies of the first term: an empty one is rejected
            try:
                case.solve(0, terms)
            except dlib.DedalusB200Error as exc:
                assert "bad arguments" in str(exc)
            else:
                raise AssertionError("an empty right-hand side was accepted")
            continue
        case.solve(0, terms)
        pencils = {i: sorted({0, db.S - 1, db.S // 2}) for i, db in enumerate(case.bs.items)}
        check_solution(case, 0, terms, pencils, forward=False)


# ---------------------------------------------------------------------------------------------------------------------------------
# mat-vec, residual, move
# ---------------------------------------------------------------------------------------------------------------------------------
def matvec_coverage(case):
    cov = dict(unstaged=0, out_of_window=0, ragged_n=False)
    for db in case.bs.items:
        mp, lp = (np.asarray(db.prog.mv[k][0]) for k in ('M', 'L'))
        for r0 in range(0, db.n, MV_R):
            r1 = min(r0 + MV_R, db.n)
            if (mp[r1] - mp[r0]) + (lp[r1] - lp[r0]) > MV_RECMAX:
                cov["unstaged"] += 1
        for k in ('m', 'l'):
            split, ptr = case.host(db.t[k + '_split']), np.asarray(db.prog.mv[k.upper()][0])
            cov["out_of_window"] += int((split < ptr[1:]).sum())
        cov["ragged_n"] |= db.n % MV_R != 0
    return cov


def matvec_reference(db, name, x):
    """Long-double y = sum_t val_t mono_t x[col_t] and sum_t |val_t mono_t x[col_t]| for x (R, n, S)."""
    ptr, col, mono, val = (np.asarray(a) for a in db.prog.mv[name])
    rows = np.repeat(np.arange(db.n), np.diff(ptr))
    coef = val.astype(LD)[:, None] * np.asarray(db.prog.mono_vals, dtype=LD)[mono]          # (T, S)
    y = np.zeros(x.shape, dtype=LD); mag = np.zeros(x.shape, dtype=LD)
    for m in range(x.shape[0]):
        t = coef * x[m][col].astype(LD)
        np.add.at(y[m], rows, t)
        np.add.at(mag[m], rows, np.abs(t))
    return y, mag, np.diff(ptr)


def check_matvec(case):
    bs = case.bs
    case.random_vecs([1], 21)
    for ym, yl in ((4, -1), (-1, 5), (4, 5)):
        case.put_nan(4); case.put_nan(5)
        case.call("db_batches_matvec", bs.blocks['matvec'], 1, ym, yl)
        for db in bs.items:
            x = case.vec(db, 1)[:db.R, :, :db.S]
            for name, slot in (("M", ym), ("L", yl)):
                got = case.vec(db, 4 if name == "M" else 5)
                if slot < 0:
                    assert np.isnan(got).all(), (name, "skipped product was written")
                    continue
                ref, mag, nt = matvec_reference(db, name, x)
                bound = (nt[None, :, None] + 2) * U * mag
                err = np.abs(got[:db.R, :, :db.S] - ref)
                assert np.all(err <= bound), (dict(n=db.n, S=db.S), name, float((err - bound).max()))


def check_residual(case):
    """db_batches_residual against the same formula in long double; a NaN / inf in one member gives +inf for that pencil only;
    a pencil with b = Mx = Lx = 0 gives 0; padding lanes give 0."""
    bs, a0, b0 = case.bs, case.a0, case.b0
    case.random_vecs([1, 2, 3], 31, padding=7.0)
    poison = {}
    for i, db in enumerate(bs.items):
        if i == 0:
            v = case.vec(db, 2); v[db.R - 1, db.n // 2, 1] = np.nan; case.set_vec(db, 2, v); poison[(i, 1)] = np.inf
        if i == 1:
            v = case.vec(db, 3); v[0, 0, 2] = np.inf; case.set_vec(db, 3, v); poison[(i, 2)] = np.inf
        if i == bs.nb - 1:
            for slot in (1, 2, 3):
                v = case.vec(db, slot); v[:, :, 0] = 0.0; case.set_vec(db, slot, v)
            poison[(i, 0)] = 0.0
    nblk = bs.blocks['solve']
    out = case.torch.full((nblk * 64,), np.nan, dtype=case.torch.float64, device=case.dev)
    case.call("db_batches_residual", nblk, 1, 2, 3, float(a0), float(b0), out.data_ptr())
    out = case.host(out)
    start = 0
    for i, db in enumerate(bs.items):
        got = out[start:start + ((db.S + 63) // 64) * 64]
        start += len(got)
        assert not got[db.S:].any(), "padding lanes"
        b, m, l = (case.vec(db, s)[:db.R, :, :db.S].astype(LD) for s in (1, 2, 3))
        mv, lv = LD(a0) * m, LD(b0) * l
        r = (mv + lv) - b
        with np.errstate(invalid='ignore'):
            den = np.abs(b).max(axis=1) + np.abs(mv).max(axis=1) + np.abs(lv).max(axis=1)
            ref = np.where(den > 0, np.abs(r).max(axis=1) / np.where(den > 0, den, 1), 0).max(axis=0)
        for s in range(db.S):
            if (i, s) in poison:
                assert got[s] == poison[(i, s)], (i, s, got[s])
            else:
                assert abs(got[s] - ref[s]) <= 1e-14 * ref[s] + 1e-300, (i, s, got[s], float(ref[s]))


def check_move(case):
    """Gather and scatter of every member (line signs) on both sides, bitwise against program_interp."""
    bs, solver = case.bs, case.solver
    rng = np.random.default_rng(41)
    cov = dict(long_lines=False, ragged_S=False)
    for side, arena in ((0, solver.var_arena), (1, solver.eq_arena)):
        src = rng.standard_normal(arena.size)
        t = case.torch.from_numpy(src.copy()).to(case.dev)
        case.random_vecs([4], 43)
        case.call("db_batches_move", bs.blocks[f'move{side}'], side, 1, 4, t.data_ptr())
        case.random_vecs([5], 44)
        out = case.torch.zeros(arena.size, dtype=case.torch.float64, device=case.dev)
        case.call("db_batches_move", bs.blocks[f'move{side}'], side, 0, 5, out.data_ptr())
        out = case.host(out)
        ref_out = np.zeros(arena.size)
        for db in bs.items:
            maps = line_maps(db.batch, arena, 'cols' if side == 0 else 'rows')
            cov["long_lines"] |= int(np.max(maps.line_len)) > 64
            cov["ragged_S"] |= db.S % 64 != 0
            got = case.vec(db, 4)
            x5 = case.vec(db, 5)
            for c in range(db.R):
                ref = pi.gather(maps, src, db.n, db.S, member=c)
                assert got[c, :, :db.S].tobytes() == ref.tobytes(), (side, c, "gather")
                pi.scatter(maps, x5[c, :, :db.S], ref_out, member=c)
        assert out.tobytes() == ref_out.tobytes(), (side, "scatter")
    return cov


def check_set_mode_rejects(case):
    """Out-of-range fields, a deep ring shorter than its prefetch distance and a ring beyond the shared-memory opt-in limit are
    rejected by the ABI, never launched; the default selection is back afterwards."""
    bad = [(6, -1, -1, -1, -1, -1), (0, 1, -1, -1, -1, -1), (0, 25, -1, -1, -1, -1), (0, -1, 0, -1, -1, -1), (0, -1, 9, -1, -1, -1),
           (1, -1, -1, 5, -1, -1), (-1, -1, -1, -1, 3, -1), (5, -1, -1, -1, -1, 3), (5, 4, -1, -1, -1, -1), (0, 5, 8, -1, -1, -1)]
    assert all(st * cps * FSTAGE_BYTES <= MAX_SMEM for st, cps in WS_RINGS) and 5 * 8 * FSTAGE_BYTES > MAX_SMEM
    try:
        for mode in bad:
            try:
                case.set_mode(*mode)
            except dlib.DedalusB200Error as exc:
                assert "batches_solve_set_mode" in str(exc), (mode, exc)
            else:
                raise AssertionError(f"db_batches_solve_set_mode{mode} was accepted")
        # a ring left to the environment's kernel (the warp-specialised one) is checked by the solve
        case.set_mode(-1, 24, 8, -1, -1, -1)
        try:
            case.solve(0, TERMS)
        except dlib.DedalusB200Error as exc:
            assert "shared memory" in str(exc), exc
        else:
            raise AssertionError("a 24 x 8-chunk ring was launched")
    finally:
        case.reset_mode()


def assert_coverage(cases):
    """The edges the checks above are there for, asserted from host data over a list of cases."""
    cov = [solve_coverage(c, WS_RINGS + ((8, 2),)) for c in cases]
    for key in ("maskF", "maskF2", "maskR", "maskG", "pure"):
        assert sum(c[key] for c in cov) > 0, ("no chunk with", key)
    assert any(c["short"] for c in cov), "no batch with fewer stages to stream than the ring holds"
    assert any(c["partial"] for c in cov), "no batch whose chunks leave a partial last stage"
    assert max(c["wraps"] for c in cov) >= 2, "no batch wraps the ring twice"
    items = [db for c in cases for db in c.bs.items]
    assert any(db.S < 64 for db in items) and any(db.S > 64 and db.S % 64 for db in items), sorted({db.S for db in items})
    mixed = [c for c in cases if c.bs.max_nrhs == 4 and len({db.n for db in c.bs.items}) > 1 and any(db.R < 4 for db in c.bs.items)]
    assert mixed, "no launch mixes batches of different n and nrhs"
    mv = [matvec_coverage(c) for c in cases]
    assert sum(m["unstaged"] for m in mv) > 0, "no row block takes the unstaged mat-vec path"
    assert sum(m["out_of_window"] for m in mv) > 0 and any(m["ragged_n"] for m in mv)
    lines = [int(np.max(line_maps(db.batch, c.solver.var_arena, 'cols').line_len)) for c in cases for db in c.bs.items]
    assert max(lines) > 64, "no line longer than one 64-element move tile"
