"""The fused pencil-batch kernels on the GPU: the cases of tests/test_emu_pencil_batches.py (same bodies, pencil_batch_cases.py), and
the 256^3 RB3D batch set, whose default solve configuration is the benchmark's: the default kernel against the long-double references
on the first, a middle and the last (partial) tile of every batch, and every variant bitwise equal to it.  This guards against
regressions; it does not repeat runs to catch a race whose timing is unknown."""
import numpy as np, pytest
import pencil_batch_cases as PB
import dedalus_b200 as d3
from dedalus_b200 import examples

pytestmark = pytest.mark.gpu
GAMMA = (2 - np.sqrt(2)) / 2
PROBLEMS = dict(rb3d=dict(dim=3, Nh=8, Nz=12), tall=dict(dim=3, Nh=4, Nz=256), rb2d=dict(dim=2, Nh=160, Nz=8))


@pytest.fixture(scope="module")
def cases():
    mp = pytest.MonkeyPatch()
    mp.setenv("DB_SOLVE_ORDER", "natural")
    try:
        return {name: PB.Case(examples.rayleigh_benard(**kw)['problem'].build_solver(d3.RK222), 1.0, 0.01 * GAMMA)
                for name, kw in PROBLEMS.items()}
    finally:
        mp.undo()


@pytest.fixture(params=list(PROBLEMS))
def case(request, cases):
    return cases[request.param]


def test_cases_reach_the_edges(cases):
    PB.assert_coverage(list(cases.values()))


def test_assemble_and_factor(case):
    PB.check_assemble_factor(case)
    PB.check_factor_info(case)


def test_default_solve(case):
    print("worst backward error", PB.check_solve_default(case))


def test_solve_variants_bitwise(case):
    PB.check_solve_variants(case)


def test_solve_mixed_nrhs(cases):
    PB.check_solve_mixed_nrhs(cases["rb3d"])


def test_rhs_combinations(case):
    PB.check_rhs_combinations(case)


def test_matvec(case):
    PB.check_matvec(case)


def test_residual(case):
    PB.check_residual(case)


def test_move(case):
    PB.check_move(case)


def test_set_mode_rejects(cases):
    PB.check_set_mode_rejects(cases["rb2d"])


@pytest.fixture(scope="module")
def rb3d_256():
    pb = examples.rayleigh_benard(dim=3, Nh=256, Nz=256)
    return PB.Case(pb['problem'].build_solver(d3.RK222), 1.0, 0.01 * GAMMA)


def _sample(db):
    tiles = (db.S + 63) // 64
    out = set()
    for t in sorted({0, tiles // 2, tiles - 1}):
        out |= set(range(t * 64, min(db.S, t * 64 + 64), 4)) | {min(db.S, t * 64 + 64) - 1}
    return sorted(out)


def test_rb3d_256_default_solve(rb3d_256):
    """The benchmark's batch set and solve configuration against the long-double references."""
    PB.default_solve(rb3d_256, PB.TERMS)
    worst = PB.check_solution(rb3d_256, 0, PB.TERMS, {i: _sample(db) for i, db in enumerate(rb3d_256.bs.items)})
    print("worst backward error at 256^3", worst)


def test_rb3d_256_variants_bitwise(rb3d_256):
    PB.check_solve_variants(rb3d_256)
