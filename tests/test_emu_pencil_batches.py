"""The fused pencil-batch kernels (csrc/pencil.cu db_batches_*) through the CPU emulation, against long-double references, with every
solve variant bitwise equal to the default; GPU version: tests/test_gpu_1c_pencil_batches.py.  The emulation lands bulk copies only
when a thread waits on their mbarrier (DB_EMU_BULK=late) and cp.async copies only when their group retires (DB_EMU_CP=late), so a
ring stage or gather read too early holds poison here.

Problems: RB3D 8 x 8 x 12 (8 factorisation sets of 1, 2 and 4 members, short rings), the tall 4 x 4 x 256 pencils (n up to 1288,
dense boundary rows: unstaged mat-vec blocks, lines longer than 64, many ring wraps) and RB2D at Nh = 160 (S = 79 and S = 1).  All use
DB_SOLVE_ORDER=natural, which puts more than 16 row ends within three chunks, so the deep kernel's global re-reads (maskG) occur."""
import numpy as np, pytest
from emu import emu_lib as E
import pencil_batch_cases as PB
import dedalus_b200 as d3
from dedalus_b200 import examples

GAMMA = (2 - np.sqrt(2)) / 2
PROBLEMS = dict(rb3d=dict(dim=3, Nh=8, Nz=12), tall=dict(dim=3, Nh=4, Nz=256), rb2d=dict(dim=2, Nh=160, Nz=8))


@pytest.fixture(scope="module", autouse=True)
def emulation():
    E.install()
    yield
    E.uninstall()


@pytest.fixture(scope="module")
def cases(emulation):
    mp = pytest.MonkeyPatch()
    mp.setenv("DB_SOLVE_ORDER", "natural")            # read by compile_batch
    built = {}
    try:
        for name, kw in PROBLEMS.items():
            built[name] = PB.Case(examples.rayleigh_benard(**kw)['problem'].build_solver(d3.RK222), 1.0, 0.01 * GAMMA)
    finally:
        mp.undo()
    return built


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
