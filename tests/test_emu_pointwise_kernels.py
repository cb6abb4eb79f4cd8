"""The grid products and transposes of csrc/pointwise.cu -- db_pointwise (k_pointwise, k_pointwise_v3), db_pointwise_pairs and the four
db_transpose_* entries -- through the CPU emulation of the kernels, against long-double references and the header's layouts; GPU
version: tests/test_gpu_1f_pointwise_kernels.py.  Shared bodies and bounds: tests/pointwise_kernel_cases.py."""
import os, subprocess, sys, pathlib
import numpy as np, pytest
from emu import emu_lib as E
from kernel_backends import EmuArrays
import pointwise_kernel_cases as K

ROOT = pathlib.Path(__file__).resolve().parents[1]
B = EmuArrays()
_SUB = "DB_POINTWISE_SUBPROCESS"


@pytest.fixture(autouse=True)
def emulation():
    E.install()
    yield
    E.uninstall()


@pytest.fixture(scope="module", autouse=True)
def ratio_report():
    yield
    print("\nlargest error / bound per kernel (C_BOUND = %g):\n%s" % (K.C_BOUND, K.report()))


def _subprocess(select, **env):
    """The selected tests of this file in a fresh process (a fault in the emulation's alignment check fails one test, not the run)."""
    cmd = [sys.executable, "-m", "pytest", "-q", "-x", "-p", "no:cacheprovider", __file__, "-k", select]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=1200, env=dict(os.environ, **env, **{_SUB: "1"}), cwd=str(ROOT))
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-2000:]
    assert " passed" in out.stdout and "failed" not in out.stdout


# ---- hand-built programs
@pytest.mark.parametrize("n_in", [0, 1, 7, 15, 28, 29, 56, 57, 113])
@pytest.mark.parametrize("npoints", [258, 257])
def test_inputs(n_in, npoints):
    K.check_inputs_count(B, n_in, npoints)


def test_too_many_inputs():
    K.check_too_many_inputs(B)


@pytest.mark.parametrize("n_in", [57, 113])
def test_input_limit_does_not_depend_on_parity(n_in):
    K.check_odd_even_limit(B, n_in)


@pytest.mark.parametrize("npoints", [1, 2, 3, 255, 256, 257])
def test_small_shapes(npoints):
    K.check_small_shapes(B, npoints)


def test_nonfinite_inputs():
    K.check_nonfinite(B)


def test_v3_and_pointwise_bitwise_equal():
    K.check_bitwise_v3_vs_pointwise(B)


def test_return_codes():
    K.check_return_codes(B)


# ---- grid-stride loops
@pytest.mark.parametrize("tiles", [1, 2, 3])
def test_grid_stride_v3_and_pairs(tiles):
    K.check_grid_stride_v3(B, tiles)


@pytest.mark.parametrize("tiles", [1, 2])
def test_grid_stride_pointwise(tiles):
    K.check_grid_stride_pointwise(B, tiles)


@pytest.mark.parametrize("env", [dict(DB_EMU_CP="early"), dict(DB_EMU_ORDER="reverse")])
def test_grid_stride_under_other_schedules(env):
    """The double-buffered kernels with their cp.async copies landing at issue (a tile staged into the buffer still being read would
    show) and with threads and blocks in descending order."""
    if os.environ.get(_SUB):
        pytest.skip("runs in its own subprocess")
    _subprocess("grid_stride_v3 or small_shapes", **env)


# ---- programs of real plans
@pytest.mark.parametrize("case", ["rb3d_16", "shear"])
def test_rhs_plan_programs(case):
    import rhs_fused_cases as cases
    K.check_plan(B, cases.CASES[case]().rhs_plan, expect_pairs=True)


def test_complex_plan_program():
    import dedalus_b200 as d3
    from dedalus_b200 import examples
    pb = examples.complex_ginzburg_landau(16, 12)
    solver = pb['problem'].build_solver(d3.RK222)
    solver._init_device()
    prog, _ = K.check_plan(B, solver.rhs_plan)
    assert prog.fmax == 3                              # the cubic term on real / imaginary planes


def test_shell_plan_program():
    import dedalus_b200 as d3
    from dedalus_b200 import examples
    sc = examples.shell_convection(16, 8, 6)
    solver = sc['problem'].build_solver(d3.SBDF2)
    solver._init_device()
    K.check_plan(B, solver.rhs_plan)


def test_sphere_plan_program():
    import dedalus_b200 as d3
    from dedalus_b200 import examples
    sw = examples.shallow_water(16, 8)
    solver = sw['problem'].build_solver(d3.RK222)
    solver._init_device()
    K.check_plan(B, solver.rhs_plan)


def test_many_tracers():
    K.check_many_tracers(B)


# ---- transposes
@pytest.mark.parametrize("mode,B_,nA,nB,n3,P", K.tr_small_cases())
def test_transpose_layout(mode, B_, nA, nB, n3, P):
    K.check_transpose(B, mode, B_, nA, nB, n3, P)


@pytest.mark.parametrize("mode", [0, 1, 2, 3])
def test_transpose_long_chunks(mode):
    """clen > 4096 (several CTAs per chunk) with odd and even clen."""
    for n3 in (2 * 2500 + 1, 2 * 2500 + 2):
        nA, nB = (2, 2) if mode in (0, 3) else (2, 1)
        K.check_transpose(B, mode, 1, nA, nB, n3, 2 if mode in (0, 3) else 2)


def test_transpose_return_codes():
    K.check_transpose_return_codes(B)


def test_transpose_misaligned():
    """Run in a subprocess: a 16-byte access at an 8-byte aligned address aborts the emulation."""
    if os.environ.get(_SUB):
        K.check_transpose_misaligned(B)
    else:
        _subprocess("transpose_misaligned")


@pytest.mark.parametrize("P,B_,n1loc,n2,n3,complex_", [(2, 3, 2, 6, 5, False), (3, 1, 1, 9, 2, False), (8, 2, 2, 16, 3, False),
                                                       (2, 2, 3, 4, 3, True), (3, 1, 2, 6, 1, True)])
def test_transpose_round_trip(P, B_, n1loc, n2, n3, complex_):
    K.check_transpose_round_trip(B, P, B_, n1loc, n2, n3, complex_)

