"""The grid products and transposes of csrc/pointwise.cu -- db_pointwise (k_pointwise, k_pointwise_v3), db_pointwise_pairs and the four
db_transpose_* entries -- on the GPU against long-double references and the header's layouts; the same bodies run through the emulation
in tests/test_emu_pointwise_kernels.py.  Here also what the emulation leaves out: k_pointwise with 3 tiles per CTA, transposes with
chunks longer than 64 * 4096 doubles (the capped grid strides) and with about 10^5 chunks, and the misaligned cases at full size."""
import numpy as np, pytest
from kernel_backends import DeviceArrays
import pointwise_kernel_cases as K

pytestmark = pytest.mark.gpu
B = DeviceArrays()


@pytest.fixture(scope="module", autouse=True)
def ratio_report():
    yield
    print("\nlargest error / bound per kernel (C_BOUND = %g):\n%s" % (K.C_BOUND, K.report()))


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


@pytest.mark.parametrize("tiles", [1, 2, 3])
def test_grid_stride_v3_and_pairs(tiles):
    K.check_grid_stride_v3(B, tiles)
    K.check_grid_stride_v3(B, tiles, n_in=4)        # per_sm = 8


@pytest.mark.parametrize("tiles", [1, 2, 3])
def test_grid_stride_pointwise(tiles):
    K.check_grid_stride_pointwise(B, tiles)


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
    assert prog.fmax == 3


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


@pytest.mark.parametrize("mode,B_,nA,nB,n3,P", K.tr_small_cases())
def test_transpose_layout(mode, B_, nA, nB, n3, P):
    K.check_transpose(B, mode, B_, nA, nB, n3, P)


@pytest.mark.parametrize("mode", [0, 1, 2, 3])
def test_transpose_long_chunks(mode):
    """clen > 4096 (several CTAs per chunk) and > 64 * 4096 (gy capped at 64: the copy loop strides), odd and even."""
    for n3 in (5001, 5002, 64 * 4096 + 1001, 64 * 4096 + 1002):
        nA, nB = (2, 2) if mode in (0, 3) else (2, 1)
        K.check_transpose(B, mode, 1, nA, nB, n3, 2)


@pytest.mark.parametrize("mode", [0, 1, 2, 3])
def test_transpose_many_chunks(mode):
    """About 10^5 chunks of 2 doubles."""
    if mode in (0, 3):
        K.check_transpose(B, mode, 3, 4200, 16, 1, 8)          # 3 * 4200 * 8 chunks
    else:
        K.check_transpose(B, mode, 3, 33600, 1, 2, 8)          # 3 * 33600 chunks


def test_transpose_return_codes():
    K.check_transpose_return_codes(B)


def test_transpose_misaligned():
    K.check_transpose_misaligned(B)


@pytest.mark.parametrize("P,B_,n1loc,n2,n3,complex_", [(2, 3, 2, 6, 5, False), (3, 1, 1, 9, 2, False), (8, 2, 2, 16, 3, False),
                                                       (2, 2, 3, 4, 3, True), (3, 1, 2, 6, 1, True), (4, 2, 16, 64, 33, True)])
def test_transpose_round_trip(P, B_, n1loc, n2, n3, complex_):
    K.check_transpose_round_trip(B, P, B_, n1loc, n2, n3, complex_)
