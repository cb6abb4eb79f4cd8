"""The kernels of the sphere and shell paths -- dense batches (csrc/dense.cu), the matrix transform on the FP64 tensor cores and on the
FMA pipe, ragged colatitude products, pair combinations, index moves, max reductions -- on the GPU, against long-double references at
their edge shapes; the same bodies run through the emulation in tests/test_emu_curvilinear_kernels.py.  Here also the sizes the
emulation leaves out: dense systems of n = 801 and 1000, past the size at which the solve keeps its columns in global memory."""
import pytest
import curvilinear_kernel_cases as K
from kernel_backends import DeviceArrays

pytestmark = pytest.mark.gpu
B = DeviceArrays()


# ---- csrc/dense.cu
def test_dense_factor_small_sizes():
    """n = 1 .. 9, 31 .. 33, and 38, 39 (the size of the systems of the 16 x 8 x 6 shell-convection problem, and one past it)."""
    K.check_dense_factor_sizes(B, tuple(range(1, 10)) + (31, 32, 33, 38, 39))


def test_dense_factor_around_cta_width():
    """n = 255, 256, 257, 300: the strided pivot search starts to give a thread more than one row."""
    K.check_dense_factor_sizes(B, (255, 256, 257, 300))


def test_dense_factor_and_solve_config5_size():
    """n = 649, the systems of the 192 x 96 x 128 shell problem: factor and both solves."""
    K.check_dense_solve(B, 649, [33, 200], nvec=2, seed=649)


def test_dense_factor_large_sizes():
    K.check_dense_factor_sizes(B, (801, 1000))


def test_dense_solve_past_shared_memory_size():
    """n = 801 with DB_DENSE_SOLVE_SMEM unset: the launcher's own size rule keeps the columns in global memory."""
    assert 801 > K.DENSE_SMEM_MAX_N and 801 * 32 * 8 > 200 * 1024
    K.check_dense_solve(B, 801, [33, 65], nvec=2, seed=801, smem_modes=(None,))


def test_dense_factor_ties():
    K.check_dense_factor_ties(B)


def test_dense_factor_info():
    K.check_dense_info(B)


def test_dense_padded_systems():
    K.check_dense_padded(B)


def test_dense_solve_ragged_columns():
    K.check_dense_solve_ragged(B)


def test_dense_solve_nvec():
    K.check_dense_solve_nvec(B)


def test_dense_solve_remainders():
    K.check_dense_solve_remainders(B)


def test_dense_solve_long_cycle():
    K.check_dense_solve_long_cycle(B)


def test_singular_matrix_raises_in_matsolver():
    K.check_singular_matrix_raises()


@pytest.fixture
def shell_systems():
    return K.shell_systems()


def test_shell_systems_check_info_raises(shell_systems):
    K.check_shell_systems_info_raises(shell_systems)


def test_matvec_edges():
    K.check_matvec_edges(B)


def test_shell_operator_matvec(shell_systems):
    K.check_shell_operator_matvec(B, shell_systems)


def test_dense_combine():
    total = K.check_dense_combine(B, 9, 250)
    assert total > 16 * B.sms * 256                 # past the grid cap of k_dense_combine
    K.check_dense_combine(B, 1, 1)


# ---- db_mmt_apply
@pytest.mark.parametrize("m,n,outer,inner", K.mmt_tile_edge_shapes())
def test_mmt_tile_edges(m, n, outer, inner):
    K.check_mmt(B, m, n, outer, inner, "dmma")


def test_mmt_dispatch():
    K.check_mmt_dispatch(B)


@pytest.mark.parametrize("Nr,Nrg", [(6, 6), (6, 9), (12, 12), (12, 18), (96, 144), (256, 384)])
def test_mmt_jacobi_matrices(Nr, Nrg):
    K.check_mmt_jacobi_matrices(B, Nr, Nrg)


# ---- ragged products, pair combinations, index moves
def test_ragged_shapes():
    K.check_ragged_shapes(B)


def test_pair_lincomb_shapes():
    K.check_pair_lincomb_shapes(B)


def test_pair_lincomb_intertwiner_round_trip():
    K.check_intertwiner_round_trip(B)


def test_index_moves():
    K.check_index_moves(B)


# ---- reductions
def test_cfl_axis_mapping():
    K.check_cfl_axis_mapping(B)


def test_reduction_positions():
    K.check_reduction_positions(B)


def test_reductions_propagate_nan():
    K.check_reductions_propagate_nan(B)
