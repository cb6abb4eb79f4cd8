"""The kernels of the sphere and shell paths -- dense batches (csrc/dense.cu), the matrix transform on the FP64 tensor cores and on the
FMA pipe, ragged colatitude products, pair combinations, index moves, max reductions -- through the CPU emulation of the kernels, against
long-double references at their edge shapes; GPU version: tests/test_gpu_1d_curvilinear_kernels.py.  The emulation builds the 8 x 8 x 4
tensor-core product from warp shuffles and queues the zero-filling 16-byte cp.async copies like every other cp.async, so k_mmt_dmma
runs here as it does on the GPU, under both landing models of the copies and both thread orders."""
import os, subprocess, sys, pathlib
import pytest
from emu import emu_lib as E
import curvilinear_kernel_cases as K
from kernel_backends import EmuArrays

ROOT = pathlib.Path(__file__).resolve().parents[1]


@pytest.fixture(autouse=True)
def emulation():
    E.install()
    yield
    E.uninstall()


B = EmuArrays()


# ---- csrc/dense.cu
def test_dense_factor_small_sizes():
    """n = 1 .. 9, 31 .. 33, and 38, 39 (the size of the systems of the 16 x 8 x 6 shell-convection problem, and one past it)."""
    K.check_dense_factor_sizes(B, tuple(range(1, 10)) + (31, 32, 33, 38, 39))


def test_dense_factor_around_cta_width():
    """n = 255, 256, 257, 300: the strided pivot search starts to give a thread more than one row."""
    K.check_dense_factor_sizes(B, (255, 256, 257, 300))


def test_dense_factor_and_solve_config5_size():
    """n = 649, the systems of the 192 x 96 x 128 shell problem: one system, factor and both solves."""
    K.check_dense_solve(B, 649, [33], nvec=2, seed=649)


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


@pytest.mark.parametrize("env", [dict(DB_EMU_ORDER="reverse"), dict(DB_EMU_CP="early")])
def test_mmt_under_other_schedules(env):
    """k_mmt_dmma with threads and blocks in descending order, and with its cp.async copies landing at issue (a stage refilled while it
    is still being read would show)."""
    cmd = [sys.executable, "-m", "pytest", "-q", "-x", "-p", "no:cacheprovider", __file__, "-k", "mmt and not other_schedules"]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=1200, env=dict(os.environ, **env), cwd=str(ROOT))
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-2000:]
    assert " passed" in out.stdout and "failed" not in out.stdout


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
