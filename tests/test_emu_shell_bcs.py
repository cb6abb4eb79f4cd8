"""Radial / angular components and boundary data on spherical shells through the CPU emulation of the kernels, against the
unmodified reference (tests/golden/shell_bcs.npz) and analytic answers; GPU version: tests/test_gpu_t10_shell_bcs.py."""
import pathlib, subprocess, sys, os, socket
import pytest
from emu import emu_lib as E
import shell_bc_cases as C

ROOT = pathlib.Path(__file__).resolve().parents[1]


@pytest.fixture(autouse=True)
def emulation():
    E.install()
    yield
    E.uninstall()


def test_stress_free_pencil_matrices(golden):
    C.check_pencil_matrices(golden("shell_bcs.npz"))


@pytest.mark.parametrize("tag,scheme,shape", [("sf_a_sbdf2", "SBDF2", (16, 8, 6)), ("sf_a_rk222", "RK222", (16, 8, 6)),
                                              ("sf_b_sbdf2", "SBDF2", (32, 16, 12)), ("sf_strong", "SBDF2", (16, 8, 6))])
def test_stress_free_convection_matches_reference(golden, tag, scheme, shape):
    solver = C.check_stress_free(golden("shell_bcs.npz"), tag, scheme, shape)
    assert solver.bset.last_verify < 1e-12


@pytest.mark.parametrize("tag", ["drv", "drv_change"])
def test_driven_wall_with_data_matches_reference(golden, tag):
    C.check_driven(golden("shell_bcs.npz"), tag)


def test_vector_poisson_with_component_data_matches_reference(golden):
    C.check_lbvp(golden("shell_bcs.npz"))


def test_component_output_tasks_match_reference(golden):
    C.check_tasks(golden("shell_bcs.npz"))


@pytest.mark.parametrize("k", [0, 1])
@pytest.mark.parametrize("dealias", [1, 3/2])
@pytest.mark.parametrize("radius", [0.5, 1.0, 1.5])
@pytest.mark.parametrize("which", ["radial_component_vector", "radial_component_tensor", "angular_component_vector",
                                   "angular_component_tensor"])
def test_reference_component_cases(which, k, dealias, radius):
    getattr(C, "check_" + which)(k, dealias, radius)


def test_component_index_beyond_rank_raises():
    C.check_component_index_errors()


def test_two_rank_stress_free_convection_matches_reference():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", str(port), str(ROOT / "tests" / "dist_worker_shell_bcs.py"), "sf_strong"]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=600, env=dict(os.environ, OMP_NUM_THREADS="1"))
    assert "DIST_OK" in out.stdout, out.stdout[-2000:] + out.stderr[-4000:]
