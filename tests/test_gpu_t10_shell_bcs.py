"""Radial / angular components and boundary data on spherical shells on the GPU: stress-free shell convection up to 64 x 32 x 24,
a driven inner wall with field data, a vector Poisson LBVP with component data and output tasks against the unmodified reference
(tests/golden/shell_bcs.npz), and the reference's component tests against analytic answers."""
import pytest
import shell_bc_cases as C

pytestmark = pytest.mark.gpu


def test_stress_free_pencil_matrices(golden):
    C.check_pencil_matrices(golden("shell_bcs.npz"))


@pytest.mark.parametrize("tag,scheme,shape", [("sf_a_sbdf2", "SBDF2", (16, 8, 6)), ("sf_a_rk222", "RK222", (16, 8, 6)),
                                              ("sf_b_sbdf2", "SBDF2", (32, 16, 12)), ("sf_strong", "SBDF2", (16, 8, 6)),
                                              ("sf_big", "SBDF2", (64, 32, 24))])
def test_stress_free_convection_matches_reference(golden, tag, scheme, shape):
    solver = C.check_stress_free(golden("shell_bcs.npz"), tag, scheme, shape)
    assert solver.bset.last_verify < 1e-12


@pytest.mark.parametrize("tag", ["drv", "drv_change"])
def test_driven_wall_with_data_matches_reference(golden, tag):
    solver = C.check_driven(golden("shell_bcs.npz"), tag)
    assert solver.bset.last_verify < 1e-12


def test_vector_poisson_with_component_data_matches_reference(golden):
    solver = C.check_lbvp(golden("shell_bcs.npz"))
    assert solver.bset.last_verify < 1e-12


def test_component_output_tasks_match_reference(golden):
    C.check_tasks(golden("shell_bcs.npz"))


@pytest.mark.parametrize("k", [0, 1])
@pytest.mark.parametrize("dealias", [1, 3/2])
@pytest.mark.parametrize("radius", [0.5, 1.0, 1.5])
@pytest.mark.parametrize("which", ["radial_component_vector", "radial_component_tensor", "angular_component_vector",
                                   "angular_component_tensor"])
def test_reference_component_cases(which, k, dealias, radius):
    getattr(C, "check_" + which)(k, dealias, radius)
