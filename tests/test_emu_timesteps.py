"""The IMEX step loops of solvers.py through the CPU emulation of the kernels, replayed in long double (bodies: timestep_cases.py); GPU
version: tests/test_gpu_1g_timesteps.py.  Every scheme's coefficients against exact rational arithmetic; every scheme's device step on a
2-D Rayleigh-Benard problem (16 x 16, O(1) velocity); CNAB2, SBDF4 and RKSMR on the complex Ginzburg-Landau problem; SBDF3, CNLF2,
MCNAB2, RKSMR and RK443 on shallow water (16 x 8); SBDF4, CNAB2 and RKSMR on shell convection (16 x 8 x 6); a multistep history
across a forced re-order of the Cartesian pivot order, a host edit of the state between steps and Hermitian-symmetry enforcement
inside the history."""
import pytest
from emu import emu_lib as E
import timestep_cases as T

WORST = {}


@pytest.fixture(scope="module", autouse=True)
def emulation():
    E.install()
    yield
    E.uninstall()
    print("\nworst backward error per system set:", {k: f"{v:.2e}" for k, v in sorted(WORST.items())})


@pytest.mark.parametrize("scheme", T.MULTISTEP)
def test_multistep_coefficients_exact(scheme):
    T.check_multistep_coefficients(scheme, seed=len(scheme))


@pytest.mark.parametrize("scheme", T.RUNGE_KUTTA)
def test_rk_tableau_exact(scheme):
    nlu = T.check_rk_tableau(scheme)
    assert nlu == (3 if scheme == "RKSMR" else 1)


@pytest.mark.parametrize("scheme", T.ALL_SCHEMES)
def test_cartesian_real_step(scheme):
    out = T.check_scheme(T.rayleigh_benard, scheme, WORST)
    assert out['kind'] == "cartesian"
    if scheme in ("SBDF4", "RK443"):
        assert out['max_terms'] == 8
    if scheme == "RKSMR":
        assert out['lu_slots'] == 3


@pytest.mark.parametrize("scheme", ["CNAB2", "SBDF4", "RKSMR"])
def test_cartesian_complex_step(scheme):
    out = T.check_scheme(T.ginzburg_landau, scheme, WORST)
    assert out['kind'] == "cartesian"


@pytest.mark.parametrize("scheme", ["SBDF3", "CNLF2", "MCNAB2", "RKSMR", "RK443"])
def test_sphere_step(scheme):
    out = T.check_scheme(T.shallow_water, scheme, WORST)
    assert out['kind'] == "sphere"


@pytest.mark.parametrize("scheme", ["SBDF4", "CNAB2", "RKSMR"])
def test_shell_step(scheme):
    out = T.check_scheme(T.shell_convection, scheme, WORST)
    assert out['kind'] == "shell"


def test_history_survives_reorder():
    out = T.check_reorder_keeps_history(T.rayleigh_benard, WORST)
    assert out['reorders'] == 1


def test_host_edit_between_steps():
    T.check_host_edit(T.rayleigh_benard)


def test_hermitian_enforcement_inside_history():
    T.check_hermitian_cadence(T.rayleigh_benard)
