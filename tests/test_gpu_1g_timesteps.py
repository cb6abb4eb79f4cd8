"""The IMEX step loops of solvers.py on the GPU, replayed in long double (bodies: timestep_cases.py): the cases of
tests/test_emu_timesteps.py, and sizes where the device takes the production paths the emulation is too slow for -- SBDF4, RKSMR and
RK443 on tall 3-D Rayleigh-Benard pencils (4 x 4 x 256), RKSMR and SBDF3 on shallow water at 128 x 64, SBDF2 and RKSMR on shell
convection at 32 x 16 x 24.  The worst backward error per system set is printed at the end."""
import pytest
import timestep_cases as T

pytestmark = pytest.mark.gpu
WORST = {}


@pytest.fixture(scope="module", autouse=True)
def backward_error_report():
    yield
    print("\nworst backward error per system set:", {k: f"{v:.2e}" for k, v in sorted(WORST.items())})


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
    assert T.check_scheme(T.ginzburg_landau, scheme, WORST)['kind'] == "cartesian"


@pytest.mark.parametrize("scheme", ["SBDF3", "CNLF2", "MCNAB2", "RKSMR", "RK443"])
def test_sphere_step(scheme):
    assert T.check_scheme(T.shallow_water, scheme, WORST)['kind'] == "sphere"


@pytest.mark.parametrize("scheme", ["SBDF4", "CNAB2", "RKSMR"])
def test_shell_step(scheme):
    assert T.check_scheme(T.shell_convection, scheme, WORST)['kind'] == "shell"


def test_history_survives_reorder():
    assert T.check_reorder_keeps_history(T.rayleigh_benard, WORST)['reorders'] == 1


def test_host_edit_between_steps():
    T.check_host_edit(T.rayleigh_benard)


def test_hermitian_enforcement_inside_history():
    T.check_hermitian_cadence(T.rayleigh_benard)


def _tall():
    return T.rayleigh_benard(dim=3, Nh=4, Nz=256)


@pytest.mark.parametrize("scheme", ["SBDF4", "RKSMR", "RK443"])
def test_tall_pencils_step(scheme):
    out = T.check_scheme(_tall, scheme, WORST)
    assert out['kind'] == "cartesian"
    assert out['max_terms'] == (8 if scheme != "RKSMR" else 6) and out['lu_slots'] == (3 if scheme == "RKSMR" else 1)


@pytest.mark.parametrize("scheme", ["RKSMR", "SBDF3"])
def test_sphere_128x64_step(scheme):
    assert T.check_scheme(lambda: T.shallow_water(128, 64), scheme, WORST)['kind'] == "sphere"


@pytest.mark.parametrize("scheme", ["SBDF2", "RKSMR"])
def test_shell_32x16x24_step(scheme):
    assert T.check_scheme(lambda: T.shell_convection(32, 16, 24), scheme, WORST)['kind'] == "shell"
