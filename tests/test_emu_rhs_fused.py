"""The fused x pass of the right-hand side (csrc/rfft_regs.cu k_rfft_x_products: backward x transforms, quadratic products and
forward x transforms in one kernel) against the separate passes it replaces, under the kernel emulation.  Both paths are evaluated
on the same plan (RHSPlan.use_x_products) into the equation arena, on states with O(1) velocities."""
import os, pathlib, subprocess, sys
import numpy as np, pytest
import dedalus_b200 as d3
from dedalus_b200 import examples
from emu import emu_lib as E
import rhs_fused_cases as cases

ROOT = pathlib.Path(__file__).resolve().parents[1]


@pytest.fixture(autouse=True)
def emulation():
    E.install()
    yield
    E.uninstall()


@pytest.mark.parametrize("case", ["rb3d_16", "rb3d_x384", "rb2d_nz32", "shear"])
def test_fused_matches_separate_passes(case):
    plan, fused, separate = cases.compare(cases.CASES[case]())
    assert plan.use_x_products
    scale = np.abs(separate).max()
    assert scale > 0
    # the shared register DFT stages and the k_pointwise_pairs term arithmetic make the two paths bitwise equal
    assert np.array_equal(fused, separate), np.abs(fused - separate).max() / scale


def test_one_launch_replaces_the_x_passes_and_the_products():
    from dedalus_b200.lib import get_lib
    solver = cases.CASES["rb3d_16"]()
    plan = solver.rhs_plan
    assert (plan.n_in, plan.n_out) == (15, 4)
    lib = get_lib()
    names = []
    raw = lib.call

    def record(name, *args):
        names.append(name)
        return raw(name, *args)

    lib.call = record
    try:
        counts = {}
        for use in (True, False):
            plan.use_x_products = use
            names.clear()
            plan.evaluate(solver.eq_t)
            counts[use] = dict((n, names.count(n)) for n in set(names))
    finally:
        del lib.call
    fused, sep = counts[True], counts[False]
    assert fused.get("db_rfft_x_products") == 1 and "db_rfft_x_products" not in sep
    assert sep.get("db_pointwise_pairs") == 1 and "db_pointwise_pairs" not in fused
    # the 15 backward x transforms, the product kernel and the forward x transform of the 4 stacked outputs are gone; every
    # other launch is the same
    assert sep["db_rfft_backward"] - fused["db_rfft_backward"] == 15
    assert sep["db_rfft_forward"] - fused["db_rfft_forward"] == 1
    assert sum(sep.values()) - sum(fused.values()) == 15 + 1 + 1 - 1


def test_separate_passes_stay_where_the_fused_kernel_does_not_apply():
    # a cubic term
    pb = examples.rayleigh_benard(dim=3, Nh=16, Nz=16, Rayleigh=1e6)
    u, b = pb['u'], pb['b']
    problem = pb['problem']
    eq = problem.equations[1]
    eq['RHS'] = eq['RHS'] - b * b * b
    solver = problem.build_solver(d3.RK222)
    solver._init_device()
    assert solver.rhs_plan.xprod is None and not solver.rhs_plan.use_x_products
    # grid_only evaluations (the grid-function stages) take the separate passes on a plan that is otherwise fused
    solver = cases.CASES["rb3d_16"]()
    plan = solver.rhs_plan
    assert plan.use_x_products
    grid = plan.evaluate(None, grid_only=True)
    assert tuple(grid.shape) == (plan.n_out,) + tuple(plan.gshape)


@pytest.mark.parametrize("env", [dict(DB_EMU_CP="early"), dict(DB_EMU_ORDER="reverse")])
def test_fused_kernel_under_the_other_emulation_models(env):
    """cp.async copies landing at issue (a staging buffer refilled while still read) and threads scheduled in reverse order (a
    missing barrier)."""
    cmd = [sys.executable, "-m", "pytest", "-q", "-x", "-p", "no:cacheprovider", str(ROOT / "tests" / "test_emu_rhs_fused.py"),
           "-k", "fused_matches or one_launch"]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=1800, env=dict(os.environ, **env), cwd=str(ROOT))
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-2000:]
    assert " passed" in out.stdout and "failed" not in out.stdout
