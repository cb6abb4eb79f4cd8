"""Whole-solver orchestration (dedalus_b200/solvers.py, evaluator.py, transforms.py) executed on the CPU through
the test-only kernel emulation, against reference states.  The GPU versions of these tests are in
test_gpu_solver.py; this file exists so the launch sequences can be checked on the GPU-less build container."""
import numpy as np, pytest
import dedalus_b200 as d3
from dedalus_b200 import examples
from emu import emu_lib as E

TOL = dict(rtol=1e-8, atol=1e-12)


@pytest.fixture(autouse=True)
def emulation():
    E.install()
    yield
    E.uninstall()


@pytest.mark.parametrize("dense", [None, "4"])
def test_rb3d_steps(golden, dense, monkeypatch):
    """dense="4": forward rows with >= 4 entries count as dense, so the segmented dense-run visits (partial sums kept in
    x, re-entered rows, same-chunk re-reads) of the fused solve kernel are exercised at this tiny size."""
    if dense:
        monkeypatch.setenv("DB_SOLVE_DENSE", dense)
    g = golden("rb3d_8.npz")
    pb = examples.rayleigh_benard(dim=3, Nh=8, Nz=8, Rayleigh=1e6)
    solver = pb['problem'].build_solver(d3.RK222)
    examples.rayleigh_benard_initial_condition(pb['b'], pb['bases'], pb['Lz'])
    assert np.allclose(pb['b']['c'], g['b0_c'], rtol=1e-12, atol=1e-14)
    for i in range(2):
        solver.step(0.01)
        if i == 0:
            for name in ('p', 'b', 'u'):
                assert np.allclose(pb[name]['c'], g[f"{name}_c_step1"], **TOL), name


@pytest.mark.parametrize("prefix", ["kdv_", "kdv443_"])
def test_kdv(golden, prefix):
    g = golden("kdv.npz")
    pk = examples.kdv_burgers(N=int(g[prefix + "N"]))
    examples.kdv_initial_condition(pk['u'], pk['xbasis'], pk['Lx'])
    solver = pk['problem'].build_solver(getattr(d3, str(g[prefix + "scheme"])))
    for i in range(int(g[prefix + "steps"])):
        solver.step(float(g[prefix + "dt"]))
    assert np.allclose(pk['u']['c'], g[prefix + "u_c"], **TOL)
    assert np.allclose(pk['u']['g'], g[prefix + "u_g"], **TOL)


def test_cfl_controller_matches_reference(golden):
    """dt sequence of the CFL controller and the resulting state vs the reference (extras/flow_tools.py:139-233)."""
    g = golden("rb2d_cfl.npz")
    pb = examples.rayleigh_benard(dim=2, Nh=32, Nz=16, Rayleigh=2e6)
    solver = pb['problem'].build_solver(d3.RK222)
    pb['b']['c'] = g['b0_c']; pb['u']['c'] = g['u0_c']
    cfl = d3.CFL(solver, initial_dt=0.01, cadence=2, safety=0.5, threshold=0.05, max_change=1.5, min_change=0.5, max_dt=0.05)
    cfl.add_velocity(pb['u'])
    dts = []
    for i in range(len(g['dts'])):
        dt = cfl.compute_timestep(); dts.append(dt)
        solver.step(dt)
    assert np.allclose(dts, g['dts'], rtol=1e-9, atol=0), (dts, g['dts'])
    assert np.allclose(pb['b']['c'], g['b_c'], **TOL)
    assert np.allclose(pb['u']['c'], g['u_c'], **TOL)


@pytest.mark.parametrize("timestepper", list(d3.schemes.keys()) + ["RKGFY"])
def test_heat_periodic_every_timestepper(timestepper):
    """Reference integration test tests/test_ivp.py:18-49 (1-D heat equation, every scheme in `schemes`, 20 steps,
    analytic solution), here on the real Fourier basis: dt(u) - dx(dx(u)) = F, F = sin(x).  A consistency check only (1 x 1 and 2 x 2
    systems, a solution of 2e-4, default allclose tolerances): the device step of every scheme is checked against a long-double
    replay in test_emu_timesteps.py / test_gpu_1g_timesteps.py."""
    from dedalus_b200 import timesteppers as ts
    scheme = ts.schemes.get(timestepper, getattr(ts, timestepper))
    c = d3.Coordinate('x')
    d = d3.Distributor(c, dtype=np.float64)
    b = d3.RealFourier(c, size=8, bounds=(0, 2 * np.pi), dealias=1)
    x = d.local_grid(b, scale=1)
    u = d.Field(bases=b); F = d.Field(bases=b)
    F['g'] = np.sin(x)
    dx = lambda A: d3.Differentiate(A, c)
    problem = d3.IVP([u], namespace=locals())
    problem.add_equation("dt(u) - dx(dx(u)) = F")
    solver = problem.build_solver(scheme)
    for i in range(20):
        solver.step(1e-5)
    amp = 1 - np.exp(-solver.sim_time)
    u.change_scales(1)
    assert np.allclose(u['g'], amp * np.sin(x))


def test_rb3d_16_register_kernels_match_oracle():
    """16^3 (24-point dealiased lines): the x passes and the z passes run through csrc/rfft_regs.cu inside the solver; two
    RK222 steps against the oracle (oracle/rb_oracle.py, itself pinned to the reference fixtures in test_oracle.py)."""
    from oracle import rb_oracle
    from dedalus_b200.lib import get_lib
    Nh, Nz, steps, dt = 16, 16, 2, 0.01
    pb = examples.rayleigh_benard(dim=3, Nh=Nh, Nz=Nz, Rayleigh=1e6)
    solver = pb['problem'].build_solver(d3.RK222)
    examples.rayleigh_benard_initial_condition(pb['b'], pb['bases'], pb['Lz'])
    b0 = pb['b']['c'].copy()
    served = get_lib().rfft_regs_launches()
    for _ in range(steps):
        solver.step(dt)
    assert get_lib().rfft_regs_launches() > served
    ref = rb_oracle.run(dim=3, Nh=Nh, Nz=Nz, Ra=1e6, b0_c=b0, steps=steps, dt=dt, scheme="RK222")
    for name in ("p", "b", "u"):
        assert np.allclose(pb[name]['c'], ref[name], rtol=1e-8, atol=1e-12), name


@pytest.mark.parametrize("Nz,steps", [(192, 2), (256, 2)])
def test_tall_pencils_match_oracle(Nz, steps):
    """Round-1 regression (VERDICT / ADVICE): Nz = 256 pencils -- the benchmark's -- were solved wrongly in the n = Nz + 2
    Helmholtz batches.  4 x 4 x Nz, O(1) velocity, RK222 at the benchmark's dt, against the oracle."""
    from tall_pencils import run_and_compare
    solver, worst = run_and_compare(4, Nz, [0.0025] * steps)
    assert solver.bset.reorders == 0 and solver.bset.last_verify < 1e-12


def test_timestep_changes_are_reverified():
    """The pivot order is computed at the first LHS and every later factorisation (dt change) is verified on all systems
    (ADVICE round 1: the frozen order silently lost accuracy at larger dt): dt from 2.5e-3 up to 1 and back down."""
    from tall_pencils import run_and_compare
    solver, worst = run_and_compare(4, 64, [0.0025, 0.02, 0.1, 1.0, 1e-4])
    assert solver.bset.last_verify < 1e-10


def test_unstable_pivot_order_is_detected_and_repaired(monkeypatch):
    """Safety net: with round 1's pivot threshold (0.1) the Helmholtz batches are unstable at Nz = 192; the device-side
    verification must flag them, the batches get a new order, and the states then match the oracle."""
    from tall_pencils import run_and_compare
    monkeypatch.setenv("DB_PIVOT_THRESHOLD", "0.1")
    solver, worst = run_and_compare(4, 192, [0.0025] * 2)
    assert solver.bset.reorders > 0 and solver.bset.last_verify < 1e-10


def test_solve_then_multiply_back_residual():
    """(M + b0 L) solve(b) == b through the fused solve and mat-vec kernels, every system of every batch."""
    from residual_check import solve_residual
    pb = examples.rayleigh_benard(dim=3, Nh=8, Nz=16, Rayleigh=1e6)
    solver = pb['problem'].build_solver(d3.RK222)
    examples.rayleigh_benard_initial_condition(pb['b'], pb['bases'], pb['Lz'])
    solver.step(0.01)
    assert solve_residual(solver, 0.01) < 1e-11


@pytest.mark.parametrize("dim,Nh,Nz,scheme,steps", [(2, 16, 16, "RK443", 2), (2, 16, 16, "RK111", 3), (3, 8, 8, "RK443", 2), (2, 16, 24, "SBDF2", 4)])
def test_rayleigh_benard_schemes_match_oracle(dim, Nh, Nz, scheme, steps):
    """More tableaux on the pencil path (several implicit stages sharing / not sharing a factorisation, multistep history
    rotation) against the oracle's own IMEX loops (oracle/imex.py restates core/timesteppers.py:205-495, 647-740)."""
    from oracle import rb_oracle
    dt = 0.004
    pb = examples.rayleigh_benard(dim=dim, Nh=Nh, Nz=Nz, Rayleigh=1e5)
    solver = pb['problem'].build_solver(getattr(d3, scheme))
    examples.rayleigh_benard_initial_condition(pb['b'], pb['bases'], pb['Lz'])
    b0 = pb['b']['c'].copy()
    for _ in range(steps):
        solver.step(dt)
    ref = rb_oracle.run(dim=dim, Nh=Nh, Nz=Nz, Ra=1e5, b0_c=b0, steps=steps, dt=dt, scheme=scheme)
    for name in ("p", "b", "u"):
        assert np.allclose(pb[name]['c'], ref[name], rtol=1e-8, atol=1e-12), name


def test_software_pipelined_solve_variant_matches_oracle():
    """DB_SOLVE_PIPE=1 (opt-in kernel k_batches_solve_pipe: gathers issued one chunk early) in a fresh process, because the
    switch is read once per process; 3-D RB 8x8x16, dense threshold lowered so segmented rows and late re-reads occur."""
    import subprocess, sys, os, pathlib
    root = pathlib.Path(__file__).resolve().parents[1]
    script = r"""
import sys
sys.path.insert(0, %r); sys.path.insert(0, %r)
from emu import emu_lib as E
E.install()
import numpy as np
import dedalus_b200 as d3
from dedalus_b200 import examples
from oracle import rb_oracle
pb = examples.rayleigh_benard(dim=3, Nh=8, Nz=16, Rayleigh=1e6)
solver = pb['problem'].build_solver(d3.RK222)
examples.rayleigh_benard_initial_condition(pb['b'], pb['bases'], pb['Lz'])
b0 = pb['b']['c'].copy()
for _ in range(2):
    solver.step(0.01)
ref = rb_oracle.run(dim=3, Nh=8, Nz=16, Ra=1e6, b0_c=b0, steps=2, dt=0.01, scheme="RK222")
ok = all(np.allclose(pb[n]['c'], ref[n], rtol=1e-8, atol=1e-12) for n in ("p", "b", "u"))
print("PIPE_OK" if ok else "PIPE_FAIL")
""" % (str(root), str(root / "tests"))
    for dense in ("64", "5"):
        out = subprocess.run([sys.executable, "-c", script], capture_output=True, text=True, timeout=600,
                             env=dict(os.environ, DB_SOLVE_PIPE="1", DB_SOLVE_DENSE=dense))
        assert "PIPE_OK" in out.stdout, out.stdout[-1000:] + out.stderr[-2000:]


def test_rb3d_16_matches_reference_fixture(golden):
    """16^3 against the UNMODIFIED reference's states (tests/golden/rb3d_16.npz): the smallest size at which the
    register-resident Fourier / Chebyshev kernels sit on the solver's path."""
    g = golden("rb3d_16.npz")
    pb = examples.rayleigh_benard(dim=3, Nh=16, Nz=16, Rayleigh=float(g['Ra']))
    solver = pb['problem'].build_solver(getattr(d3, str(g['scheme'])))
    examples.rayleigh_benard_initial_condition(pb['b'], pb['bases'], pb['Lz'])
    assert np.allclose(pb['b']['c'], g['b0_c'], rtol=1e-12, atol=1e-14)
    for i in range(int(g['steps'])):
        solver.step(float(g['dt']))
        if i == 0:
            for name in ('p', 'b', 'u'):
                assert np.allclose(pb[name]['c'], g[f"{name}_c_step1"], **TOL), name
    for name in ('p', 'b', 'u'):
        assert np.allclose(pb[name]['c'], g[f"{name}_c"], **TOL), name


def test_global_flow_property_reductions():
    """GlobalFlowProperty.max / min (reference extras/flow_tools.py:64-130: reductions of the grid data of a field) equal the
    same reductions of the field's grid values read back through the host mirror."""
    from dedalus_b200.extras import flow_tools
    pb = examples.rayleigh_benard(dim=2, Nh=16, Nz=16, Rayleigh=1e5)
    solver = pb['problem'].build_solver(d3.RK222)
    examples.rayleigh_benard_initial_condition(pb['b'], pb['bases'], pb['Lz'])
    for _ in range(2):
        solver.step(0.01)
    flow = flow_tools.GlobalFlowProperty(solver, cadence=1)
    flow.add_property(pb['b'], name='b')
    vmax, vmin = flow.max('b'), flow.min('b')
    bg = np.array(pb['b']['g'])
    assert np.isclose(vmax, bg.max(), rtol=1e-13, atol=0) and np.isclose(vmin, bg.min(), rtol=1e-13, atol=1e-15)


def test_file_handler_checkpoint_and_restart(tmp_path):
    """Analysis output / checkpoint from the device state and restart (reference core/evaluator.py:208-300, 366-865;
    core/solvers.py:632-673): snapshots fire on the iteration cadence, a run restarted from a checkpoint with load_state
    reproduces the uninterrupted run, and the scales / tasks bookkeeping matches the reference's layout."""
    def make():
        pb = examples.rayleigh_benard(dim=2, Nh=16, Nz=16, Rayleigh=1e5)
        solver = pb['problem'].build_solver(d3.RK222)
        examples.rayleigh_benard_initial_condition(pb['b'], pb['bases'], pb['Lz'])
        return pb, solver
    dt = 0.01
    pb, solver = make()
    snaps = solver.evaluator.add_file_handler(tmp_path / "snapshots", iter=2, max_writes=2)
    snaps.add_task(pb['b'], name='buoyancy', layout='g')
    chk = solver.evaluator.add_file_handler(tmp_path / "checkpoints", iter=3)
    chk.add_tasks(solver.state, layout='g')
    for _ in range(6):
        solver.step(dt)
    final = {n: np.array(pb[n]['c']) for n in ('p', 'b', 'u')}
    # snapshots at iterations 0, 2, 4 -> sets of 2 writes
    s1 = np.load(tmp_path / "snapshots" / "snapshots_s1.npz"); s2 = np.load(tmp_path / "snapshots" / "snapshots_s2.npz")
    assert list(s1['scales/iteration']) == [0, 2] and list(s2['scales/iteration']) == [4]
    assert list(s1['scales/write_number']) == [1, 2] and list(s2['scales/write_number']) == [3]
    assert s1['tasks/buoyancy'].shape == (2, 16, 16) and np.isclose(s1['scales/sim_time'][1], 2 * dt)
    # restart from the checkpoint written at iteration 3 and run to iteration 6
    pb2, solver2 = make()
    write, dt_loaded = solver2.load_state(tmp_path / "checkpoints" / "checkpoints_s1.npz", index=1)
    assert (write, solver2.iteration) == (2, 3) and np.isclose(solver2.sim_time, 3 * dt) and np.isclose(dt_loaded, dt)
    for _ in range(3):
        solver2.step(dt)
    for n in ('p', 'b', 'u'):
        assert np.allclose(pb2[n]['c'], final[n], rtol=1e-9, atol=1e-12), n
