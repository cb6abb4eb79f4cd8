"""Generate tests/golden/shell_bcs.npz by running the UNMODIFIED reference (single process, under tests/golden/ref_shim.py) on the
problems of tests/shell_bc_cases.py: radial / angular components and boundary data on spherical shells (reference
core/operators.py:2190-2310, core/basis.py:5892-5970).  Writes reference outputs only.

Run in a container that holds the reference checkout, never on the GPU machine:   python tests/golden/make_golden_shell_bcs.py
"""
import sys, pathlib
import numpy as np
HERE = pathlib.Path(__file__).resolve().parent
sys.path.insert(0, str(HERE)); sys.path.insert(0, str(HERE.parent))
import ref_shim
d3 = ref_shim.activate()
import shell_bc_cases as SBC


def natural_matrices(sp):
    """Reference pencil matrices expanded back to natural (field-major, un-permuted) ordering."""
    return {name: (sp.pre_left.T @ getattr(sp, name + "_min") @ sp.pre_right.T).toarray() for name in ("M", "L")}


def _run(sc, scheme, steps, tstep, start, change=None, rows=None):
    """K steps; rows: store only the first `rows` rows of the azimuthal coefficient axis (the large case: the rows of the first
    azimuthal pairs are enough to pin the state and keep the fixture small; its start is recomputed by the test)."""
    solver = sc['problem'].build_solver(getattr(d3, scheme))
    out = {}
    if start == "noise":
        SBC.noise_start(sc)
    elif start == "strong":
        g = np.load(HERE / "shell_tasks.npz")
        sc['b']['c'] = g['b_c']; sc['u']['c'] = g['u_c'] * 100
    elif start == "flow":
        SBC.noise_start(sc); SBC.flow_start(sc)
    if rows is None:
        out.update(b0=sc['b']['c'].copy(), u0=sc['u']['c'].copy())
    for i in range(steps):
        if change is not None and i == change:
            SBC.set_wall_data(sc['uw'], sc['bt'], sc['shell'], U0=-0.3, A=0.25)
        solver.step(tstep)
    fields = [(name, sc[name]) for name in ('p', 'b', 'u')] + list(sc['taus'].items())
    for name, f in fields:
        c = f['c'].copy()
        out[name + "1"] = c if rows is None or c.shape[-3] == 1 else np.ascontiguousarray(c[..., :rows, :, :])
    out['meta'] = np.array([steps, tstep])
    if rows is not None:
        out['rows'] = np.array(rows)
    return solver, out


def gen_shell_bcs():
    """Stress-free shell convection (pencil matrices of l = 0..3, states from noise and from strong flows), a driven inner wall
    with field data on both walls (RK222, and a run whose wall data changes between steps), a vector Poisson LBVP with radial and
    angular data, and the output tasks radial(u(r=Ro)) / angular(radial(strain_rate(r=Ri), 0), 0)."""
    out = {}
    sc = SBC.convection(d3, (16, 8, 6))
    solver, res = _run(sc, "SBDF2", 3, 0.05, "noise")
    out.update({f"sf_a_sbdf2_{k}": v for k, v in res.items()})
    for sp in solver.subproblems:
        ell = sp.group[1]
        if ell in (0, 1, 2, 3):
            for name, mat in natural_matrices(sp).items():
                out[f"sf_l{ell}_{name}"] = mat
    for tag, shape, scheme, steps, tstep, start, rows in (("sf_a_rk222", (16, 8, 6), "RK222", 3, 0.05, "noise", None),
                                                           ("sf_b_sbdf2", (32, 16, 12), "SBDF2", 3, 0.05, "noise", None),
                                                           ("sf_strong", (16, 8, 6), "SBDF2", 3, 0.02, "strong", None),
                                                           ("sf_big", (64, 32, 24), "SBDF2", 2, 0.02, "flow", SBC.BIG_ROWS)):
        _, res = _run(SBC.convection(d3, shape), scheme, steps, tstep, start, rows=rows)
        out.update({f"{tag}_{k}": v for k, v in res.items()})
    for tag, change in (("drv", None), ("drv_change", 2)):
        _, res = _run(SBC.convection(d3, (16, 8, 6), walls="driven", Ri=0.5, Ro=1.5), "RK222", 4, 0.02, "noise", change)
        out.update({f"{tag}_{k}": v for k, v in res.items()})
    lb = SBC.vector_poisson(d3)
    lb['problem'].build_solver().solve()
    out["lbvp_u"] = lb['u']['c'].copy()
    for name, f in lb['taus'].items():
        out[f"lbvp_{name}"] = f['c'].copy()
    # output tasks, evaluated the way a file handler evaluates them (scheduled, every task walked to the grid)
    t = SBC.task_inputs(d3)
    u = t['u']
    out["task_u_c"] = u['c'].copy()
    problem = d3.IVP([u], namespace=locals())
    problem.add_equation("dt(u) = 0")
    solver = problem.build_solver(d3.SBDF1)
    handler = solver.evaluator.add_dictionary_handler(iter=1)
    for name, op in t['tasks'].items():
        handler.add_task(op, layout='g', name=name, scales=3/2)
    solver.evaluator.evaluate_handlers([handler], iteration=0, wall_time=0, sim_time=0, timestep=1)
    for name in t['tasks']:
        out[f"task_{name}_g"] = handler.fields[name]['g'].copy()
    np.savez_compressed(HERE / "shell_bcs.npz", **out)
    print({k: (v.shape, float(np.abs(v).max())) for k, v in out.items()})


if __name__ == "__main__":
    gen_shell_bcs()
