"""Radial and angular components and boundary data on spherical shells.  The problem builders take the package as an argument:
the fixture generator (tests/golden/make_golden_shell_bcs.py) runs them with the unmodified reference, the tests
(tests/test_emu_shell_bcs.py through the emulation, tests/test_gpu_t10_shell_bcs.py on the GPU) with dedalus_b200."""
import numpy as np

# the 64 x 32 x 24 case is compared on the rows of its first two azimuthal pairs (m = 0, 1 and their folded partners)
BIG_ROWS = 4


def _shell_setup(d3, shape, Ri, Ro, dealias=3/2):
    coords = d3.SphericalCoordinates('phi', 'theta', 'r')
    dist = d3.Distributor(coords, dtype=np.float64)
    shell = d3.ShellBasis(coords, shape=shape, radii=(Ri, Ro), dealias=dealias, dtype=np.float64)
    return coords, dist, shell


def convection(d3, shape, walls="stress_free", Ri=14, Ro=15, Rayleigh=3500, Prandtl=1):
    """The Boussinesq shell problem of examples/ivp_shell_convection/shell_convection.py with stress-free, impenetrable walls on
    both sides (the walls of examples/evp_shell_rotating_convection/rotating_convection.py:93-97), or -- walls="driven" -- a
    driven inner wall with given data: radial(u(r=Ri)) = 0, angular(u(r=Ri)) = uw, b(r=Ro) = bt, no-slip at Ro."""
    coords, dist, shell = _shell_setup(d3, shape, Ri, Ro)
    sphere = shell.outer_surface
    p = dist.Field(name='p', bases=shell); b = dist.Field(name='b', bases=shell)
    u = dist.VectorField(coords, name='u', bases=shell)
    tau_p = dist.Field(name='tau_p')
    tau_b1 = dist.Field(name='tau_b1', bases=sphere); tau_b2 = dist.Field(name='tau_b2', bases=sphere)
    tau_u1 = dist.VectorField(coords, name='tau_u1', bases=sphere); tau_u2 = dist.VectorField(coords, name='tau_u2', bases=sphere)
    kappa = (Rayleigh * Prandtl)**(-1/2); nu = (Rayleigh / Prandtl)**(-1/2)
    phi, theta, r = dist.local_grids(shell)
    er = dist.VectorField(coords, bases=shell.radial_basis); er['g'][2] = 1
    rvec = dist.VectorField(coords, bases=shell.radial_basis); rvec['g'][2] = r
    lift_basis = shell.derivative_basis(1)
    lift = lambda A: d3.Lift(A, lift_basis, -1)
    grad_u = d3.grad(u) + rvec*lift(tau_u1)
    grad_b = d3.grad(b) + rvec*lift(tau_b1)
    strain_rate = d3.grad(u) + d3.transpose(d3.grad(u))
    uw = dist.VectorField(coords.S2coordsys, name='uw', bases=shell.inner_surface)
    bt = dist.Field(name='bt', bases=shell.outer_surface)
    problem = d3.IVP([p, b, u, tau_p, tau_b1, tau_b2, tau_u1, tau_u2], namespace=locals())
    problem.add_equation("trace(grad_u) + tau_p = 0")
    problem.add_equation("dt(b) - kappa*div(grad_b) + lift(tau_b2) = - u@grad(b)")
    problem.add_equation("dt(u) - nu*div(grad_u) + grad(p) - b*er + lift(tau_u2) = - u@grad(u)")
    problem.add_equation("b(r=Ri) = 1")
    if walls == "stress_free":
        problem.add_equation("radial(u(r=Ri)) = 0")
        problem.add_equation("angular(radial(strain_rate(r=Ri), 0), 0) = 0")
        problem.add_equation("b(r=Ro) = 0")
        problem.add_equation("radial(u(r=Ro)) = 0")
        problem.add_equation("angular(radial(strain_rate(r=Ro), 0), 0) = 0")
    else:
        set_wall_data(uw, bt, shell)
        problem.add_equation("radial(u(r=Ri)) = 0")
        problem.add_equation("angular(u(r=Ri)) = uw")
        problem.add_equation("b(r=Ro) = bt")
        problem.add_equation("u(r=Ro) = 0")
    problem.add_equation("integ(p) = 0")
    return dict(problem=problem, dist=dist, shell=shell, p=p, b=b, u=u, uw=uw, bt=bt, Ri=Ri, Ro=Ro,
                taus=dict(tau_p=tau_p, tau_b1=tau_b1, tau_b2=tau_b2, tau_u1=tau_u1, tau_u2=tau_u2))


def set_wall_data(uw, bt, shell, U0=0.5, A=0.1):
    """uw: a zonal rotation of the inner wall (axisymmetric) plus the surface gradient of sin^2(theta) cos(2 phi) (m = 2);
    bt: a temperature varying with latitude plus an m = 2 part."""
    dist = uw.dist
    phi, theta = dist.local_grids(shell.inner_surface)[:2]
    uw.change_scales(1)
    uw['g'] = 0
    uw['g'][0] = U0 * np.sin(theta) - 2 * A * np.sin(theta) * np.sin(2 * phi)
    uw['g'][1] = 2 * A * np.sin(theta) * np.cos(theta) * np.cos(2 * phi)
    phi, theta = dist.local_grids(shell.outer_surface)[:2]
    bt.change_scales(1)
    bt['g'] = 0.1 * np.cos(theta) + 0.05 * np.sin(theta)**2 * np.cos(2 * phi)


def noise_start(sc, seed=42):
    """The stock script's buoyancy start: noise damped at the walls on top of the conductive profile."""
    Ri, Ro = sc['Ri'], sc['Ro']
    phi, theta, r = sc['dist'].local_grids(sc['shell'])
    b = sc['b']
    b.fill_random('g', seed=seed, distribution='normal', scale=1e-3)
    b['g'] *= (r - Ri) * (Ro - r)
    b['g'] += (Ri - Ri*Ro/r) / (Ri - Ro)


def flow_start(sc, seed=7, scale=0.5):
    """An O(scale) smooth velocity vanishing at the walls (the noise starts keep |u| ~ 1e-6 |b|)."""
    Ri, Ro = sc['Ri'], sc['Ro']
    phi, theta, r = sc['dist'].local_grids(sc['shell'])
    u = sc['u']
    u.fill_random('g', seed=seed, distribution='normal', scale=scale)
    u.low_pass_filter(scales=0.5)
    u['g'] *= (r - Ri) * (Ro - r)


def vector_poisson(d3, shape=(16, 8, 6), Ri=0.5, Ro=1.5):
    """Shell LBVP: div(grad(u)) = 0 with radial(u(r=Ri)) = ur, angular(u(r=Ri)) = uw and u(r=Ro) = 0."""
    coords, dist, shell = _shell_setup(d3, shape, Ri, Ro)
    sphere = shell.outer_surface
    u = dist.VectorField(coords, name='u', bases=shell)
    tau_u1 = dist.VectorField(coords, name='tau_u1', bases=sphere); tau_u2 = dist.VectorField(coords, name='tau_u2', bases=sphere)
    phi, theta, r = dist.local_grids(shell)
    rvec = dist.VectorField(coords, bases=shell.radial_basis); rvec['g'][2] = r
    lift_basis = shell.derivative_basis(1)
    lift = lambda A: d3.Lift(A, lift_basis, -1)
    grad_u = d3.grad(u) + rvec*lift(tau_u1)
    uw = dist.VectorField(coords.S2coordsys, name='uw', bases=shell.inner_surface)
    bt = dist.Field(name='bt', bases=shell.outer_surface)
    set_wall_data(uw, bt, shell)
    ur = dist.Field(name='ur', bases=shell.inner_surface)
    phi_i, theta_i = dist.local_grids(shell.inner_surface)[:2]
    ur['g'] = 0.3 + 0.2 * np.cos(theta_i) + 0.1 * np.sin(theta_i) * np.cos(phi_i)
    problem = d3.LBVP([u, tau_u1, tau_u2], namespace=locals())
    problem.add_equation("div(grad_u) + lift(tau_u2) = 0")
    problem.add_equation("radial(u(r=Ri)) = ur")
    problem.add_equation("angular(u(r=Ri)) = uw")
    problem.add_equation("u(r=Ro) = 0")
    return dict(problem=problem, dist=dist, shell=shell, u=u, ur=ur, uw=uw, taus=dict(tau_u1=tau_u1, tau_u2=tau_u2))


def task_inputs(d3, u_c=None, Ri=14, Ro=15):
    """The output tasks radial(u(r=Ro)) and the surface shear angular(radial(strain_rate(r=Ri), 0), 0) of a velocity that does
    not vanish on the walls (smooth noise; u_c: its stored coefficients)."""
    coords, dist, shell = _shell_setup(d3, (16, 8, 6), Ri, Ro)
    u = dist.VectorField(coords, name='u', bases=shell)
    if u_c is None:
        u.fill_random('g', seed=11, distribution='normal', scale=0.1)
        u.low_pass_filter(scales=0.5)
    else:
        u['c'] = u_c
    strain_rate = d3.grad(u) + d3.transpose(d3.grad(u))
    tasks = dict(ur_outer=d3.radial(u(r=Ro)), shear_inner=d3.angular(d3.radial(strain_rate(r=Ri), 0), 0),
                 uang_outer=d3.angular(u(r=Ro)))
    return dict(dist=dist, shell=shell, u=u, tasks=tasks)


# ------------------------------------------------------------------------------------------------------------------------------
# checks (dedalus_b200 against tests/golden/shell_bcs.npz)
# ------------------------------------------------------------------------------------------------------------------------------
def _close(got, ref, rtol, atol, what):
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    assert np.allclose(got, ref, rtol=rtol, atol=atol), (what, np.abs(got - ref).max(), np.abs(ref).max())


def _check_state(g, tag, sc):
    """p, b, u: rtol 1e-8 with atol 1e-10 max|field| + 1e-13 max|b| (rounding relative to the buoyancy the noise-started
    velocity is coupled to); the tau fields: atol 1e-4 max|tau| (tests/shell_cases.py check_shell_convection)."""
    rows = int(g[f"{tag}_rows"]) if f"{tag}_rows" in g else None
    part = lambda c: c if rows is None or c.shape[-3] == 1 else c[..., :rows, :, :]
    floor = 1e-13 * np.abs(g[f"{tag}_b1"]).max()
    for name in ('p', 'b', 'u'):
        ref = g[f"{tag}_{name}1"]
        _close(part(sc[name]['c']), ref, 1e-8, 1e-10 * np.abs(ref).max() + floor, (tag, name))
    for name, f in sc['taus'].items():
        ref = g[f"{tag}_{name}1"]
        _close(part(f['c']), ref, 1e-6, 1e-4 * np.abs(ref).max() + 1e-15, (tag, name))     # tau_p: 0 up to rounding


def _run(d3, g, tag, sc, scheme, start, change=None):
    steps, tstep = g[f"{tag}_meta"]
    solver = sc['problem'].build_solver(getattr(d3, scheme))
    if start == "noise":
        noise_start(sc)
    elif start == "flow":
        noise_start(sc); flow_start(sc)
    else:
        sc['b']['c'] = g[f"{tag}_b0"]; sc['u']['c'] = g[f"{tag}_u0"]
    if f"{tag}_b0" in g:
        assert np.allclose(sc['b']['c'], g[f"{tag}_b0"], rtol=1e-11, atol=1e-13)
    for i in range(int(steps)):
        if change is not None and i == change:
            set_wall_data(sc['uw'], sc['bt'], sc['shell'], U0=-0.3, A=0.25)
        solver.step(float(tstep))
    _check_state(g, tag, sc)
    return solver


def check_pencil_matrices(g):
    """M and L of the stress-free problem for l = 0..3 in natural ordering against the reference's subproblem matrices, and the
    count of valid rows / columns per degree (tau_u1's 3 components pair with radial (1) + angular (2); at l = 0 only spin 0)."""
    import dedalus_b200 as d3
    from dedalus_b200 import shell_ivp
    sc = convection(d3, (16, 8, 6))
    problem = sc['problem']
    low = shell_ivp.ShellLowering(problem)
    for ell in (0, 1, 2, 3):
        M, L, rows, cols = shell_ivp.assemble(low, ell)

        def ref_index(layout, kinds):
            idx, off = [], 0
            for c, kd in zip(layout, kinds):
                if kd == 'const' and ell > 0:
                    idx += [-1]
                    continue
                idx += list(range(off, off + c['n']))
                off += c['n'] * (1 if kd == 'const' else 2)
            return np.array(idx)
        ci = ref_index(cols, [low.kind_of(low.variables[c['item']])[0] for c in cols])
        ri = ref_index(rows, [low.kind_of(problem.equations[r['item']]['LHS'])[0] for r in rows])
        vr = np.array([r['valid'] for r in rows for _ in range(r['n'])])
        vc = np.array([c['valid'] for c in cols for _ in range(c['n'])])
        assert vr.sum() == vc.sum(), ell
        for name, mine in (("M", M), ("L", L)):
            R = g[f"sf_l{ell}_{name}"]
            Rp = np.zeros((R.shape[0] + 1, R.shape[1] + 1)); Rp[:-1, :-1] = R
            ref = Rp[np.ix_(ri, ci)]
            got = mine * np.outer(vr, vc)
            assert np.allclose(got, ref, rtol=1e-11, atol=1e-12 * np.abs(ref).max()), (ell, name, np.abs(got - ref).max())
        # the boundary rows: radial (spin 0) valid at every l, angular (spins -, +) from l = 1 on
        for ie, eq in enumerate(problem.equations):
            if len(eq['tensorsig']) == 1 and type(eq['tensorsig'][0]).__name__ == "S2Coordinates":
                assert [r['valid'] for r in rows if r['item'] == ie] == [ell >= 1, ell >= 1]


def check_stress_free(g, tag, scheme, shape):
    import dedalus_b200 as d3
    start = {"sf_strong": "strong", "sf_big": "flow"}.get(tag, "noise")
    return _run(d3, g, tag, convection(d3, shape), scheme, start)


def check_driven(g, tag):
    """Driven inner wall: radial(u(r=Ri)) = 0, angular(u(r=Ri)) = uw, b(r=Ro) = bt (RK222); "drv_change": uw and bt are set
    anew after two steps, which must take effect in the next stage."""
    import dedalus_b200 as d3
    sc = convection(d3, (16, 8, 6), walls="driven", Ri=0.5, Ro=1.5)
    return _run(d3, g, tag, sc, "RK222", "noise", change=2 if tag == "drv_change" else None)


def check_lbvp(g):
    import dedalus_b200 as d3
    lb = vector_poisson(d3)
    solver = lb['problem'].build_solver()
    solver.solve()
    ref = g["lbvp_u"]
    _close(lb['u']['c'], ref, 1e-8, 1e-10 * np.abs(ref).max(), "u")
    for name, f in lb['taus'].items():
        ref = g[f"lbvp_{name}"]
        _close(f['c'], ref, 1e-6, 1e-4 * np.abs(ref).max(), name)
    return solver


def check_tasks(g):
    """radial(u(r=Ro)), angular(u(r=Ro)) and the surface shear angular(radial(strain_rate(r=Ri), 0), 0) -- radial interpolation of a
    rank-2 field in the k = 1 basis -- as handler tasks against the reference's handler output."""
    import dedalus_b200 as d3
    t = task_inputs(d3, g["task_u_c"])
    u = t['u']
    problem = d3.IVP([u], namespace=locals())
    problem.add_equation("dt(u) = 0")
    solver = problem.build_solver(d3.SBDF1)
    handler = solver.evaluator.add_dictionary_handler(iter=1)
    for name, op in t['tasks'].items():
        handler.add_task(op, layout='g', name=name, scales=3/2)
    solver.evaluator.evaluate_handlers([handler], iteration=0, wall_time=0, sim_time=0, timestep=1)
    for name in t['tasks']:
        ref = g[f"task_{name}_g"]
        _close(np.asarray(handler.fields[name]), ref, 1e-9, 1e-11 * np.abs(ref).max(), name)


def _component_case(k, dealias, radius, Nr=10):
    """The reference's radial / angular component tests (tests/test_spherical_operators.py:565-660) on the shell, real dtype."""
    import dedalus_b200 as d3
    coords = d3.SphericalCoordinates('phi', 'theta', 'r')
    dist = d3.Distributor(coords, dtype=np.float64)
    shell = d3.ShellBasis(coords, (16, 8, Nr), radii=(0.5, 1.5), k=k, dealias=(dealias,) * 3, dtype=np.float64)
    phi, theta, r = dist.local_grids(shell, scales=(dealias,) * 3)
    x, y, z = coords.cartesian(phi, theta, r)
    return d3, coords, dist, shell, phi, theta, r, x, y, z


def check_radial_component_vector(k, dealias, radius):
    d3, c, dist, b, phi, theta, r, x, y, z = _component_case(k, dealias, radius)
    ct, st, cp, sp = np.cos(theta), np.sin(theta), np.cos(phi), np.sin(phi)
    u = dist.VectorField(c, bases=b)
    u.preset_scales(dealias)
    _velocity(u, r, ct, st, cp, sp, theta, phi)
    v = d3.RadialComponent(d3.interp(u, r=radius)).evaluate()
    vg = radius**2*st*(2*ct**2*cp-radius*ct**3*sp+radius**3*cp**3*st**5*sp**3+radius*ct*st**2*(cp**3+sp**3))
    assert np.allclose(v['g'], vg)


def check_angular_component_vector(k, dealias, radius):
    d3, c, dist, b, phi, theta, r, x, y, z = _component_case(k, dealias, radius)
    ct, st, cp, sp = np.cos(theta), np.sin(theta), np.cos(phi), np.sin(phi)
    u = dist.VectorField(c, bases=b)
    u.preset_scales(dealias)
    _velocity(u, r, ct, st, cp, sp, theta, phi)
    v = d3.AngularComponent(d3.interp(u, r=radius)).evaluate()
    vg = 0 * v['g']
    vg[0] = radius**2*sp*(-2*ct**2+radius*ct*cp*st**2*sp-radius**3*cp**2*st**5*sp**3)
    vg[1] = radius**2*(2*ct**3*cp-radius*cp**3*st**4+radius**3*ct*cp**3*st**5*sp**3-1/16*radius*np.sin(2*theta)**2*(-7*sp+np.sin(3*phi)))
    assert np.allclose(v['g'], vg)


def check_radial_component_tensor(k, dealias, radius):
    d3, c, dist, b, phi, theta, r, x, y, z = _component_case(k, dealias, radius)
    T = dist.TensorField((c, c), bases=b)
    T.preset_scales(dealias)
    _tensor(T, r, theta, x, y, z)
    A = d3.RadialComponent(d3.interp(T, r=radius)).evaluate()
    Ag = 0 * A['g']
    Ag[2] = 2*np.sin(theta)*(3*np.cos(phi)**2*np.sin(theta)+2*np.cos(theta)*np.sin(phi))
    Ag[1] = 6*np.cos(theta)*np.cos(phi)**2*np.sin(theta) + 2*np.cos(2*theta)*np.sin(phi)
    Ag[0] = 2*np.cos(phi)*(np.cos(theta) - 3*np.sin(theta)*np.sin(phi))
    assert np.allclose(A['g'], Ag)


def check_angular_component_tensor(k, dealias, radius):
    d3, c, dist, b, phi, theta, r, x, y, z = _component_case(k, dealias, radius)
    T = dist.TensorField((c, c), bases=b)
    T.preset_scales(dealias)
    _tensor(T, r, theta, x, y, z)
    A = d3.AngularComponent(d3.interp(T, r=radius), index=1).evaluate()
    Ag = 0 * A['g']
    Ag[2, 1] = 6*np.cos(theta)*np.cos(phi)**2*np.sin(theta) + 2*np.cos(2*theta)*np.sin(phi)
    Ag[2, 0] = 2*np.cos(phi)*(np.cos(theta) - 3*np.sin(theta)*np.sin(phi))
    Ag[1, 1] = 2*np.cos(theta)*(3*np.cos(theta)*np.cos(phi)**2 - 2*np.sin(theta)*np.sin(phi))
    Ag[1, 0] = Ag[0, 1] = -2*np.cos(phi)*(np.sin(theta) + 3*np.cos(theta)*np.sin(phi))
    Ag[0, 0] = 6*np.sin(phi)**2
    assert np.allclose(A['g'], Ag)
    # the spin components of the mixed (spherical, S2) result transform back to the same grid values
    A['c']
    assert np.allclose(A['g'], Ag)


def check_component_index_errors():
    import dedalus_b200 as d3
    import pytest
    coords = d3.SphericalCoordinates('phi', 'theta', 'r')
    dist = d3.Distributor(coords, dtype=np.float64)
    shell = d3.ShellBasis(coords, (16, 8, 6), radii=(0.5, 3), dtype=np.float64)
    u = dist.VectorField(coords, bases=shell)
    for op in (d3.radial, d3.angular):
        with pytest.raises(ValueError):
            op(u(r=1), index=1)
    T = dist.TensorField((coords, coords), bases=shell)
    assert d3.angular(T(r=1), 1).tensorsig == (coords, coords.S2coordsys)
    assert d3.radial(T(r=1), -1).tensorsig == (coords,)


def _velocity(u, r, ct, st, cp, sp, theta, phi):
    u['g'][2] = r**2*st*(2*ct**2*cp-r*ct**3*sp+r**3*cp**3*st**5*sp**3+r*ct*st**2*(cp**3+sp**3))
    u['g'][1] = r**2*(2*ct**3*cp-r*cp**3*st**4+r**3*ct*cp**3*st**5*sp**3-1/16*r*np.sin(2*theta)**2*(-7*sp+np.sin(3*phi)))
    u['g'][0] = r**2*sp*(-2*ct**2+r*ct*cp*st**2*sp-r**3*cp**2*st**5*sp**3)


def _tensor(T, r, theta, x, y, z):
    T['g'][2, 2] = (6*x**2+4*y*z)/r**2
    T['g'][2, 1] = T['g'][1, 2] = -2*(y**3+x**2*(y-3*z)-y*z**2)/(r**3*np.sin(theta))
    T['g'][2, 0] = T['g'][0, 2] = 2*x*(z-3*y)/(r**2*np.sin(theta))
    T['g'][1, 1] = 6*x**2/(r**2*np.sin(theta)**2) - (6*x**2+4*y*z)/r**2
    T['g'][1, 0] = T['g'][0, 1] = -2*x*(x**2+y**2+3*y*z)/(r**3*np.sin(theta)**2)
    T['g'][0, 0] = 6*y**2/(x**2+y**2)
