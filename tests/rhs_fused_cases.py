"""Problems whose right-hand sides take the fused x pass (k_rfft_x_products), on O(1)-velocity states, and the comparison of
the fused and the separate evaluation on one plan.  Shared by the emulated and the GPU tests."""
import numpy as np
import dedalus_b200 as d3
from dedalus_b200 import examples


def _randomize(fields, seed):
    rng = np.random.default_rng(seed)
    for f in fields:
        f['c'] = rng.uniform(-1.0, 1.0, size=np.shape(f['c']))


def _solver(problem, fields, seed=1):
    solver = problem.build_solver(d3.RK222)
    _randomize(fields, seed)
    solver._init_device()
    return solver


def rayleigh_benard(dim=3, **kw):
    pb = examples.rayleigh_benard(dim=dim, Rayleigh=1e6, **kw)
    return _solver(pb['problem'], [pb['u'], pb['b']])


def shear_flow(Nx=16, Nz=32):
    """The right-hand sides of the stock 2-D shear flow: - u@grad(u), - u@grad(s) on a doubly periodic domain."""
    coords = d3.CartesianCoordinates('x', 'z')
    dist = d3.Distributor(coords, dtype=np.float64)
    xbasis = d3.RealFourier(coords['x'], size=Nx, bounds=(0, 1), dealias=3/2)
    zbasis = d3.RealFourier(coords['z'], size=Nz, bounds=(-1, 1), dealias=3/2)
    p = dist.Field(name='p', bases=(xbasis, zbasis))
    s = dist.Field(name='s', bases=(xbasis, zbasis))
    u = dist.VectorField(coords, name='u', bases=(xbasis, zbasis))
    tau_p = dist.Field(name='tau_p')
    problem = d3.IVP([u, s, p, tau_p], namespace=dict(u=u, s=s, p=p, tau_p=tau_p, nu=2e-5, D=2e-5))
    problem.add_equation("dt(u) + grad(p) - nu*lap(u) = - u@grad(u)")
    problem.add_equation("dt(s) - D*lap(s) = - u@grad(s)")
    problem.add_equation("div(u) + tau_p = 0")
    problem.add_equation("integ(p) = 0")
    return _solver(problem, [u, s])


CASES = {
    "rb3d_16": lambda: rayleigh_benard(dim=3, Nh=16, Nz=16),
    "rb3d_x384": lambda: rayleigh_benard(dim=3, Nx=256, Nh=16, Nz=16),      # the benchmark's 384-point x line
    "rb2d_nz32": lambda: rayleigh_benard(dim=2, Nh=32, Nz=32),               # 48 z grid lines
    "shear": shear_flow,
}


def evaluate(solver, fused):
    import torch
    plan = solver.rhs_plan
    plan.use_x_products = fused
    out = torch.zeros_like(solver.eq_t)
    plan.set_static(out)
    plan.evaluate(out)
    return out.cpu().numpy().copy()


def compare(solver):
    """(plan, arena after the fused evaluation, arena after the separate passes); the plan is left on its automatic choice."""
    plan = solver.rhs_plan
    auto = plan.use_x_products
    try:
        fused = evaluate(solver, True) if plan.xprod is not None else None
        separate = evaluate(solver, False)
    finally:
        plan.use_x_products = auto
    return plan, fused, separate
