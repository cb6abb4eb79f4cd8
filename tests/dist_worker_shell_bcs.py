"""Worker for the 2-rank run in tests/test_emu_shell_bcs.py: stress-free shell convection (radial / angular boundary components)
distributed over the azimuthal pairs / colatitude, against the single-rank reference state of tests/golden/shell_bcs.npz.
gloo on the CPU (test-only kernel emulation), or nccl with DB_DIST_BACKEND=nccl."""
import os, sys, pathlib
import numpy as np
ROOT = pathlib.Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "tests"))
import torch
import torch.distributed as dist


def main():
    backend = os.environ.get("DB_DIST_BACKEND", "gloo")
    if backend == "nccl":
        local = int(os.environ.get("LOCAL_RANK", "0"))
        torch.cuda.set_device(local)
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    else:
        dist.init_process_group("gloo")
        from emu import emu_lib as E
        E.install()                      # CPU run: test-only kernel emulation
    rank = dist.get_rank()
    import dedalus_b200 as d3
    import shell_bc_cases as SBC
    tag = sys.argv[1] if len(sys.argv) > 1 else "sf_strong"
    g = np.load(ROOT / "tests" / "golden" / "shell_bcs.npz")
    steps, dtv = g[f"{tag}_meta"]
    sc = SBC.convection(d3, (16, 8, 6))
    solver = sc['problem'].build_solver(d3.SBDF2)
    rows = sc['dist'].coeff_local_slice(0, sc['shell'])
    sc['b']['c'] = g[f"{tag}_b0"][rows]; sc['u']['c'] = g[f"{tag}_u0"][:, rows]
    for _ in range(int(steps)):
        solver.step(float(dtv))
    ok = type(solver.rhs_plan).__name__ == "ShellRHSPlan"
    for name in ('p', 'b', 'u'):
        full = g[f"{tag}_{name}1"]
        ok = ok and bool(np.allclose(sc[name]['c'], full[..., rows, :, :], rtol=1e-8, atol=1e-10 * np.abs(full).max()))
    for name in ('tau_b1', 'tau_b2', 'tau_u1', 'tau_u2'):
        full = g[f"{tag}_{name}1"]
        ok = ok and bool(np.allclose(sc['taus'][name]['c'], full[..., rows, :, :], rtol=1e-6, atol=1e-4 * np.abs(full).max() + 1e-20))
    flag = torch.tensor([1 if ok else 0], device='cuda' if backend == "nccl" else 'cpu')
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    if rank == 0:
        print("DIST_OK" if int(flag.item()) == 1 else "DIST_FAIL")
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
