"""Peak device memory of the 3-D Rayleigh-Benard benchmark problem (bench.py's workload): build, warm up, time-step, then
torch.cuda.max_memory_allocated.  DB_RHS_FUSED=0 gives the figure with the separate x passes and product kernel.

    python scripts/rhs_peak_memory.py [--size 256] [--steps 10] [--warmup 3]
"""
import argparse, json, os, pathlib, sys
sys.path.insert(0, str(pathlib.Path(__file__).resolve().parents[1]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=256)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    import dedalus_b200 as d3
    from dedalus_b200 import examples
    pb = examples.rayleigh_benard(dim=3, Nh=args.size, Nz=args.size, Rayleigh=1e6)
    solver = pb['problem'].build_solver(d3.RK222)
    examples.rayleigh_benard_initial_condition(pb['b'], pb['bases'], pb['Lz'])
    for _ in range(args.warmup + args.steps):
        solver.step(1e-4)
    torch.cuda.synchronize()
    print(json.dumps(dict(size=args.size, fused=bool(getattr(solver.rhs_plan, 'use_x_products', False)),
                          max_memory_allocated_GB=round(torch.cuda.max_memory_allocated() / 1e9, 3))))


if __name__ == "__main__":
    main()
