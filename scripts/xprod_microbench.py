"""Time the fused x pass of the right-hand side (db_rfft_x_products) alone at the RB3D 256^3 shape, and the y-pass-shaped register
transforms.

The fused pass runs the schedule of a real RB3D RHSPlan (15 inputs, 4 outputs, 3 held factors) on M = 256 coefficient rows of
n = 384 points and inner = 384^2 random lines.  Each kernel is timed with CUDA events over 20 launches after a warm-up, 3 rounds,
and the median round is reported.  Algorithmic traffic is every input and output array read
or written once.  Blocks per SM come from cudaOccupancyMaxActiveBlocksPerMultiprocessor (db_rfft_blocks_per_sm).

usage: python scripts/xprod_microbench.py [--json PATH]"""
import argparse, json, pathlib, statistics, subprocess, sys
sys.path.insert(0, str(pathlib.Path(__file__).resolve().parents[1]))
import torch

LAUNCHES, ROUNDS = 20, 3


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as exc:
        q = f"{torch.cuda.get_device_name()} (nvidia-smi unavailable: {exc})"
    return q


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(LAUNCHES):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / LAUNCHES


def rounds(fn):
    """ms per launch in each of ROUNDS rounds, after a warm-up launch (module load, attributes)."""
    fn()
    torch.cuda.synchronize()
    return [timed(fn) for _ in range(ROUNDS)]


def row(name, res, gb, bps):
    ms = statistics.median(res)
    print(f"{name:18s} {ms:12.3f} {min(res):8.3f} {max(res):8.3f} {gb / (ms * 1e-3):8.1f} {bps:8d}")
    return dict(ms=res, gbps=gb / (ms * 1e-3), blocks_per_sm=bps)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    import dedalus_b200 as d3
    from dedalus_b200 import examples
    from dedalus_b200.lib import get_lib
    from dedalus_b200.transforms import RealFourierTransform
    torch.cuda.set_device(0)
    lib = get_lib()
    out = dict(card=card(), y_pass={})
    print(f"card: {out['card']}")

    # the RB3D schedule at a 384-point x line (the y and z sizes do not enter it)
    pb = examples.rayleigh_benard(dim=3, Nx=256, Nh=16, Nz=16, Rayleigh=1e6)
    solver = pb['problem'].build_solver(d3.RK222)
    solver._init_device()
    xp = solver.rhs_plan.xprod
    px = xp['plan']
    n, M, n_out = px.N, px.M, solver.rhs_plan.n_out
    inner = n * n
    loads = xp['loads']
    n_src = int(loads.max().item()) + 1
    cin = torch.randn((n_src, M, inner), dtype=torch.float64, device='cuda')
    cout = torch.empty((n_out, M, inner), dtype=torch.float64, device='cuda')
    gb = 8 * (int(loads.numel()) + n_out) * M * inner / 1e9
    res = rounds(lambda: px.x_products(cin, cout, inner, xp['items'], xp['n_items'], loads, xp['n_held']))
    print(f"\nfused x pass: n = {n}, M = {M}, inner = {inner}, {loads.numel()} inputs, {n_out} outputs, {xp['n_held']} held, "
          f"{gb:.2f} GB per launch")
    print(f"{'kernel':18s} {'ms (median)':>12s} {'min':>8s} {'max':>8s} {'GB/s':>8s} {'CTAs/SM':>8s}")
    out['fused'] = row("fused", res, gb, lib._raw_db_rfft_blocks_per_sm(2, n, M, xp['n_held']))
    del cin, cout

    # y pass of RB3D 256^3: (256, 256, 384) coefficients <-> (256, 384, 384) grid along axis 1
    N, G = 256, 384
    rf = RealFourierTransform(G, N)
    c = torch.randn((N, N, G), dtype=torch.float64, device='cuda')
    g = torch.randn((N, G, G), dtype=torch.float64, device='cuda')
    gb = 8 * (c.numel() + g.numel()) / 1e9
    print(f"\ny pass: n = {G}, M = {N}, outer = {N}, inner = {G}, {gb:.2f} GB per launch")
    print(f"{'kernel':18s} {'ms (median)':>12s} {'min':>8s} {'max':>8s} {'GB/s':>8s} {'CTAs/SM':>8s}")
    for kind, label, fn in ((0, "backward", lambda: rf.backward(c, g, 1)), (1, "forward", lambda: rf.forward(g, c, 1))):
        out['y_pass'][label] = row(label, rounds(fn), gb, lib._raw_db_rfft_blocks_per_sm(kind, G, N, 0))
    if args.json:
        pathlib.Path(args.json).parent.mkdir(parents=True, exist_ok=True)
        pathlib.Path(args.json).write_text(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
