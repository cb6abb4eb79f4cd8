"""Tile heights of the register real-Fourier kernels at the benchmark's 256^3 on the GPU: the fused x pass of the RB3D right-hand
side at 4 and 8 line pairs per tile (DB_XPROD_P), and the y-pass transforms at 4 and 8 (DB_FFT_P), bitwise."""
import numpy as np, pytest
import rhs_fused_cases as cases


@pytest.mark.gpu
def test_fused_pass_at_4_line_pairs_equals_8_at_256(monkeypatch):
    solver = cases.rayleigh_benard(dim=3, Nh=256, Nz=256)
    plan = solver.rhs_plan
    assert plan.use_x_products and plan.n_in == 15 and plan.n_out == 4
    fused = {}
    for p in ("8", "4"):
        monkeypatch.setenv("DB_XPROD_P", p)
        fused[p] = cases.evaluate(solver, True)
    assert np.abs(fused["8"]).max() > 0
    assert np.array_equal(fused["4"], fused["8"])


@pytest.mark.gpu
def test_y_pass_at_4_line_pairs_equals_8_at_256(monkeypatch):
    import torch
    from dedalus_b200.transforms import RealFourierTransform
    N, G = 256, 384
    rf = RealFourierTransform(G, N)
    gen = torch.Generator(device='cuda').manual_seed(5)
    c = torch.randn((N, N, G), dtype=torch.float64, device='cuda', generator=gen)
    g = torch.randn((N, G, G), dtype=torch.float64, device='cuda', generator=gen)
    out = {}
    for p in ("8", "4"):
        monkeypatch.setenv("DB_FFT_P", p)
        gb, cf, gd = torch.empty_like(g), torch.empty_like(c), torch.empty_like(g)
        rf.backward(c, gb, 1)
        rf.backward(c, gd, 1, deriv=1)
        rf.forward(g, cf, 1)
        out[p] = [t.cpu().numpy() for t in (gb, gd, cf)]
    for a, b in zip(out["4"], out["8"]):
        assert np.array_equal(a, b)
