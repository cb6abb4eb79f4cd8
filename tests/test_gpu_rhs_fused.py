"""The fused x pass of the right-hand side (k_rfft_x_products) against the separate passes at the benchmark's 256^3, on the GPU."""
import numpy as np, pytest
import rhs_fused_cases as cases


@pytest.mark.gpu
def test_fused_matches_separate_passes_256():
    plan, fused, separate = cases.compare(cases.rayleigh_benard(dim=3, Nh=256, Nz=256))
    assert plan.use_x_products and plan.n_in == 15 and plan.n_out == 4
    scale = np.abs(separate).max()
    err = np.abs(fused - separate).max() / scale
    # the two paths share the register DFT stages and the product arithmetic; nvcc may contract a multiply-add differently
    # where the stages are inlined into another kernel, which is the only room left for a difference
    assert err <= 1e-14, err
    print(f"fused vs separate at 256^3: max |diff| / max |rhs| = {err:.3e} (bitwise equal: {np.array_equal(fused, separate)})")
