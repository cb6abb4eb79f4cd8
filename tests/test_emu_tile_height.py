"""Tile heights of the register real-Fourier kernels (csrc/rfft_regs.cu), under the kernel emulation.  The fused x pass of the
right-hand side (k_rfft_x_products) at 4 line pairs per tile (DB_XPROD_P) is compared with 8 and with the separate passes,
and the standalone transforms at 4 line pairs (DB_FFT_P) with 8, in plain and blocked row addressing.  The arithmetic applied to a
line pair does not depend on the tile height, so every comparison is bitwise."""
import os, pathlib, subprocess, sys
import numpy as np, pytest
from emu import emu_lib as E
import rhs_fused_cases as cases

ROOT = pathlib.Path(__file__).resolve().parents[1]


@pytest.fixture
def emulation():
    E.install()
    yield
    E.uninstall()


@pytest.mark.parametrize("case", sorted(cases.CASES))
def test_fused_pass_is_bitwise_equal_at_every_tile_height(case, emulation, monkeypatch):
    solver = cases.CASES[case]()
    plan = solver.rhs_plan
    assert plan.use_x_products
    fused = {}
    for p in ("8", "4"):
        monkeypatch.setenv("DB_XPROD_P", p)
        fused[p] = cases.evaluate(solver, True)
    separate = cases.evaluate(solver, False)
    assert np.abs(separate).max() > 0
    assert np.array_equal(fused["4"], fused["8"])
    assert np.array_equal(fused["4"], separate)


def test_lower_tiles_fit_more_ctas_per_sm():
    # fused x pass at n = 384, M = 256, three held factors: 224 KB at 8 line pairs, 112 KB at 4.  The emulation has no occupancy
    # calculator: it reports the shared-memory fit (226 KB per SM), capped by the launch bounds.
    lib = E.emu()
    per_sm = {p: lib._raw_db_rfft_blocks_per_sm(2, 384, 256, 3, p) for p in (8, 4, 2)}
    assert per_sm == {8: 1, 4: 2, 2: -1}
    assert lib._raw_db_rfft_blocks_per_sm(0, 384, 256, 0, 4) == 4
    assert lib._raw_db_rfft_blocks_per_sm(0, 96, 64, 0, 4) == -1          # P = 4 exists at n = 192 and 384 only


def _blocked(a, rows, rpb):
    # (nf, outer, rows, inner) -> (rows // rpb, nf, outer, rpb, inner): the per-peer blocks of an all-to-all buffer
    nf, outer, _, inner = a.shape
    return np.ascontiguousarray(a.reshape(nf, outer, rows // rpb, rpb, inner).transpose(2, 0, 1, 3, 4))


def _standalone(lib, plan, N, M, blocks, c, g, deriv, kscale):
    """backward of c and forward of g, plain (blocks = 1) or with blocked input and output rows (blocks peers)"""
    nf, outer, _, inner = c.shape
    gout = np.full((nf, outer, N, inner), np.nan); cout = np.full((nf, outer, M, inner), np.nan)
    if blocks == 1:
        for f in range(nf):
            lib.call("db_rfft_backward", plan.ref(), E.ptr(np.ascontiguousarray(c[f])), E.ptr(gout[f]), outer, M, inner, deriv, kscale, None)
            lib.call("db_rfft_forward", plan.ref(), E.ptr(np.ascontiguousarray(g[f])), E.ptr(cout[f]), outer, M, inner, None)
        return gout, cout
    cin, gin = _blocked(c, M, M // blocks), _blocked(g, N, N // blocks)
    gout, cout = _blocked(gout, N, N // blocks), _blocked(cout, M, M // blocks)
    per_c, per_g = outer * (M // blocks) * inner, outer * (N // blocks) * inner
    for f in range(nf):
        assert lib.call_optional("db_rfft_backward_blocked", plan.ref(), E.ptr(cin.reshape(-1)[f * per_c:]), E.ptr(gout.reshape(-1)[f * per_g:]),
                                 outer, M, inner, deriv, kscale, M // blocks, nf * per_c, N // blocks, nf * per_g, None)
        assert lib.call_optional("db_rfft_forward_blocked", plan.ref(), E.ptr(gin.reshape(-1)[f * per_g:]), E.ptr(cout.reshape(-1)[f * per_c:]),
                                 outer, M, inner, N // blocks, nf * per_g, M // blocks, nf * per_c, None)
    return gout, cout


@pytest.mark.parametrize("N", [192, 384])
@pytest.mark.parametrize("blocks", [1, 4])
@pytest.mark.parametrize("deriv", [0, 1])
def test_standalone_transforms_are_bitwise_equal_at_4_and_8_line_pairs(N, blocks, deriv, monkeypatch):
    lib = E.emu(); plan = E.EmuPlan(N, 'real')
    M = 2 * N // 3
    rng = np.random.default_rng(N + blocks + deriv)
    nf, outer, inner = 2, 3, 48                     # 9 tiles of 8 line pairs, 18 of 4, over a few persistent CTAs
    c = rng.standard_normal((nf, outer, M, inner)); c[:, :, 1, :] = 0
    g = rng.standard_normal((nf, outer, N, inner))
    out = {}
    for p in ("8", "4"):
        monkeypatch.setenv("DB_FFT_P", p)
        served = lib.rfft_regs_launches()
        out[p] = _standalone(lib, plan, N, M, blocks, c, g, deriv, 1.3)
        assert lib.rfft_regs_launches() == served + 2 * nf
    for a, b in zip(out["4"], out["8"]):
        assert not np.isnan(b).any()
        assert np.array_equal(a, b)


@pytest.mark.parametrize("env", [dict(DB_EMU_CP="early"), dict(DB_EMU_ORDER="reverse")])
def test_tile_heights_under_the_other_emulation_models(env):
    """cp.async copies landing at issue (a staging buffer refilled while still read) and threads scheduled in reverse order (a
    missing barrier)."""
    cmd = [sys.executable, "-m", "pytest", "-q", "-x", "-p", "no:cacheprovider", str(ROOT / "tests" / "test_emu_tile_height.py"),
           "-k", "bitwise_equal"]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=1800, env=dict(os.environ, **env), cwd=str(ROOT))
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-2000:]
    assert " passed" in out.stdout and "failed" not in out.stdout
