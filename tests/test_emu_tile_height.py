"""The tile of the register real-Fourier kernels (csrc/rfft_regs.cu: 8 line pairs, 16 lines), under the kernel emulation: the CTAs
per SM their persistent grids launch, and the standalone transforms in blocked row addressing against plain rows.  The arithmetic
applied to a line pair does not depend on where its rows are, so the comparison is bitwise.  The fused x pass of the right-hand side
against the separate passes: tests/test_emu_rhs_fused.py."""
import os, pathlib, subprocess, sys
import numpy as np, pytest
from emu import emu_lib as E

ROOT = pathlib.Path(__file__).resolve().parents[1]


def test_ctas_per_sm_at_8_line_pairs():
    # The emulation has no occupancy calculator: it reports the shared-memory fit (226 KB per SM), capped by the launch bounds.
    lib = E.emu()
    assert lib._raw_db_rfft_blocks_per_sm(2, 384, 256, 3) == 1             # fused x pass, three held factors: 224 KB
    assert lib._raw_db_rfft_blocks_per_sm(0, 384, 256, 0) == 2             # backward: 96 KB
    assert lib._raw_db_rfft_blocks_per_sm(0, 96, 64, 0) == 8               # 24 KB, capped at 8
    assert lib._raw_db_rfft_blocks_per_sm(0, 100, 64, 0) == -1             # no register kernel at n = 100
    assert lib._raw_db_rfft_blocks_per_sm(3, 384, 256, 0) == -1


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
@pytest.mark.parametrize("blocks", [2, 4])
@pytest.mark.parametrize("deriv", [0, 1])
def test_blocked_standalone_transforms_equal_plain(N, blocks, deriv):
    lib = E.emu(); plan = E.EmuPlan(N, 'real')
    M = 2 * N // 3
    rng = np.random.default_rng(N + blocks + deriv)
    nf, outer, inner = 2, 3, 48                     # 9 tiles of 8 line pairs over a few persistent CTAs
    c = rng.standard_normal((nf, outer, M, inner)); c[:, :, 1, :] = 0
    g = rng.standard_normal((nf, outer, N, inner))
    out = {}
    for b in (1, blocks):
        served = lib.rfft_regs_launches()
        out[b] = _standalone(lib, plan, N, M, b, c, g, deriv, 1.3)
        assert lib.rfft_regs_launches() == served + 2 * nf
    # back to (nf, outer, rows, inner) from the per-peer blocks
    unblocked = [a.transpose(1, 2, 0, 3, 4).reshape(nf, outer, -1, inner) for a in out[blocks]]
    for a, b in zip(unblocked, out[1]):
        assert not np.isnan(b).any()
        assert np.array_equal(a, b)


@pytest.mark.parametrize("env", [dict(DB_EMU_CP="early"), dict(DB_EMU_ORDER="reverse")])
def test_blocked_transforms_under_the_other_emulation_models(env):
    """cp.async copies landing at issue (a staging buffer refilled while still read) and threads scheduled in reverse order (a
    missing barrier)."""
    cmd = [sys.executable, "-m", "pytest", "-q", "-x", "-p", "no:cacheprovider", str(ROOT / "tests" / "test_emu_tile_height.py"),
           "-k", "equal_plain"]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=1800, env=dict(os.environ, **env), cwd=str(ROOT))
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-2000:]
    assert " passed" in out.stdout and "failed" not in out.stdout
