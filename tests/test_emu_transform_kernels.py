"""The spectral transform kernels -- real and complex Fourier and Chebyshev in csrc/fft.cu (k_fft) and csrc/rfft_regs.cu (register
kernels, blocked / peer entries, the fused x pass) -- through the CPU emulation of the kernels, against long-double references at
every path they dispatch to; GPU version: tests/test_gpu_1e_transform_kernels.py.  Shared bodies and bounds:
tests/transform_kernel_cases.py."""
import os, subprocess, sys, pathlib
import numpy as np, pytest
from emu import emu_lib as E
from kernel_backends import EmuArrays
import transform_kernel_cases as K

ROOT = pathlib.Path(__file__).resolve().parents[1]
B = EmuArrays()


@pytest.fixture(autouse=True)
def emulation():
    E.install()
    yield
    E.uninstall()


@pytest.fixture(scope="module", autouse=True)
def ratio_report():
    yield
    print("\nlargest error / bound per path (C_BOUND = %g):\n%s" % (K.C_BOUND, K.report()))


# ---- db_rfft_forward / db_rfft_backward on the register kernels
@pytest.mark.parametrize("n,M,outer,inner", K.register_rfft_shapes())
def test_rfft_register(n, M, outer, inner):
    assert K.check_rfft(B, n, M, outer, inner, derivs=(0, 1, 2, 3, 4)) is True


def test_rfft_register_many_tiles_per_cta():
    """inner = 16 * 20 at n = 48: 20 tiles per outer index and 3 outer indices walk through the persistent CTAs (one SM here)."""
    assert K.check_rfft(B, 48, 32, 3, 320, derivs=(0, 3), impulse=False) is True


# ---- fall-backs to k_fft and its own sizes
def test_rfft_fallbacks():
    K.check_rfft_fallbacks(B)


def test_rfft_generic_lengths():
    K.check_rfft_generic_lengths(B)


def test_rfft_narrow_tile():
    K.check_rfft_narrow_tile(B)


def test_rfft_backward_odd_M_reads_no_row_past_the_line():
    K.check_rfft_backward_odd_M_reads_no_row_past_the_line(B)


# ---- db_cfft_*
@pytest.mark.parametrize("n,M,outer,inner", [(16, 16, 3, 1), (16, 15, 1, 5), (24, 16, 2, 3), (22, 15, 4, 1), (15, 15, 2, 2),
                                             (96, 64, 1, 2), (12, 12, 1, 7)])
def test_cfft(n, M, outer, inner):
    K.check_cfft(B, n, M, outer, inner)


# ---- Chebyshev
@pytest.mark.parametrize("n,M,lines", K.register_cheb_shapes())
def test_cheb_register(n, M, lines):
    K.check_cheb(B, n, M, lines, 1, nds=(0, 3, 5) if M >= 6 else (0, 3))


@pytest.mark.parametrize("n,M,outer,inner,pre_sol", [
    (24, 16, 2, 5, ((2, 1), (3, 2))),          # strided axis
    (20, 15, 9, 1, ((1, 1),)),                 # n outside the register list, odd M
    (48, 33, 3, 3, ((3, 1),)),                 # odd M on a strided axis
    (30, 40, 5, 1, ((2, 1),)),                 # M > n: modes past n dropped
    (96, 64, 17, 1, ((2, 1), (0, 2))),         # contiguous lines with banded work: k_fft, the scan entry is separate
    (15, 10, 2, 4, ()),                        # odd n: the full-length complex FFT
])
def test_cheb_generic(n, M, outer, inner, pre_sol):
    K.check_cheb(B, n, M, outer, inner, nds=(0, 3), pre_sol=pre_sol)


def test_cheb_misaligned_falls_back():
    for mis in ((True, False), (False, True)):
        K.check_cheb(B, 48, 32, 5, 1, nds=(0, 3), misalign=mis, impulse=False)


@pytest.mark.parametrize("n,M,lines", [(48, 32, 17), (384, 256, 5), (24, 16, 1)])
@pytest.mark.parametrize("npre", [0, 1, 2, 3])
def test_cheb_backward_scan(n, M, lines, npre):
    K.check_cheb_scan(B, n, M, lines, npre)


def test_cheb_backward_scan_declines():
    K.check_cheb_scan_declines(B)


@pytest.mark.parametrize("stride", [1, 2])
@pytest.mark.parametrize("n,lines,npre", [(64, 45, 0), (50, 33, 2), (96, 70, 3)])
def test_band_lines(n, lines, npre, stride):
    assert lines % 32 != 0
    K.check_band_lines(B, n, lines, npre, stride)


# ---- blocked and peer entries
@pytest.mark.parametrize("n_peers", [1, 2, 3, 4, 8])
@pytest.mark.parametrize("in_blocked", [False, True])
def test_blocked_and_peer(n_peers, in_blocked):
    n, M = {1: (24, 16), 2: (48, 32), 3: (96, 48), 4: (96, 64), 8: (192, 128)}[n_peers]
    K.check_blocked_and_peer(B, n, M, 2, 16, n_peers, in_blocked)


def test_blocked_and_peer_decline():
    K.check_blocked_declines(B)


# ---- db_rfft_x_products
@pytest.mark.parametrize("n,M", K.xprod_shapes())
def test_x_products_shapes(n, M):
    sched = ("linear_no_held", "one_held", "held_reuse", "three_held")[(n + M) % 4]
    K.check_x_products(B, n, M, 16, sched)


@pytest.mark.parametrize("sched", sorted(K.xprod_schedules()))
def test_x_products_schedules(sched):
    """Every schedule at n = 48 with padded strides (NaN between the inputs and between the outputs), random and impulse inputs,
    and 4 tiles walking through the persistent CTA."""
    for impulse in (False, True):
        K.check_x_products(B, 48, 30, 64, sched, in_pad=10, out_pad=6, impulse=impulse)


@pytest.mark.parametrize("n", [192, 384])
def test_x_products_long_lines(n):
    if n == 192:
        K.check_x_products(B, 192, 128, 32, "three_held", in_pad=2, out_pad=4)
    else:
        K.check_x_products(B, 384, 254, 16, "held_reuse", impulse=True)


def test_x_products_rejections():
    K.check_x_products_rejections(B)


def test_x_products_supported_agrees():
    K.check_x_products_supported_agrees(B)


# ---- the other emulation schedules
@pytest.mark.parametrize("env", [dict(DB_EMU_ORDER="reverse"), dict(DB_EMU_CP="early")])
def test_register_kernels_under_other_schedules(env):
    """The register kernels and the fused x pass with threads and blocks in descending order, and with their cp.async copies landing
    at issue (a staging buffer refilled while it is still being read would show)."""
    cmd = [sys.executable, "-m", "pytest", "-q", "-x", "-p", "no:cacheprovider", __file__, "-k",
           "(rfft_register and 96) or x_products_schedules or cheb_register and 96 or many_tiles"]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=1200, env=dict(os.environ, **env), cwd=str(ROOT))
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-2000:]
    assert " passed" in out.stdout and "failed" not in out.stdout
