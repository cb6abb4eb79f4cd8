"""The spectral transform kernels -- real and complex Fourier and Chebyshev in csrc/fft.cu (k_fft) and csrc/rfft_regs.cu (register
kernels, blocked / peer entries, the fused x pass) -- on the GPU against long-double references at every path they dispatch to; the
same bodies run through the emulation in tests/test_emu_transform_kernels.py.  Here also what the emulation leaves out: persistent
grids with fewer tiles than CTAs and with many more, the fused x pass at the benchmark's 256^3 shapes (checked on a sample of lines),
and a contiguous generic launch with more than 32768 tiles (a 2-D grid)."""
import numpy as np, pytest
from kernel_backends import DeviceArrays
import transform_kernel_cases as K

pytestmark = pytest.mark.gpu
B = DeviceArrays()


@pytest.fixture(scope="module", autouse=True)
def ratio_report():
    yield
    print("\nlargest error / bound per path (C_BOUND = %g):\n%s" % (K.C_BOUND, K.report()))


@pytest.mark.parametrize("n,M,outer,inner", K.register_rfft_shapes(full=True))
def test_rfft_register(n, M, outer, inner):
    assert K.check_rfft(B, n, M, outer, inner, derivs=(0, 1, 2, 3, 4)) is True


@pytest.mark.parametrize("n,M", [(96, 64), (384, 256)])
def test_rfft_register_persistent_grid_extremes(n, M):
    """The persistent grid with a single tile (inner = 16: one CTA), and with 4 tiles per SM (inner = 16 * SMs * 4)."""
    K.check_rfft(B, n, M, 1, 16, derivs=(0, 1), impulse=False)
    inner = 16 * B.sms * 4
    K.check_rfft(B, n, M, 1, inner, derivs=(0, 2), impulse=False)


def test_rfft_fallbacks():
    K.check_rfft_fallbacks(B)


def test_rfft_generic_lengths():
    K.check_rfft_generic_lengths(B)


def test_rfft_narrow_tile():
    K.check_rfft_narrow_tile(B)


def test_rfft_backward_odd_M_reads_no_row_past_the_line():
    K.check_rfft_backward_odd_M_reads_no_row_past_the_line(B)


def test_rfft_generic_contiguous_2d_grid():
    """inner = 1 with 16 * 32768 + 5 lines: more than 32768 tiles, so the generic kernel's grid has gy = 2 (a ragged last row)."""
    lines = 16 * 32768 + 5
    n, M = 20, 12
    K.check_rfft(B, n, M, lines, 1, derivs=(1,), impulse=False, forward=True)


@pytest.mark.parametrize("n,M,outer,inner", [(16, 16, 3, 1), (16, 15, 1, 5), (24, 16, 2, 3), (22, 15, 4, 1), (15, 15, 2, 2),
                                             (96, 64, 1, 2), (12, 12, 1, 7), (384, 256, 2, 33)])
def test_cfft(n, M, outer, inner):
    K.check_cfft(B, n, M, outer, inner)


@pytest.mark.parametrize("n,M,lines", K.register_cheb_shapes())
def test_cheb_register(n, M, lines):
    K.check_cheb(B, n, M, lines, 1, nds=(0, 3, 5) if M >= 6 else (0, 3))


@pytest.mark.parametrize("n,M,outer,inner,pre_sol", [
    (24, 16, 2, 5, ((2, 1), (3, 2))),
    (20, 15, 9, 1, ((1, 1),)),
    (48, 33, 3, 3, ((3, 1),)),
    (30, 40, 5, 1, ((2, 1),)),
    (96, 64, 17, 1, ((2, 1), (0, 2))),
    (15, 10, 2, 4, ()),
])
def test_cheb_generic(n, M, outer, inner, pre_sol):
    K.check_cheb(B, n, M, outer, inner, nds=(0, 3), pre_sol=pre_sol)


def test_cheb_misaligned_falls_back():
    for mis in ((True, False), (False, True)):
        K.check_cheb(B, 48, 32, 5, 1, nds=(0, 3), misalign=mis, impulse=False)


@pytest.mark.parametrize("n,M,lines", [(48, 32, 17), (384, 256, 5), (24, 16, 1), (384, 384, 1000)])
@pytest.mark.parametrize("npre", [0, 1, 2, 3])
def test_cheb_backward_scan(n, M, lines, npre):
    K.check_cheb_scan(B, n, M, lines, npre)


def test_cheb_backward_scan_declines():
    K.check_cheb_scan_declines(B)


@pytest.mark.parametrize("stride", [1, 2])
@pytest.mark.parametrize("n,lines,npre", [(64, 45, 0), (50, 33, 2), (96, 70, 3), (256, 1001, 2)])
def test_band_lines(n, lines, npre, stride):
    K.check_band_lines(B, n, lines, npre, stride)


@pytest.mark.parametrize("n_peers", [1, 2, 3, 4, 8])
@pytest.mark.parametrize("in_blocked", [False, True])
def test_blocked_and_peer(n_peers, in_blocked):
    n, M = {1: (24, 16), 2: (48, 32), 3: (96, 48), 4: (96, 64), 8: (192, 128)}[n_peers]
    K.check_blocked_and_peer(B, n, M, 2, 16, n_peers, in_blocked)


def test_blocked_and_peer_decline():
    K.check_blocked_declines(B)


@pytest.mark.parametrize("n,M", K.xprod_shapes())
def test_x_products_shapes(n, M):
    sched = ("linear_no_held", "one_held", "held_reuse", "three_held")[(n + M) % 4]
    K.check_x_products(B, n, M, 16, sched)


@pytest.mark.parametrize("sched", sorted(K.xprod_schedules()))
def test_x_products_schedules(sched):
    for impulse in (False, True):
        K.check_x_products(B, 48, 30, 64, sched, in_pad=10, out_pad=6, impulse=impulse)


@pytest.mark.parametrize("case", ["192", "384", "many_tiles"])
def test_x_products_long_lines(case):
    if case == "192":
        K.check_x_products(B, 192, 128, 32, "three_held", in_pad=2, out_pad=4)
    elif case == "384":
        K.check_x_products(B, 384, 254, 16, "held_reuse", impulse=True)
    else:                                               # many more tiles than the persistent grid has CTAs
        K.check_x_products(B, 96, 64, 16 * B.sms * 6, "three_held", in_pad=2, out_pad=2)


@pytest.mark.parametrize("sched", ["three_held", "held_reuse"])
def test_x_products_benchmark_shape(sched):
    """The x-line length and coefficient count of the 256^3 benchmark (n = 384, M = 256) over 49152 lines, checked on a sample of
    line pairs: the benchmark's schedule (three held factors) and one that reuses a held factor."""
    K.check_x_products_large(B, 384, 256, 192 * 256, sched, sample=96)


def test_x_products_rejections():
    K.check_x_products_rejections(B)


def test_x_products_supported_agrees():
    K.check_x_products_supported_agrees(B)
