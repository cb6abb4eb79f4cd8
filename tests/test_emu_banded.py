"""The banded pencil kernels (combine / factor / solve / matvec), through the CPU emulation of the kernels, against LAPACK; GPU
version: tests/test_gpu_1b_banded.py."""
import numpy as np, pytest
from emu import emu_lib as E
import banded_cases as BC


@pytest.fixture(autouse=True)
def emulation():
    E.install()
    yield
    E.uninstall()


class _EmuArrays:
    """numpy arrays + the emulated library, behind the interface banded_cases uses."""
    lib = property(lambda self: E.emu())
    stream = None

    def dev(self, a):
        return np.ascontiguousarray(a).copy()

    def ptr(self, a):
        return E.ptr(a)

    def host(self, a):
        return a


@pytest.mark.parametrize("kl,ku", [(1, 1), (5, 3), (7, 7), (40, 2), (12, 20)])
def test_banded_small_systems(kl, ku):
    """n = 1 .. 9, 31, 32, 33, 100; 1, 8, 9 and 33 right-hand sides; x also solved in place.  (40, 2) and (12, 20) have more than 32
    rows per factor column (ldf = 83, 45), so each lane handles more than one entry of a column."""
    ns, nrhs = BC.small_batch()
    BC.check_banded(_EmuArrays(), kl, ku, ns, nrhs, seed=kl * 100 + ku)


@pytest.mark.parametrize("kl,ku", [(5, 3), (40, 2)])
def test_banded_config4_size(kl, ku):
    """n = 1530, the largest per-m system of the 512 x 256 shallow-water problem, next to short systems in the same batch."""
    BC.check_banded(_EmuArrays(), kl, ku, [1530, 3, 6, 1], [9, 9, 1, 33], seed=4)


@pytest.mark.parametrize("kl,ku", [(1, 1), (7, 7)])
def test_banded_past_eight_column_chunks(kl, ku):
    """max_n = 1600 > 1536: the solve stages 4 right-hand-side columns per CTA instead of 8."""
    BC.check_banded(_EmuArrays(), kl, ku, [1600, 2, 5, 1537], [9, 9, 8, 33], seed=5)
