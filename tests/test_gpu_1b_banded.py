"""The banded pencil kernels (combine / factor / solve / matvec) on the GPU, against LAPACK; the same bodies run through the emulation
in tests/test_emu_banded.py.  This guards against regressions; it does not repeat runs to catch a race whose timing is unknown."""
import ctypes as C
import numpy as np, pytest
import banded_cases as BC

pytestmark = pytest.mark.gpu


class _CudaArrays:
    @property
    def lib(self):
        from dedalus_b200.lib import get_lib
        return get_lib()

    @property
    def stream(self):
        from dedalus_b200.lib import current_stream
        return current_stream()

    def dev(self, a):
        import torch
        return torch.from_numpy(np.ascontiguousarray(a).copy()).cuda()

    def ptr(self, t):
        return C.c_void_p(t.data_ptr())

    def host(self, t):
        return t.cpu().numpy()


@pytest.mark.parametrize("kl,ku", [(1, 1), (5, 3), (7, 7), (40, 2), (12, 20)])
def test_banded_small_systems(kl, ku):
    """n = 1 .. 9, 31, 32, 33, 100; 1, 8, 9 and 33 right-hand sides; x also solved in place.  (40, 2) and (12, 20) have more than 32
    rows per factor column (ldf = 83, 45), so each lane handles more than one entry of a column."""
    ns, nrhs = BC.small_batch()
    BC.check_banded(_CudaArrays(), kl, ku, ns, nrhs, seed=kl * 100 + ku)


@pytest.mark.parametrize("kl,ku", [(5, 3), (40, 2)])
def test_banded_config4_size(kl, ku):
    """n = 1530, the largest per-m system of the 512 x 256 shallow-water problem, next to short systems in the same batch."""
    BC.check_banded(_CudaArrays(), kl, ku, [1530, 3, 6, 1], [9, 9, 1, 33], seed=4)


@pytest.mark.parametrize("kl,ku", [(1, 1), (7, 7)])
def test_banded_past_eight_column_chunks(kl, ku):
    """max_n = 1600 > 1536: the solve stages 4 right-hand-side columns per CTA instead of 8."""
    BC.check_banded(_CudaArrays(), kl, ku, [1600, 2, 5, 1537], [9, 9, 8, 33], seed=5)
