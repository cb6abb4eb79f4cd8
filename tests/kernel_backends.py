"""The array backends of the kernel-level test bodies (curvilinear_kernel_cases.py, transform_kernel_cases.py): the same body runs
through the CPU emulation of the kernels (EmuArrays: numpy arrays) and on the GPU (DeviceArrays: torch tensors).

B.dev(numpy) -> device array, B.ptr(device array) -> c_void_p, B.host(device array) -> numpy, B.lib, B.stream, B.sms (streaming
multiprocessors), B.dev_at(numpy, off) -> device array whose first element sits 8 bytes past a 16-byte boundary when off is true, and on
one otherwise, B.plan(n, kind) -> FFT plan tables of fftplan.HostPlan where the kernels read them (.ref() is the struct pointer)."""
import ctypes as C
import numpy as np


class EmuArrays:
    """numpy arrays + the emulated library."""
    stream = None
    sms = 132                       # csrc/core.cu: db_num_sms() of the emulation
    emulated = True

    @property
    def lib(self):
        from emu import emu_lib as E
        return E.emu()

    def dev(self, a):
        return self.dev_at(a, False)

    def dev_at(self, a, off):
        a = np.ascontiguousarray(a)
        raw = np.empty(a.nbytes + 32, dtype=np.uint8)
        start = (-raw.ctypes.data) % 16 + (8 if off else 0)
        out = raw[start:start + a.nbytes].view(a.dtype).reshape(a.shape)
        out[...] = a
        return out

    def ptr(self, a):
        from emu import emu_lib as E
        return E.ptr(a)

    def host(self, a):
        return a

    def plan(self, n, kind):
        from emu import emu_lib as E
        return E.EmuPlan(n, kind)


class DeviceArrays:
    """torch tensors on the compute device + the bound library."""
    emulated = False

    @property
    def lib(self):
        from dedalus_b200.lib import get_lib
        return get_lib()

    @property
    def stream(self):
        from dedalus_b200.lib import current_stream
        return current_stream()

    @property
    def sms(self):
        import torch
        return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count if torch.cuda.is_available() else 132

    def dev(self, a):
        return self.dev_at(a, False)

    def dev_at(self, a, off):
        import torch
        from dedalus_b200.lib import compute_device
        a = np.ascontiguousarray(a)
        raw = torch.empty(a.nbytes + 32, dtype=torch.uint8, device=compute_device())
        start = (-raw.data_ptr()) % 16 + (8 if off else 0)
        out = raw[start:start + a.nbytes]
        out.copy_(torch.from_numpy(a.reshape(-1).view(np.uint8).copy()))
        out = out.view(getattr(torch, a.dtype.name)).reshape(a.shape)
        assert out.data_ptr() % 16 == (8 if off else 0)
        return out

    def ptr(self, t):
        return C.c_void_p(t.data_ptr())

    def host(self, t):
        return t.cpu().numpy()

    def plan(self, n, kind):
        from dedalus_b200.lib import compute_device
        from dedalus_b200.transforms import DevicePlan
        return DevicePlan(n, kind, compute_device())
