"""ctypes binding of the C ABI declared in include/dedalus_b200.h.

The product loads ONLY dedalus_b200/libdedalus_b200.so (nvcc, sm_90a).  If it is missing or cannot be loaded
the import of any compute path raises: there is no CPU fallback.  `bind()` is also used by the test-only CPU
emulation (tests/emu/emu_lib.py) to attach the same prototypes to tests/emu/libdedalus_b200_emu.so.
"""
import ctypes as C
import pathlib

PKG = pathlib.Path(__file__).resolve().parent
LIB_PATH = PKG / "libdedalus_b200.so"

i32, i64, f64, vp = C.c_int32, C.c_int64, C.c_double, C.c_void_p


class FftPlan(C.Structure):
    _fields_ = [("n", i32), ("nc", i32), ("half", i32), ("nrad", i32), ("rad", i32 * 16),
                ("tw", vp), ("twr", vp), ("twq", vp), ("perm", vp), ("iperm", vp), ("twn", vp)]


class LinComb(C.Structure):
    _fields_ = [("nvec", i32), ("vec", vp * 16), ("coef", f64 * 16)]


DB_MAX_VECS, DB_MAX_LU = 24, 4


class Batch(C.Structure):
    """include/dedalus_b200.h: db_batch"""
    _fields_ = [("n", i32), ("S", i32), ("ld", i32), ("n_entries", i32), ("n_fwd", i32), ("n_bwd", i32),
                ("blk_solve", i32), ("blk_matvec", i32), ("blk_move", i32 * 2), ("blk_assemble", i32),
                ("nlines", i32 * 2), ("max_len", i32 * 2),
                ("prog", vp), ("mono", vp), ("vec", vp * DB_MAX_VECS), ("lu", vp * DB_MAX_LU),
                ("m_ptr", vp), ("m_col", vp), ("m_mono", vp), ("m_val", vp),
                ("l_ptr", vp), ("l_col", vp), ("l_mono", vp), ("l_val", vp),
                ("m_rec", vp), ("l_rec", vp), ("ctrl", vp), ("n_mono", i32), ("mv_rows", i32), ("mv_win", vp), ("m_split", vp), ("l_split", vp),
                ("line_base", vp * 2), ("line_kind", vp * 2), ("line_ptr", vp * 2), ("line_pos", vp * 2), ("sys_off", vp * 2),
                ("nrhs", i32), ("line_sign", vp * 2),
                ("diag_eid", vp), ("fl_ptr", vp), ("fl_eid", vp), ("fu_ptr", vp), ("fu_eid", vp), ("fd_eid", vp),
                ("asm_ptr", vp), ("asm_mono", vp), ("asm_val", vp), ("info", vp)]


class RaggedEntry(C.Structure):
    """include/dedalus_b200.h: db_ragged_entry"""
    _fields_ = [("mat_off", i64), ("nrow", i32), ("ncol", i32), ("in_i0", i32), ("in_row0", i32), ("in_step", i32),
                ("out_i0", i32), ("out_row0", i32), ("out_step", i32), ("nm", i32), ("zero", i32)]


class SlotComb(C.Structure):
    _fields_ = [("nvec", i32), ("slot", i32 * 16), ("coef", f64 * 16)]


class BandedSys(C.Structure):
    """include/dedalus_b200.h: db_banded_sys"""
    _fields_ = [("n", i32), ("nrhs", i32), ("op_off", i64), ("lu_off", i64), ("piv_off", i64), ("vec_off", i64)]


class VecComb(C.Structure):
    """include/dedalus_b200.h: db_veccomb"""
    _fields_ = [("nvec", i32), ("vec", vp * 16), ("coef", f64 * 16)]


class DenseSys(C.Structure):
    """include/dedalus_b200.h: db_dense_sys"""
    _fields_ = [("ncols", i32), ("pad", i32), ("vec_off", i64)]


class PairLinTerm(C.Structure):
    """include/dedalus_b200.h: db_pair_lin_term"""
    _fields_ = [("re", f64), ("im", f64), ("sym_off", i64), ("src", i32), ("pad", i32)]


PFFT = C.POINTER(FftPlan)
PLIN = C.POINTER(LinComb)

SIGNATURES = {
    "db_last_error": (C.c_char_p, []),
    "db_version": (C.c_int, []),
    "db_device_arch": (C.c_int, []),
    "db_rfft_regs_launches": (C.c_longlong, []),
    "db_rfft_forward": (C.c_int, [PFFT, vp, vp, i64, i32, i64, vp]),
    "db_rfft_forward_blocked": (C.c_int, [PFFT, vp, vp, i64, i32, i64, i32, i64, i32, i64, vp]),
    "db_rfft_backward_blocked": (C.c_int, [PFFT, vp, vp, i64, i32, i64, i32, f64, i32, i64, i32, i64, vp]),
    "db_rfft_forward_peer": (C.c_int, [PFFT, vp, vp, i64, i32, i64, i32, i64, i32, i32, C.POINTER(vp), vp]),
    "db_rfft_backward_peer": (C.c_int, [PFFT, vp, vp, i64, i32, i64, i32, f64, i32, i64, i32, i32, C.POINTER(vp), vp]),
    "db_rfft_backward": (C.c_int, [PFFT, vp, vp, i64, i32, i64, i32, f64, vp]),
    "db_cfft_forward": (C.c_int, [PFFT, vp, vp, i64, i32, i64, vp]),
    "db_cfft_backward": (C.c_int, [PFFT, vp, vp, i64, i32, i64, i32, f64, vp]),
    "db_cheb_forward": (C.c_int, [PFFT, vp, vp, i64, i32, i64, vp, i32, vp]),
    "db_cheb_backward": (C.c_int, [PFFT, vp, vp, i64, i32, i64, vp, i32, vp, i32, vp]),
    "db_cheb_backward_scan": (C.c_int, [PFFT, vp, vp, i64, i32, vp, i32, vp, vp]),
    "db_band_lines": (C.c_int, [vp, vp, i64, i32, vp, i32, vp, i32, i32, vp]),
    "db_mmt_apply": (C.c_int, [vp, i32, i32, vp, vp, i64, i64, vp]),
    "db_mmt_dmma_launches": (C.c_longlong, []),
    "db_ragged_matvec": (C.c_int, [vp, vp, i32, i32, vp, vp, i64, i32, i32, i32, i32, i64, vp]),
    "db_pointwise": (C.c_int, [vp, vp, i64, i32, i32, vp, vp, vp, vp, i32, vp]),
    "db_pointwise_pairs": (C.c_int, [vp, vp, i64, i32, i32, vp, vp, vp]),
    "db_pointwise_launches": (C.c_longlong, [i32]),
    "db_rfft_x_products": (C.c_int, [PFFT, vp, i64, vp, i64, i32, i64, f64, vp, i32, vp, i32, i32, vp]),
    "db_rfft_blocks_per_sm": (C.c_int, [i32, i32, i32, i32]),
    "db_pencil_gather": (C.c_int, [vp, vp, i32, i32, i32, i32, vp, vp, vp, vp, vp, i32, vp]),
    "db_pencil_scatter": (C.c_int, [vp, vp, i32, i32, i32, i32, vp, vp, vp, vp, vp, i32, vp]),
    "db_pencil_matvec": (C.c_int, [i32, i32, i32, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp]),
    "db_pencil_assemble": (C.c_int, [vp, i32, i32, i32, vp, vp, vp, vp, vp]),
    "db_pencil_factor": (C.c_int, [vp, i32, i32, i32, vp, vp, vp, vp, vp, vp, vp, vp]),
    "db_pencil_solve": (C.c_int, [vp, i32, i32, i32, vp, i32, i32, PLIN, vp, vp]),
    "db_batches_move": (C.c_int, [vp, i32, i32, i32, i32, i32, vp, vp]),
    "db_batches_matvec": (C.c_int, [vp, i32, i32, i32, i32, i32, vp]),
    "db_batches_solve": (C.c_int, [vp, i32, i32, i32, i32, i32, C.c_void_p, vp]),
    "db_batches_solve_set_mode": (C.c_int, [i32, i32, i32, i32, i32, i32]),
    "db_batches_assemble": (C.c_int, [vp, i32, i32, i32, vp]),
    "db_batches_factor": (C.c_int, [vp, i32, i32, i32, vp]),
    "db_batches_residual": (C.c_int, [vp, i32, i32, i32, i32, i32, f64, f64, vp, vp]),
    "db_lincomb_apply": (C.c_int, [PLIN, vp, i64, vp]),
    "db_transpose_pack": (C.c_int, [vp, vp, i64, i64, i64, i64, i32, vp]),
    "db_transpose_unpack": (C.c_int, [vp, vp, i64, i64, i64, i64, i32, vp]),
    "db_transpose_pack_rev": (C.c_int, [vp, vp, i64, i64, i64, i64, i32, vp]),
    "db_transpose_unpack_rev": (C.c_int, [vp, vp, i64, i64, i64, i64, i32, vp]),
    "db_banded_combine": (C.c_int, [vp, i32, i32, i32, f64, vp, f64, vp, vp, vp]),
    "db_banded_factor": (C.c_int, [vp, i32, i32, i32, vp, vp, vp, vp]),
    "db_banded_solve": (C.c_int, [vp, i32, i32, i32, i32, i32, vp, vp, C.POINTER(VecComb), vp, vp]),
    "db_banded_matvec": (C.c_int, [vp, i32, i32, i32, vp, vp, vp, vp, vp, vp]),
    "db_dense_combine": (C.c_int, [i32, i32, f64, vp, f64, vp, vp, vp]),
    "db_dense_factor": (C.c_int, [i32, i32, vp, vp, vp, vp]),
    "db_dense_solve": (C.c_int, [vp, i32, i32, i32, vp, vp, C.POINTER(VecComb), vp, vp]),
    "db_dense_matvec": (C.c_int, [vp, i32, i32, vp, vp, vp, vp, vp, vp]),
    "db_csr_matvec": (C.c_int, [vp, i32, i32, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp]),
    "db_index_move": (C.c_int, [vp, i64, vp, vp, i32, vp]),
    "db_index_move_runs": (C.c_int, [vp, i64, i64, vp, vp, i32, vp]),
    "db_pair_lincomb": (C.c_int, [vp, vp, i64, i64, i32, vp, vp, vp, i64, vp]),
    "db_absmax": (C.c_int, [vp, i64, vp, vp]),
    "db_cfl_max": (C.c_int, [C.POINTER(vp), C.POINTER(vp), i32, i64, i64, i64, vp, vp]),
    "db_cfl_max_spherical": (C.c_int, [vp, vp, vp, vp, vp, i64, i64, vp, vp]),
}


class DedalusB200Error(RuntimeError):
    pass


class BoundLib:
    def __init__(self, cdll):
        self._cdll = cdll
        missing = []
        for name, (res, args) in SIGNATURES.items():
            try:
                fn = getattr(cdll, name)
            except AttributeError:
                missing.append(name)
                continue
            fn.restype = res
            fn.argtypes = args
            setattr(self, "_raw_" + name, fn)
        if missing:
            raise DedalusB200Error(f"library is missing C-ABI symbols: {missing}")

    launches = 0      # number of kernel-launching C-ABI calls made through this binding

    def call(self, name, *args):
        self.launches += 1
        rc = getattr(self, "_raw_" + name)(*args)
        if rc != 0:
            msg = self._raw_db_last_error()
            raise DedalusB200Error(f"{name} failed (code {rc}): {msg.decode() if msg else ''}")

    def call_optional(self, name, *args):
        """For entries that may decline a case: True if it ran, False if it returned 2 ("not covered")."""
        rc = getattr(self, "_raw_" + name)(*args)
        if rc == 2:
            return False
        self.launches += 1
        if rc != 0:
            msg = self._raw_db_last_error()
            raise DedalusB200Error(f"{name} failed (code {rc}): {msg.decode() if msg else ''}")
        return True

    def version(self):
        return self._raw_db_version()

    def rfft_regs_launches(self):
        return self._raw_db_rfft_regs_launches()

    def device_arch(self):
        return self._raw_db_device_arch()


def bind(path):
    return BoundLib(C.CDLL(str(path)))


class CudaBackend:
    """Where data lives and which library executes: the current CUDA device, torch's current stream and
    dedalus_b200/libdedalus_b200.so.  There is no other backend in the product and no CPU fallback: every method raises if
    CUDA or the library is missing.  (`_BACKEND` below is the single indirection point; the GPU-less build container's
    tests replace it with their own object defined in tests/emu/emu_lib.py -- the product contains no emulation code.)"""

    _lib = None

    def device(self):
        import torch
        if not torch.cuda.is_available():
            raise DedalusB200Error("dedalus_b200 requires a CUDA device (sm_90a); there is no CPU fallback.")
        return torch.device('cuda', torch.cuda.current_device())

    def stream(self):
        import torch
        return C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def lib(self):
        if CudaBackend._lib is None:
            from . import build as _build
            if not _build.lib_is_current():
                # missing, or built from other sources than the ones in the tree (a stale library would lack entry points or,
                # worse, run old kernels): rebuild it if nvcc is here, else say so -- never continue with it
                try:
                    import fcntl
                    with open(str(LIB_PATH) + ".lock", "w") as lock:       # several ranks may get here at once: one builds, the others wait
                        fcntl.flock(lock, fcntl.LOCK_EX)
                        if not _build.lib_is_current():
                            _build.build(force=not LIB_PATH.exists())
                except Exception as exc:
                    raise DedalusB200Error(
                        f"{LIB_PATH} is missing or was not built from the current sources and could not be rebuilt ({exc}): "
                        "run `python -m dedalus_b200.build` (nvcc, sm_90a).  dedalus_b200 has no CPU fallback.")
            CudaBackend._lib = bind(LIB_PATH)
        return CudaBackend._lib

    def accepts(self, tensor):
        return tensor.is_cuda


_BACKEND = CudaBackend()


def compute_device():
    """torch device for all data: the current CUDA device (required)."""
    return _BACKEND.device()


def current_stream():
    return _BACKEND.stream()


def get_lib():
    """The CUDA library (built in-tree by dedalus_b200/build.py). Fails loudly if it is absent."""
    return _BACKEND.lib()


def device_tensor_ok(tensor):
    """True if `tensor` lives where the kernels can reach it (a CUDA tensor)."""
    return _BACKEND.accepts(tensor)
