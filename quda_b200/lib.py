"""ctypes binding of libquda_b200.so (C ABI: include/b200_dslash.h).

The structures mirror the header field by field.  There is NO CPU fallback: if the shared library is missing,
or no CUDA device is present, every entry point raises."""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# B200_LIB lets the tuning tools load an alternative build of the same library (e.g. another occupancy target)
LIB_PATH = os.environ.get("B200_LIB") or os.path.join(_HERE, "libquda_b200.so")
ABI_VERSION = 3

DOUBLE, SINGLE, HALF = 8, 4, 2
OP_WILSON, OP_CLOVER, OP_CLOVER_PC, OP_TWISTED_MASS, OP_TWISTED_MASS_PC = 0, 1, 2, 3, 4
KERNEL_AUTO, KERNEL_INTERIOR, KERNEL_EXTERIOR, KERNEL_INTERIOR_TILES, KERNEL_BOUNDARY_TILES = 0, 1, 2, 3, 4
KERNEL_INTERIOR_SITES, KERNEL_BOUNDARY_SITES = 5, 6


class B200Error(RuntimeError):
    pass


class Spinor(C.Structure):
    _fields_ = [("v", C.c_void_p), ("norm", C.c_void_p), ("parity_stride_bytes", C.c_size_t),
                ("volume_cb", C.c_int), ("n_parity", C.c_int)]


class Gauge(C.Structure):
    _fields_ = [("gauge", C.c_void_p), ("parity_stride_bytes", C.c_size_t), ("stride", C.c_int),
                ("reconstruct", C.c_int), ("anisotropy", C.c_double), ("link_max", C.c_double),
                ("t_boundary", C.c_int), ("first_time_slice", C.c_int), ("last_time_slice", C.c_int)]


class Clover(C.Structure):
    _fields_ = [("clover", C.c_void_p), ("parity_stride_bytes", C.c_size_t), ("compressed", C.c_int),
                ("dynamic_inverse", C.c_int), ("diagonal", C.c_double), ("max_element", C.c_double)]


class Halo(C.Structure):
    _fields_ = [("comm_dim", C.c_int * 4), ("ghost", (C.c_void_p * 2) * 4), ("ghost_norm", (C.c_void_p * 2) * 4),
                ("wait_flag", (C.c_void_p * 2) * 4), ("seq", C.c_uint), ("timeout_flag", C.c_void_p),
                ("src_stride", C.c_size_t * 4)]


class DslashArgs(C.Structure):
    _fields_ = [("abi_version", C.c_int), ("op", C.c_int), ("kernel", C.c_int), ("precision", C.c_int),
                ("X", C.c_int * 4), ("parity", C.c_int), ("dagger", C.c_int), ("a", C.c_double),
                ("b", C.c_double), ("asymmetric", C.c_int),
                ("out", Spinor), ("in_", Spinor), ("x", Spinor), ("U", Gauge), ("A", Clover), ("halo", Halo),
                ("tile", C.c_int * 4), ("stream", C.c_void_p)]


class PackArgs(C.Structure):
    _fields_ = [("abi_version", C.c_int), ("precision", C.c_int), ("X", C.c_int * 4), ("parity", C.c_int),
                ("dagger", C.c_int), ("in_", Spinor), ("comm_dim", C.c_int * 4), ("dst", (C.c_void_p * 2) * 4),
                ("dst_norm", (C.c_void_p * 2) * 4), ("signal", (C.c_void_p * 2) * 4), ("block_counter", C.c_void_p),
                ("seq", C.c_uint), ("stream", C.c_void_p)]


class Comm(C.Structure):
    _fields_ = [("comm_dim", C.c_int * 4), ("send_dst", ((C.c_void_p * 2) * 4) * 2),
                ("send_signal", ((C.c_void_p * 2) * 4) * 2), ("recv", ((C.c_void_p * 2) * 4) * 2),
                ("recv_flag", ((C.c_void_p * 2) * 4) * 2), ("block_counter", C.c_void_p),
                ("timeout_flag", C.c_void_p), ("seq", C.c_uint), ("pack_stream", C.c_void_p),
                ("allreduce_sum", C.c_void_p), ("user", C.c_void_p),
                ("rank", C.c_int), ("n_ranks", C.c_int), ("reduce_peer", C.c_void_p * 16), ("reduce_seq", C.c_uint)]


MAX_RANKS, REDUCE_MAILBOX_BYTES = 16, 2 * 16 * 64


ALLREDUCE_FN = C.CFUNCTYPE(None, C.POINTER(C.c_double), C.c_int, C.c_void_p)


class SolverParam(C.Structure):
    _fields_ = [("tol", C.c_double), ("maxiter", C.c_int), ("delta", C.c_double), ("iter", C.c_int),
                ("reliable_updates", C.c_int), ("true_res", C.c_double), ("secs", C.c_double), ("gflops", C.c_double),
                ("host_syncs", C.c_int)]


MAX_SHIFTS = 32


class MultiShiftParam(C.Structure):
    _fields_ = [("n_shift", C.c_int), ("offset", C.c_double * MAX_SHIFTS), ("tol_offset", C.c_double * MAX_SHIFTS),
                ("maxiter", C.c_int), ("delta", C.c_double), ("iter", C.c_int), ("iter_offset", C.c_int * MAX_SHIFTS),
                ("refine_iter", C.c_int * MAX_SHIFTS), ("iter_res_offset", C.c_double * MAX_SHIFTS),
                ("true_res_offset", C.c_double * MAX_SHIFTS), ("reliable_updates", C.c_int), ("secs", C.c_double),
                ("gflops", C.c_double), ("host_syncs", C.c_int)]


MAX_MULTI_RHS = 16
DIRAC_WILSON, DIRAC_WILSONPC, DIRAC_CLOVER, DIRAC_CLOVERPC, DIRAC_TWISTED_MASS, DIRAC_TWISTED_MASSPC = 0, 1, 2, 3, 4, 5
APPLY_M, APPLY_MDAG, APPLY_MDAGM, APPLY_DSLASH, APPLY_DSLASH_XPAY = 0, 1, 2, 3, 4


def declare(lib, prefix="b200"):
    """Attach argtypes/restypes for the entry points shared by the CUDA library and the test-only host twin."""
    f = getattr(lib, prefix + "_dslash_apply")
    f.argtypes, f.restype = [C.POINTER(DslashArgs)], C.c_int
    f = getattr(lib, prefix + "_dslash_apply_multi")
    f.argtypes = [C.POINTER(DslashArgs), C.c_int, C.POINTER(Spinor), C.POINTER(Spinor), C.POINTER(Spinor)]
    f.restype = C.c_int
    f = getattr(lib, prefix + "_clover_apply")
    f.argtypes = [C.POINTER(Spinor), C.POINTER(Spinor), C.POINTER(Clover), C.c_int, C.c_int, C.c_int, C.c_void_p]
    f.restype = C.c_int
    f = getattr(lib, prefix + "_twist_gamma5")
    f.argtypes = [C.POINTER(Spinor), C.POINTER(Spinor), C.c_int, C.c_double, C.c_double, C.c_int, C.c_int, C.c_void_p]
    f.restype = C.c_int
    f = getattr(lib, prefix + "_pack_ghost")
    f.argtypes, f.restype = [C.POINTER(PackArgs)], C.c_int
    f = getattr(lib, prefix + "_pack_ghost_multi")
    f.argtypes, f.restype = [C.POINTER(PackArgs), C.c_int, C.POINTER(Spinor), C.POINTER(C.c_size_t)], C.c_int
    f = getattr(lib, prefix + "_dslash_apply_fused")
    f.argtypes, f.restype = [C.POINTER(DslashArgs), C.POINTER(PackArgs)], C.c_int
    f = getattr(lib, prefix + "_last_error")
    f.argtypes, f.restype = [], C.c_char_p
    return lib


def declare_clover(lib, prefix="b200"):
    """Attach argtypes/restypes for the clover construction, shared by the CUDA library and its test-only twin."""
    f = getattr(lib, prefix + "_compute_clover")
    f.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_int), C.POINTER(C.c_int), C.c_int, C.c_double, C.c_void_p]
    f.restype = C.c_int
    f = getattr(lib, prefix + "_clover_invert_packed")
    f.argtypes = [C.c_void_p, C.POINTER(C.c_double), C.c_void_p, C.POINTER(C.c_int), C.c_int, C.c_void_p]
    f.restype = C.c_int
    f = getattr(lib, prefix + "_last_error")
    f.argtypes, f.restype = [], C.c_char_p
    return lib


def declare_clover_force(lib, prefix="b200"):
    """Attach argtypes/restypes for the kernel-level clover force, shared by the CUDA library and its test-only twin."""
    f = getattr(lib, prefix + "_clover_force_accumulate")
    f.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.c_void_p, C.POINTER(C.c_int), C.c_int, C.c_int, C.POINTER(C.c_void_p),
                  C.POINTER(C.c_void_p), C.POINTER(C.c_double), C.POINTER(C.c_double), C.c_double, C.c_int, C.c_void_p]
    f.restype = C.c_int
    f = getattr(lib, prefix + "_last_error")
    f.argtypes, f.restype = [], C.c_char_p
    return lib


def declare_gauge(lib, prefix="b200"):
    """Attach argtypes/restypes for the gauge force, link update, momentum action and plaquette, shared by the CUDA library and
    their test-only twin."""
    P4 = C.POINTER(C.c_void_p)
    f = getattr(lib, prefix + "_gauge_force")
    f.argtypes = [C.c_void_p, P4, C.POINTER(C.c_int), C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_double),
                  C.c_int, C.c_int, C.c_double, C.c_void_p]
    f.restype = C.c_int
    f = getattr(lib, prefix + "_update_gauge")
    f.argtypes = [P4, P4, C.c_void_p, C.POINTER(C.c_int), C.c_int, C.c_double, C.c_int, C.c_int, C.c_void_p]
    f.restype = C.c_int
    f = getattr(lib, prefix + "_mom_action")
    f.argtypes = [C.POINTER(C.c_double), C.c_void_p, C.POINTER(C.c_int), C.c_int, C.c_void_p]
    f.restype = C.c_int
    f = getattr(lib, prefix + "_plaquette")
    f.argtypes = [C.POINTER(C.c_double), P4, C.POINTER(C.c_int), C.c_int, C.c_void_p]
    f.restype = C.c_int
    f = getattr(lib, prefix + "_last_error")
    f.argtypes, f.restype = [], C.c_char_p
    return lib


def declare_flow(lib, prefix="b200"):
    """Attach argtypes/restypes for the gradient flow and the gauge observables, shared by the CUDA library and their
    test-only twin."""
    P4 = C.POINTER(C.c_void_p)
    f = getattr(lib, prefix + "_gauge_flow")
    f.argtypes = [P4, P4, C.POINTER(C.c_int), C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_double), C.c_int,
                  C.c_int, C.c_double, C.c_int, C.c_void_p]
    f.restype = C.c_int
    f = getattr(lib, prefix + "_gauge_observables")
    f.argtypes = [C.POINTER(C.c_double), C.POINTER(C.c_double), C.c_void_p, P4, C.POINTER(C.c_int), C.c_int, C.c_void_p]
    f.restype = C.c_int
    f = getattr(lib, prefix + "_last_error")
    f.argtypes, f.restype = [], C.c_char_p
    return lib


def declare_smear(lib, prefix="b200"):
    """Attach argtypes/restypes for gauge smearing, shared by the CUDA library and its test-only twin."""
    P4 = C.POINTER(C.c_void_p)
    f = getattr(lib, prefix + "_gauge_smear")
    f.argtypes = [P4, P4, C.POINTER(C.c_int), C.c_int, C.c_int, C.POINTER(C.c_double), C.c_int, C.c_int, C.c_void_p]
    f.restype = C.c_int
    f = getattr(lib, prefix + "_last_error")
    f.argtypes, f.restype = [], C.c_char_p
    return lib


SMEAR_APE, SMEAR_STOUT, SMEAR_OVRIMP_STOUT, SMEAR_HYP = 0, 1, 2, 3  # B200_SMEAR_*
GAUGE_MAX_PATHS, GAUGE_MAX_LENGTH = 64, 12  # B200_GAUGE_MAX_PATHS, B200_GAUGE_MAX_LENGTH

_lib = None


def load():
    """Load libquda_b200.so (raises if it has not been built: run __graft_entry__.build() / make -C quda_b200/csrc)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise B200Error(f"{LIB_PATH} not built -- the engine has no fallback path; run __graft_entry__.build()")
        lib = C.CDLL(LIB_PATH)
        declare(lib)
        declare_clover(lib)
        declare_clover_force(lib)
        declare_gauge(lib)
        declare_flow(lib)
        declare_smear(lib)
        lib.b200_abi_version.restype = C.c_int
        lib.b200_launch_count.restype = C.c_long
        lib.b200_ghost_face_bytes.argtypes = [C.c_int, C.POINTER(C.c_int), C.c_int]
        lib.b200_ghost_face_bytes.restype = C.c_size_t
        lib.b200_copy_spinor.argtypes = [C.POINTER(Spinor), C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p]
        lib.b200_copy_spinor.restype = C.c_int
        lib.b200_copy_gauge.argtypes = [C.POINTER(Gauge), C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_void_p),
                                        C.POINTER(C.c_void_p), C.c_int, C.c_void_p]
        lib.b200_copy_gauge.restype = C.c_int
        lib.b200_copy_clover.argtypes = [C.POINTER(Clover), C.c_int, C.POINTER(C.c_int), C.c_void_p, C.c_int, C.c_void_p]
        lib.b200_copy_clover.restype = C.c_int
        lib.b200_comm_alloc.argtypes, lib.b200_comm_alloc.restype = [C.POINTER(C.c_void_p), C.c_size_t], C.c_int
        lib.b200_comm_free.argtypes, lib.b200_comm_free.restype = [C.c_void_p], C.c_int
        lib.b200_ipc_get_handle.argtypes, lib.b200_ipc_get_handle.restype = [C.c_void_p, C.c_char_p], C.c_int
        lib.b200_ipc_open_handle.argtypes = [C.c_char_p, C.POINTER(C.c_void_p)]
        lib.b200_ipc_open_handle.restype = C.c_int
        lib.b200_ipc_close_handle.argtypes, lib.b200_ipc_close_handle.restype = [C.c_void_p], C.c_int
        lib.b200_comm_copy.argtypes, lib.b200_comm_copy.restype = [C.c_void_p, C.c_void_p, C.c_size_t], C.c_int
        lib.b200_dirac_create.argtypes = [C.POINTER(C.c_void_p), C.c_int, C.c_int, C.POINTER(C.c_int), C.POINTER(Gauge),
                                          C.POINTER(Clover), C.POINTER(Clover), C.c_double, C.c_int, C.POINTER(Comm),
                                          C.c_void_p]
        lib.b200_dirac_create.restype = C.c_int
        lib.b200_dirac_destroy.argtypes, lib.b200_dirac_destroy.restype = [C.c_void_p], C.c_int
        lib.b200_dirac_set_twist.argtypes, lib.b200_dirac_set_twist.restype = [C.c_void_p, C.c_double], C.c_int
        lib.b200_dirac_apply.argtypes = [C.c_void_p, C.c_int, C.POINTER(Spinor), C.POINTER(Spinor), C.c_int,
                                         C.POINTER(Spinor), C.c_double, C.c_int]
        lib.b200_dirac_apply.restype = C.c_int
        lib.b200_dirac_prepare.argtypes = [C.c_void_p, C.POINTER(Spinor), C.POINTER(Spinor), C.POINTER(C.c_int),
                                           C.POINTER(C.c_int)]
        lib.b200_dirac_prepare.restype = C.c_int
        lib.b200_dirac_reconstruct.argtypes = [C.c_void_p, C.POINTER(Spinor), C.POINTER(Spinor)]
        lib.b200_dirac_reconstruct.restype = C.c_int
        lib.b200_invert_cg.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(Spinor), C.POINTER(Spinor), C.POINTER(SolverParam)]
        lib.b200_invert_cg.restype = C.c_int
        lib.b200_invert_bicgstab.argtypes = lib.b200_invert_cg.argtypes
        lib.b200_invert_bicgstab.restype = C.c_int
        lib.b200_invert_multishift_cg.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(Spinor), C.POINTER(Spinor),
                                                  C.POINTER(MultiShiftParam)]
        lib.b200_invert_multishift_cg.restype = C.c_int
        lib.b200_clover_force.argtypes = [C.c_void_p, C.c_double, C.POINTER(Spinor), C.POINTER(C.c_double), C.c_double,
                                          C.c_double, C.c_int, C.c_double, C.POINTER(C.c_void_p), C.c_void_p, C.c_void_p]
        lib.b200_clover_force.restype = C.c_int
        lib.b200_comm_check.argtypes, lib.b200_comm_check.restype = [C.POINTER(Comm), C.c_void_p], C.c_int
        if lib.b200_abi_version() != ABI_VERSION:
            raise B200Error("libquda_b200.so ABI version mismatch")
        _lib = lib
    return _lib


def check(rc, lib=None, prefix="b200"):
    if rc != 0:
        lib = lib or load()
        msg = getattr(lib, prefix + "_last_error")().decode()
        raise B200Error(f"{prefix} error {rc}: {msg}")


EXPORTED_SYMBOLS = ["b200_dslash_apply", "b200_dslash_apply_fused", "b200_dslash_apply_multi", "b200_clover_apply", "b200_twist_gamma5", "b200_pack_ghost", "b200_pack_ghost_multi", "b200_ghost_face_bytes",
                    "b200_copy_spinor", "b200_copy_gauge", "b200_copy_clover", "b200_compute_clover", "b200_clover_invert_packed",
                    "b200_clover_force_accumulate", "b200_clover_force", "b200_gauge_force", "b200_update_gauge",
                    "b200_mom_action", "b200_plaquette", "b200_gauge_flow", "b200_gauge_observables", "b200_gauge_smear",
                    "b200_comm_alloc", "b200_comm_free", "b200_ipc_get_handle", "b200_ipc_open_handle",
                    "b200_ipc_close_handle", "b200_comm_copy",
                    "b200_dirac_create", "b200_dirac_set_twist", "b200_dirac_destroy", "b200_dirac_apply", "b200_dirac_prepare",
                    "b200_dirac_reconstruct", "b200_invert_cg", "b200_invert_bicgstab", "b200_invert_multishift_cg",
                    "b200_comm_check",
                    "b200_last_error", "b200_abi_version", "b200_launch_count", "b200_reset_launch_count"]
