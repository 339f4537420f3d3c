"""ctypes binding of libfcma_b200.so (the C ABI declared in include/fcma_b200.h).

There is no fallback: if the shared library is missing or a compute call is made without an
sm_90 device, an exception is raised — results never silently come from anywhere else.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libfcma_b200.so")

FCMA_OK, FCMA_EINVAL, FCMA_ECUDA, FCMA_ENODEV, FCMA_ENOMEM = 0, -1, -2, -3, -4

PREC = {"bf16": 0, "tf32": 1, "bf16x3": 2, "tf32x3": 3, "f32simt": 4, "fp16x3": 5}
PREC_NAMES = tuple(PREC) + ("fp32",)      # "fp32" = auto-select fp16x3 / tf32x3 (engine.resolve_precision)
FLAG_MASK_SELF = 1
FLAG_FISHER_IN_PASS2 = 2
FLAG_F16_INTERMEDIATE = 4   # fp16 internal Fisher-z block (default only in the bf16 / tf32 operand modes)
# alternate code paths with the same results (tests compare them against the defaults)
FLAG_STRIDED_BLOCK = 8      # strided [nb][E][ld] correlation block instead of the tiled one
FLAG_SYM_TRANSPOSED = 16    # symmetric pipeline: transposed copy + row pass instead of the column-direction pass
FLAG_COLS_V2 = 64           # column-direction pass, version 2 (thread-per-row normalisation + ldmatrix); not the default
FLAG_COLS_PAD32 = 128       # E <= 16: the padded 32-epoch column kernel instead of the 16-epoch one
FLAG_COLS_WIDE = 256        # 32 < E <= 64: column pass over the block (k_norm_syrk_cols64) instead of the transposed copy
FLAG_COLS_TMA = 32          # column-direction pass fed by TMA bricks + mbarrier ring instead of cp.async (E % 4 == 0)

c_void_p, c_int, c_long, c_size_t, c_float = (ctypes.c_void_p, ctypes.c_int, ctypes.c_long,
                                               ctypes.c_size_t, ctypes.c_float)
c_int_p = ctypes.POINTER(ctypes.c_int)
c_float_pp = ctypes.POINTER(ctypes.POINTER(ctypes.c_float))

# name -> (restype, argtypes); mirrors include/fcma_b200.h one to one
SIGNATURES = {
    "fcma_version": (c_int, []),
    "fcma_last_error": (ctypes.c_char_p, []),
    "fcma_device_count": (c_int, []),
    "fcma_operand_kp": (c_int, [c_int, c_int]),
    "fcma_operand_planes": (c_int, [c_int]),
    "fcma_operand_bytes": (c_size_t, [c_int, c_int, c_int, c_long]),
    "fcma_pack_operand": (c_int, [c_void_p, c_int, c_int, c_long, c_long, c_int_p, c_int, c_int,
                                  c_void_p, c_size_t, c_void_p]),
    "fcma_pack_operand_range": (c_int, [c_void_p, c_int, c_int, c_long, c_long, c_int_p, c_int, c_int, c_long, c_long,
                                        c_void_p, c_size_t, c_void_p]),
    "fcma_epoch_normalize": (c_int, [c_void_p, c_int, c_int, c_long, c_long, c_int_p, c_void_p]),
    "fcma_corr_block": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_long, c_long, c_long,
                                c_long, c_void_p, c_long, c_long, c_int, c_void_p]),
    "fcma_corr_block_f32": (c_int, [c_void_p, c_long, c_void_p, c_long, c_int, c_int, c_long,
                                    c_long, c_long, c_long, c_void_p, c_long, c_long, c_void_p]),
    "fcma_within_subject_norm": (c_int, [c_void_p, c_long, c_int, c_long, c_int, c_void_p]),
    "fcma_kernel_matrices": (c_int, [c_void_p, c_long, c_int, c_long, c_long, c_long, c_float,
                                     c_void_p, c_int, c_void_p]),
    "fcma_norm_kernel_matrices": (c_int, [c_void_p, c_long, c_int, c_long, c_long, c_long, c_int,
                                          c_int, c_long, c_float, c_void_p, c_int, c_void_p]),
    "fcma_work_bytes_per_row": (c_size_t, [c_int, c_long]),
    "fcma_voxel_kernels": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_long, c_long, c_long,
                                   c_long, c_int, c_int, c_void_p, c_size_t, c_void_p, c_void_p]),
    "fcma_voxel_kernels_sym": (c_int, [c_void_p, c_int, c_int, c_int, c_long, c_long, c_long, c_int, c_int,
                                       c_void_p, c_size_t, c_void_p, c_void_p]),
    "fcma_voxel_kernels_sym_grouped": (c_int, [c_void_p, c_int_p, c_int, c_void_p, c_size_t, c_int, c_int, c_int, c_long,
                                               c_long, c_long, c_int, c_int, c_int, c_int_p, c_int_p,
                                               ctypes.POINTER(c_void_p), c_void_p, c_size_t, c_void_p, c_void_p]),
    "fcma_sym_uses_column_pass": (c_int, [c_int, c_int, c_int, c_int]),
    "fcma_sym_rows_per_pass": (c_long, [c_int, c_int, c_int, c_int, c_long, c_long, c_size_t]),
    "fcma_classifier_kernel": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_long, c_long,
                                       c_long, c_long, c_int, c_int, c_void_p, c_size_t, c_void_p,
                                       c_void_p]),
    "fcma_classifier_kernel_sym": (c_int, [c_void_p, c_int, c_int, c_int, c_long, c_int, c_int, c_void_p, c_size_t, c_void_p,
                                           c_void_p]),
    "fcma_shrink_kernels": (c_int, [c_void_p, c_long, c_int, c_void_p, c_void_p]),
    "fcma_subset_kernels": (c_int, [c_void_p, c_long, c_int, c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p]),
    "fcma_subset_kernels_f64": (c_int, [c_void_p, c_long, c_int, c_void_p, c_int, c_void_p, c_void_p]),
    "fcma_svm_cv_precomputed": (c_int, [c_void_p, c_long, c_int, c_int, c_void_p, ctypes.c_double,
                                        ctypes.c_double, c_int, c_void_p, c_void_p, c_void_p]),
    "fcma_svm_cv_solve": (c_int, [c_void_p, c_long, c_int, c_int, c_void_p, ctypes.c_double, ctypes.c_double, c_int, c_int,
                                  c_void_p, c_void_p, c_void_p, c_void_p]),
    "fcma_svm_cv_solve_f64": (c_int, [c_void_p, c_void_p, c_long, c_int, c_int, c_void_p, ctypes.c_double, ctypes.c_double,
                                      c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "fcma_svm_cv_solve_wide": (c_int, [c_void_p, c_long, c_int, c_int, c_void_p, ctypes.c_double, ctypes.c_double, c_int,
                                       c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "fcma_svm_cv_solve_f64_wide": (c_int, [c_void_p, c_void_p, c_long, c_int, c_int, c_void_p, ctypes.c_double,
                                           ctypes.c_double, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "fcma_searchlight_kernels": (c_int, [c_void_p, c_long, c_long, c_long, c_int, c_void_p, c_int, c_void_p, c_void_p,
                                         c_long, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "fcma_searchlight_kernels_wide": (c_int, [c_void_p, c_long, c_long, c_long, c_int, c_void_p, c_int, c_void_p,
                                              c_void_p, c_long, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "fcma_voxel_feature_kernels": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_long, c_long, c_long, c_long, c_int,
                                           c_int, ctypes.c_double, c_void_p, c_size_t, c_void_p, c_void_p, c_void_p]),
    "fcma_voxel_feature_kernels_wide": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_long, c_long, c_long, c_long,
                                                c_int, c_int, ctypes.c_double, c_void_p, c_size_t, c_void_p, c_void_p,
                                                c_void_p]),
    "fcma_voxel_feature_gram_wide": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_long, c_long, c_long, c_long,
                                             c_int, c_void_p, c_size_t, c_void_p, c_void_p, c_void_p, c_void_p]),
    "fcma_searchlight_gram_wide": (c_int, [c_void_p, c_long, c_long, c_long, c_int, c_void_p, c_int, c_void_p, c_void_p,
                                           c_long, c_void_p, c_void_p, c_void_p, c_void_p]),
    "fcma_fold_gammas": (c_int, [c_void_p, c_long, c_int, c_int, c_void_p, c_void_p, c_long, c_void_p, c_void_p,
                                 c_void_p]),
    "fcma_rbf_fold_kernels": (c_int, [c_void_p, c_void_p, c_long, c_int, c_void_p, c_int, c_int, c_void_p, c_void_p,
                                      c_void_p]),
    "fcma_gemm_nt": (c_int, [c_void_p, c_void_p, c_void_p, c_long, c_long, c_long, c_long, c_long,
                             c_long, c_void_p]),
    "fcma_row_normalize": (c_int, [c_void_p, c_long, c_long, c_long, c_int, c_void_p]),
    "fcma_host_voxel_kernels": (c_int, [c_float_pp, c_float_pp, c_int_p, c_int, c_long, c_long,
                                        c_long, c_long, c_int, c_int, c_int, c_int, c_int,
                                        c_void_p]),
    "fcma_host_voxel_kernels_sym": (c_int, [c_float_pp, c_int_p, c_int, c_long, c_int, c_int, c_int, c_int, c_int, c_long,
                                            c_void_p]),
    "fcma_ipc_get_handle": (c_int, [c_void_p, c_void_p, ctypes.POINTER(c_size_t)]),
    "fcma_ipc_open_handle": (c_int, [c_void_p, ctypes.POINTER(c_void_p)]),
    "fcma_ipc_close_handle": (c_int, [c_void_p]),
    "fcma_peer_copy_async": (c_int, [c_void_p, c_void_p, c_size_t, c_void_p]),
    "fcma_host_within_subject_norm": (c_int, [c_void_p, c_long, c_int, c_long, c_int, c_int]),
    "fcma_launch_count": (c_long, []),
    "fcma_timing_enable": (None, [c_int]),
    "fcma_timing_read": (c_long, [ctypes.POINTER(ctypes.c_double), ctypes.POINTER(ctypes.c_double)]),
    "fcma_timing_read3": (c_long, [ctypes.POINTER(ctypes.c_double), ctypes.POINTER(ctypes.c_double),
                                   ctypes.POINTER(ctypes.c_double)]),
}

_lib = None


def use_diag_build():
    """tools/ only: bind the diagnostic build (libfcma_b200_diag.so, compiled with -DFCMA_DIAG, the only build that
    reads the FCMA_* A/B and debug environment knobs).  Must be called before the first load()."""
    global LIB_PATH
    if _lib is not None:
        raise RuntimeError("use_diag_build() must be called before the library is loaded")
    LIB_PATH = os.path.join(_HERE, "libfcma_b200_diag.so")


class FcmaLibraryMissing(RuntimeError):
    pass


def load():
    """Load libfcma_b200.so; raises FcmaLibraryMissing (never falls back) if it is not built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise FcmaLibraryMissing(
            "%s not found: build it with `python -m brainiak_b200.build` "
            "(nvcc, sm_90a). brainiak_b200 has no CPU fallback." % LIB_PATH)
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)      # AttributeError here = header/library mismatch
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def last_error():
    return load().fcma_last_error().decode("utf-8", "replace")


def check(rc):
    """Map a C status to the exception the reference's native modules would raise
    (ValueError from Cython typed memoryviews, RuntimeError from fcma_extension.cc:47)."""
    if rc == FCMA_OK:
        return
    msg = last_error()
    if rc == FCMA_EINVAL:
        raise ValueError(msg)
    if rc == FCMA_ENOMEM:
        raise MemoryError(msg)
    raise RuntimeError(msg)


def device_count():
    return load().fcma_device_count()


def require_device():
    if device_count() == 0:
        raise RuntimeError("brainiak_b200 needs an sm_90 (H100) CUDA device; none is visible "
                           "and there is no CPU fallback")
