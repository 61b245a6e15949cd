"""ctypes binding of libcape_b200.so (include/cape_b200.h).  There is no CPU fallback: if the shared
library is missing the import of any compute entry point fails loudly."""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# CAPE_B200_LIB: another build of the same library (A/B measurements of compile-time variants)
LIB_PATH = os.environ.get("CAPE_B200_LIB") or os.path.join(_HERE, "libcape_b200.so")

MAX_TERMS = 8
EPI_LINEAR, EPI_AFFINE, EPI_SLOPE, EPI_DUALMASK, EPI_TANHGRAD = 0, 1, 2, 3, 4
ACT_NONE, ACT_LEAKY, ACT_RELU, ACT_TANH = 0, 1, 2, 3
RECON_L1, RECON_L2, RECON_HUBER = 0, 1, 2

f32p = C.c_void_p  # device pointers travel as integers


class Term(C.Structure):
    _fields_ = [("src", C.c_void_p), ("op", C.c_int), ("F", C.c_int), ("src_rows", C.c_int),
                ("src_stride", C.c_int), ("w_stride", C.c_int), ("w2_stride", C.c_int), ("w", C.c_void_p), ("w2", C.c_void_p),
                ("wc", C.c_void_p), ("wc2", C.c_void_p), ("wT", C.c_void_p), ("w2T", C.c_void_p),
                ("wT_stride", C.c_int), ("w2T_stride", C.c_int), ("stash", C.c_void_p), ("stash_stride", C.c_int)]


class ConvArgs(C.Structure):
    _fields_ = [("N", C.c_int), ("rows_out", C.c_int), ("ncols", C.c_int), ("nterms", C.c_int),
                ("terms", Term * MAX_TERMS), ("cond", C.c_void_p), ("C", C.c_int), ("epilogue", C.c_int),
                ("act", C.c_int), ("alpha", C.c_float), ("bias", C.c_void_p), ("bias_per_row", C.c_int),
                ("aux", C.c_void_p), ("out", C.c_void_p), ("out2", C.c_void_p), ("plain_only", C.c_int)]


class ApplyTerm(C.Structure):
    _fields_ = [("src", C.c_void_p), ("op", C.c_int), ("src_rows", C.c_int), ("src_stride", C.c_int), ("acc", C.c_int),
                ("scale", C.c_float), ("wc", C.c_void_p), ("wc_stride", C.c_int)]


class ApplyArgs(C.Structure):
    _fields_ = [("N", C.c_int), ("rows_out", C.c_int), ("ncols", C.c_int), ("nterms", C.c_int),
                ("terms", ApplyTerm * MAX_TERMS), ("cond", C.c_void_p), ("C", C.c_int), ("epilogue", C.c_int),
                ("act", C.c_int), ("alpha", C.c_float), ("bias", C.c_void_p), ("bias_per_row", C.c_int),
                ("aux", C.c_void_p), ("out", C.c_void_p), ("out_stride", C.c_int), ("out2", C.c_void_p),
                ("term_stride", C.c_int64)]


class WPrep(C.Structure):
    _fields_ = [("w", C.c_void_p), ("Fin", C.c_int), ("K", C.c_int), ("Fout", C.c_int), ("wt", C.c_void_p),
                ("wk", C.c_void_p)]


class GemmItem(C.Structure):
    _fields_ = [("a", C.c_void_p), ("a_rs", C.c_int64), ("a_cs", C.c_int64), ("b", C.c_void_p), ("b_rs", C.c_int64),
                ("b_cs", C.c_int64), ("c", C.c_void_p), ("c_rs", C.c_int64), ("M", C.c_int), ("N", C.c_int), ("K", C.c_int),
                ("alpha", C.c_float), ("beta", C.c_float)]


class DwArgs(C.Structure):
    _fields_ = [("N", C.c_int), ("rows_out", C.c_int), ("ncols", C.c_int), ("src", C.c_void_p), ("op", C.c_int),
                ("F", C.c_int), ("src_rows", C.c_int), ("src_stride", C.c_int), ("g", C.c_void_p),
                ("dw", C.c_void_p), ("dw_stride", C.c_int), ("accumulate", C.c_int), ("nops", C.c_int),
                ("ops", C.c_int * MAX_TERMS), ("dw_term_stride", C.c_int), ("dw_col_stride", C.c_int)]


# name -> (restype, argtypes); every symbol declared in include/cape_b200.h
SIGNATURES = {
    "cape_last_error": (C.c_char_p, []),
    "cape_abi_version": (C.c_int, []),
    "cape_launch_count": (C.c_int64, []),
    "cape_topology_create": (C.c_int, [C.c_int, C.POINTER(C.c_void_p)]),
    "cape_topology_destroy": (None, [C.c_void_p]),
    "cape_topology_add_operator": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "cape_topology_reserve_workspace": (C.c_int, [C.c_void_p, C.c_int64]),
    "cape_set_tensor_cores": (C.c_int, [C.c_int]),
    "cape_tensor_cores_enabled": (C.c_int, []),
    "cape_gemm_batch": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p]),
    "cape_gemm_item_bytes": (C.c_int, []),
    "cape_gather_rows": (C.c_int, [C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "cape_weight_prep": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p]),
    "cape_set_tuning": (C.c_int, [C.c_int, C.c_int]),
    "cape_cheb_fwd": (C.c_int, [C.c_void_p, C.POINTER(ConvArgs), C.c_void_p]),
    "cape_apply": (C.c_int, [C.c_void_p, C.POINTER(ApplyArgs), C.c_void_p]),
    "cape_cheb_dw": (C.c_int, [C.c_void_p, C.POINTER(DwArgs), C.c_void_p]),
    "cape_colsum": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int), C.c_int,
                              C.c_void_p, C.c_void_p]),
    "cape_gemm": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int64, C.c_int64, C.c_void_p,
                            C.c_int64, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_int, C.c_float, C.c_float,
                            C.c_float, C.c_void_p]),
    "cape_gemm_ex": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int64, C.c_int64, C.c_void_p,
                               C.c_int64, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_int, C.c_float, C.c_float,
                               C.c_float, C.c_int, C.c_float, C.c_void_p, C.c_int64, C.c_void_p]),
    "cape_resample": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int,
                                C.c_int, C.c_void_p, C.c_int, C.c_void_p]),
    "cape_cheb_weight_transpose": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "cape_act_bwd": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_float, C.c_void_p]),
    "cape_axpy": (C.c_int, [C.c_void_p, C.c_void_p, C.c_float, C.c_int64, C.c_void_p]),
    "cape_vae_sample_fwd": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                      C.c_void_p]),
    "cape_vae_sample_bwd": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_void_p]),
    "cape_recon_losses": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_float,
                                    C.c_float, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p,
                                    C.c_void_p]),
    "cape_recon_losses_ex": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                       C.c_float, C.c_float, C.c_float, C.c_int, C.c_void_p, C.c_void_p, C.c_int,
                                       C.c_void_p, C.c_void_p, C.c_void_p]),
    "cape_recon_losses_w": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                      C.c_float, C.c_float, C.c_float, C.c_int, C.c_void_p, C.c_double, C.c_void_p,
                                      C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "cape_bce_logits": (C.c_int, [C.c_void_p, C.c_int64, C.c_float, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p]),
    "cape_sumsq": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]),
    "cape_sgd_clip_update": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_float,
                                       C.c_void_p, C.c_float, C.c_void_p]),
    "cape_adam_clip_update": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_float,
                                        C.c_void_p, C.c_float, C.c_float, C.c_float, C.c_void_p]),
    "cape_gn_relu_fwd": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, C.c_void_p,
                                   C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "cape_gn_relu_bwd": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int,
                                   C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "cape_smpl_create": (C.c_int, [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                   C.c_void_p, C.POINTER(C.c_void_p)]),
    "cape_smpl_destroy": (None, [C.c_void_p]),
    "cape_smpl_workspace_bytes": (C.c_int64, [C.c_void_p, C.c_int]),
    "cape_smpl_pose": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64,
                                 C.c_void_p]),
}

_lib = None


class CapeError(RuntimeError):
    pass


def load():
    """Load the shared library (once) and attach prototypes.  Raises if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise CapeError("libcape_b200.so not built (%s): run `python -c 'import __graft_entry__ as g; g.build()'` "
                        "or `make -C cape_b200/csrc`; there is no CPU fallback" % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if a declared symbol is not exported
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc):
    if rc < 0:
        raise CapeError("libcape_b200: " + load().cape_last_error().decode())
    return rc
