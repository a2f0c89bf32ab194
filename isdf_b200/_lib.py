"""ctypes binding of the C ABI declared in include/isdf_b200.h.

The shared library is built in-tree by `__graft_entry__.build()` (nvcc, sm_90a) as
isdf_b200/lib/libisdf_b200.so.  There is NO fallback: if the library is missing or a
symbol is absent, importing/using the product path raises.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libisdf_b200.so")

PREC_FP32, PREC_BF16X3, PREC_BF16, PREC_BF16X3G = 0, 1, 2, 3
PRECISIONS = {"fp32": PREC_FP32, "bf16x3": PREC_BF16X3, "bf16": PREC_BF16, "bf16x3g": PREC_BF16X3G}


class ModelCfg(C.Structure):
    _fields_ = [("n_freqs", C.c_int32), ("hidden", C.c_int32), ("block", C.c_int32),
                ("has_transform", C.c_int32), ("scale_input", C.c_float), ("scale_output", C.c_float),
                ("transform", C.c_float * 12), ("precision", C.c_int32), ("max_points", C.c_int32)]


class LossCfg(C.Structure):
    _fields_ = [("trunc_weight", C.c_float), ("trunc_distance", C.c_float), ("eik_weight", C.c_float),
                ("eik_apply_dist", C.c_float), ("grad_weight", C.c_float), ("orien_loss", C.c_int32),
                ("loss_type", C.c_int32), ("noise_std", C.c_float), ("inv_count", C.c_float),
                ("inv_count_dev", C.c_void_p), ("bounds_dev", C.c_void_p), ("grad_vec_dev", C.c_void_p)]


class Camera(C.Structure):
    _fields_ = [("fx", C.c_float), ("fy", C.c_float), ("cx", C.c_float), ("cy", C.c_float),
                ("H", C.c_int32), ("W", C.c_int32)]


P = C.c_void_p
I64 = C.c_int64
I32 = C.c_int32
F = C.c_float
D = C.c_double

# name -> (restype, argtypes); kept in sync with include/isdf_b200.h (tests/test_abi.py checks it)
SIGNATURES = {
    "isdfb_create": (C.c_int, [C.POINTER(ModelCfg), C.c_int, C.POINTER(P)]),
    "isdfb_destroy": (C.c_int, [P]),
    "isdfb_last_error": (C.c_char_p, [P]),
    "isdfb_param_count": (I64, [P]),
    "isdfb_embedding_size": (I32, [P]),
    "isdfb_launch_count": (I64, [P]),
    "isdfb_pack_weights": (C.c_int, [P, P, P]),
    "isdfb_gather_rays": (C.c_int, [P, P, P, P, I32, P, P, P, I64, C.POINTER(Camera), P, P, P, P]),
    "isdfb_sample_rays": (C.c_int, [P, P, P, P, P, P, P, P, P, P, P, P, P, I64, I32, I32, C.POINTER(Camera), F, F,
                                    P, P, P, P, P]),
    "isdfb_sample_fused": (C.c_int, [P, P, P, P, P, I32, I32, I32, I32, I32, C.POINTER(Camera), F, F, P, C.c_uint64,
                                     P, P, P, P, P, P, P, P, P, P, P, P, P]),
    "isdfb_ingest_normals": (C.c_int, [P, P, C.POINTER(Camera), P, P]),
    "isdfb_pe_encode": (C.c_int, [P, P, I64, P, P]),
    "isdfb_mlp_forward": (C.c_int, [P, P, P, F, I64, P, P]),
    "isdfb_mlp_forward_grad": (C.c_int, [P, P, P, F, I64, P, P, P]),
    "isdfb_mlp_forward_grid": (C.c_int, [P, P, I32, C.POINTER(F), C.POINTER(F), P, P]),
    "isdfb_bounds_pc": (C.c_int, [P, P, P, P, P, I64, I32, P, P, P]),
    "isdfb_train_fwd_bwd": (C.c_int, [P, P, P, P, P, P, P, P, P, I64, I32, C.POINTER(LossCfg), P, P, P, P, P]),
    "isdfb_zero_grad": (C.c_int, [P, P]),
    "isdfb_set_grad_exchange": (C.c_int, [P, P, P, P, P, I64]),
    "isdfb_select_grad_buffer": (C.c_int, [P, I32]),
    "isdfb_zero_grad_buffer": (C.c_int, [P, I32, P]),
    "isdfb_export_grads": (C.c_int, [P, P, P]),
    "isdfb_frame_bins": (C.c_int, [P, P, P, P, P, P, I64, I32, I32, I32, I32, I32, P, P, P]),
    "isdfb_step_finish": (C.c_int, [P, P, P, P, P, P, I64, I32, I32, I32, I32, I32, P, P, P, P, P, P, P, P]),
    "isdfb_select_window": (C.c_int, [P, P, I32, I32, C.c_uint64, P, P]),
    "isdfb_adamw": (C.c_int, [P, P, P, P, I64, D, D, D, D, D, F, P]),
    "isdfb_adamw_graph": (C.c_int, [P, P, P, P, D, D, D, D, D, F, P]),
    "isdfb_adamw_set_step": (C.c_int, [P, I64, P]),
    "isdfb_grad_buffer": (C.c_int, [P, C.POINTER(P), C.POINTER(I64)]),
    "isdfb_mesh_count": (C.c_int, [P, P, I32, C.POINTER(I64), C.POINTER(I64), P]),
    "isdfb_mesh_emit": (C.c_int, [P, P, I32, C.POINTER(F), C.POINTER(F), P, I64, P, I64, P]),
    "isdfb_mesh_cloud": (C.c_int, [P, P, P, I32, I32, I32, I32, I32, F, F, F, F, P, P, P]),
    "isdfb_mesh_crop_count": (C.c_int, [P, P, I64, F, P, I64, P, I64, C.POINTER(I64), C.POINTER(I64), P]),
    "isdfb_mesh_crop_emit": (C.c_int, [P, P, I64, P, I64, P, I64, P, I64, P]),
    "isdfb_gt_sdf_sample": (C.c_int, [P, P, I32, I32, I32, C.POINTER(C.c_double), C.POINTER(C.c_double), P, P, I64,
                                      C.c_double, P, P, P]),
    "isdfb_sdf_error_stats": (C.c_int, [P, P, P, P, P, I64, P, P]),
    "isdfb_points_visible": (C.c_int, [P, P, I64, P, P, I32, I32, I32, F, F, F, F, F, P, P]),
    "isdfb_gt_sdf_grad": (C.c_int, [P, P, I32, I32, I32, C.POINTER(C.c_double), C.POINTER(C.c_double), P, P, I64,
                                    C.c_double, P, P, P]),
    "isdfb_sdf_split_stats": (C.c_int, [P, P, P, I64, I64, P, P]),
    "isdfb_grad_cosdist": (C.c_int, [P, P, P, P, I64, C.c_double, P, P]),
    "isdfb_chomp_costs": (C.c_int, [P, P, P, P, I64, C.POINTER(C.c_double), I32, P, P]),
    "isdfb_voxelize_count": (C.c_int, [P, P, I64, P, I32, I64, D, C.POINTER(D), C.POINTER(I64), C.POINTER(I64), P]),
    "isdfb_voxelize_emit": (C.c_int, [P, P, I64, P, I32, I64, D, C.POINTER(D), C.POINTER(I64), C.POINTER(I64), P, P]),
    "isdfb_fill_holes": (C.c_int, [P, P, I32, I32, I32, P]),
    "isdfb_occupancy_sdf": (C.c_int, [P, P, I32, I32, I32, D, P, P]),
    "isdfb_profile_enable": (C.c_int, [P, I32]),
    "isdfb_profile_read": (C.c_int, [P, C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(I64), C.POINTER(I64)]),
    "isdfb_debug_program": (C.c_int, [I32, I32, I32, I32, C.POINTER(I32), I32]),
    "isdfb_debug_mc_table": (C.c_int, [C.POINTER(C.c_uint8), C.POINTER(I32)]),
    "isdfb_debug_buffers": (C.c_int, [P, C.POINTER(P), C.POINTER(I64), C.POINTER(P), C.POINTER(P), C.POINTER(I64),
                                      C.POINTER(I32), C.POINTER(I32), C.POINTER(I64), C.POINTER(P)]),
}

_lib = None


def load():
    """Load the shared library and bind every declared symbol (raises if anything is missing)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            "isdf_b200: CUDA library %s not found. Build it with `python -c 'import __graft_entry__ as g; "
            "g.build()'` (nvcc, sm_90a). There is no CPU fallback." % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)      # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


ERR_ARG, ERR_CUDA, ERR_CAPACITY, ERR_STATE = -1, -2, -3, -4


class IsdfbError(RuntimeError):
    """A C entry's failure; `rc` is its isdfb_status."""

    def __init__(self, msg, rc=None):
        super().__init__(msg)
        self.rc = rc


def check(rc, ctx=None):
    if rc != 0:
        msg = load().isdfb_last_error(ctx)
        raise IsdfbError("isdf_b200 error %d: %s" % (rc, msg.decode() if msg else "?"), rc)
