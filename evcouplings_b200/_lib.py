"""
ctypes binding of libevcplm.so (C ABI declared in include/evcplm.h).

There is NO fallback: if the CUDA library is missing or cannot be loaded the
import of the engine fails loudly (EngineUnavailableError).  Build it in-tree
with ``python -c "import __graft_entry__ as g; g.build()"`` or
``evcouplings_b200/csrc/build.sh``.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "csrc", "libevcplm.so")
ABI_VERSION = 2


class EngineUnavailableError(RuntimeError):
    """libevcplm.so (the sm_90a CUDA engine) is missing / unloadable / has no device."""


class EngineError(RuntimeError):
    """A libevcplm call returned non-zero."""


c_void_p = ctypes.c_void_p
c_i32 = ctypes.c_int32
c_i64 = ctypes.c_int64
c_f32 = ctypes.c_float
c_f64 = ctypes.c_double


class FitParams(ctypes.Structure):
    """evc_fit_params_t (include/evcplm.h)."""
    _fields_ = [("max_iterations", c_i32), ("m", c_i32), ("epsilon", c_f32), ("lambda_h", c_f32),
                ("lambda_J", c_f32), ("max_linesearch", c_i32), ("min_step", c_f64), ("max_step", c_f64),
                ("ftol", c_f64), ("gtol", c_f64), ("xtol", c_f64), ("precision_schedule", c_i32),
                ("switch_factor", c_f32)]


class FitResult(ctypes.Structure):
    """evc_fit_result_t (include/evcplm.h)."""
    _fields_ = [("status", c_i32), ("iterations", c_i32), ("evaluations", c_i32), ("switched_at", c_i32),
                ("fx", c_f64), ("negloglk", c_f64), ("seconds", c_f64)]


class FitState(ctypes.Structure):
    """evc_fit_state_t (include/evcplm.h): the fit's scalars at an iteration boundary."""
    _fields_ = [("version", c_i32), ("returning", c_i32), ("status", c_i32), ("k", c_i32), ("evaluations", c_i32),
                ("m", c_i32), ("hist", c_i32), ("end", c_i32), ("low", c_i32), ("switched_at", c_i32),
                ("n", c_i64), ("fx", c_f64), ("negloglk", c_f64), ("xnorm", c_f64), ("gnorm", c_f64),
                ("ys", c_f64 * 32), ("yy", c_f64), ("seconds", c_f64)]


FIT_STATE_VERSION = 1
FIT_VEC_X, FIT_VEC_G, FIT_VEC_S, FIT_VEC_Y = 0, 1, 2, 3
# which buffer evc_plm_copy_stage copies (EVC_STAGE_* of include/evcplm.h)
STAGE = dict(Wt_hi=0, Wt_lo=1, Wp_hi=2, Wp_lo=3, Zt=4, Xt=5, Rt_hi=6, Rt_lo=7, Gd=8, gh_part=9, fx_part=10, X=11)

ALLREDUCE_CB = ctypes.CFUNCTYPE(ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, c_i64, ctypes.c_void_p)
PROGRESS_CB = ctypes.CFUNCTYPE(ctypes.c_int, ctypes.c_void_p, c_i32, c_f64, c_f64, c_f64, c_f64, c_i32, c_f64,
                               c_f64, c_f64)
CHECKPOINT_CB = ctypes.CFUNCTYPE(ctypes.c_int, ctypes.c_void_p, ctypes.POINTER(FitState), ctypes.c_void_p)

# status codes of evc_plm_fit -> libLBFGS names (what plmc prints after "Gradient optimization:")
LBFGS_STATUS = {
    0: "LBFGS_SUCCESS", 2: "LBFGS_ALREADY_MINIMIZED", -1021: "LBFGSERR_CANCELED",
    -1000: "LBFGSERR_INVALIDPARAMETERS", -1001: "LBFGSERR_MINIMUMSTEP", -1002: "LBFGSERR_MAXIMUMSTEP",
    -1003: "LBFGSERR_MAXIMUMLINESEARCH", -1004: "LBFGSERR_MAXIMUMITERATION", -1005: "LBFGSERR_WIDTHTOOSMALL",
    -1006: "LBFGSERR_ROUNDING_ERROR", -1007: "LBFGSERR_INCREASEGRADIENT",
}

# name -> (restype, argtypes); mirrors include/evcplm.h one to one
PROTOTYPES = {
    "evc_abi_version": (ctypes.c_int, []),
    "evc_last_error": (ctypes.c_char_p, []),
    "evc_device_count": (ctypes.c_int, []),
    "evc_device_info": (ctypes.c_int, [c_i32, c_void_p, c_void_p, c_void_p, c_void_p]),
    "evc_hamming_counts": (ctypes.c_int, [c_void_p, c_i64, c_i32, c_i32, c_i32, c_void_p]),
    "evc_hamming_plane_words": (c_i64, [c_i64, c_i32]),
    "evc_hamming_num_tiles": (c_i64, [c_i64]),
    "evc_hamming_pack": (ctypes.c_int, [c_void_p, c_i64, c_i32, c_void_p, c_void_p]),
    "evc_hamming_count_tiles": (ctypes.c_int, [c_void_p, c_i64, c_i32, c_i32, c_i64, c_i64, c_void_p, c_void_p]),
    "evc_hamming_counts_mult": (ctypes.c_int, [c_void_p, c_void_p, c_i64, c_i32, c_i32, c_i32, c_void_p]),
    "evc_hamming_count_tiles_mult": (ctypes.c_int, [c_void_p, c_void_p, c_i64, c_i32, c_i32, c_i64, c_i64, c_void_p,
                                                    c_void_p]),
    "evc_msa_unique": (ctypes.c_int, [c_void_p, c_i64, c_i32, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "evc_msa_unique_host": (ctypes.c_int, [c_void_p, c_i64, c_i32, c_i32, c_void_p, c_void_p, c_void_p, c_void_p]),
    "evc_a2m_scan": (ctypes.c_int, [ctypes.c_char_p, c_void_p, c_void_p, c_void_p]),
    "evc_a2m_read": (ctypes.c_int, [ctypes.c_char_p, c_i64, c_i64, c_void_p, c_void_p, c_i64]),
    "evc_msa_encode": (ctypes.c_int, [c_void_p, c_i64, c_i64, c_void_p, c_void_p, c_i64, c_void_p, c_void_p, c_void_p]),
    "evc_identities_to_seq": (ctypes.c_int, [c_void_p, c_void_p, c_i64, c_i32, c_void_p, c_void_p]),
    "evc_plm_create": (ctypes.c_int, [c_void_p, c_void_p, c_i64, c_i32, c_i32, c_i32, c_void_p, c_i32]),
    "evc_plm_create_alphabet": (ctypes.c_int, [c_void_p, c_void_p, c_i64, c_i32, c_i32, c_i32, c_void_p, c_i32]),
    "evc_plm_destroy": (None, [c_void_p]),
    "evc_plm_num_params": (c_i64, [c_void_p]),
    "evc_plm_eval_data": (ctypes.c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "evc_plm_set_backward": (ctypes.c_int, [c_void_p, c_i32]),
    "evc_plm_set_forward": (ctypes.c_int, [c_void_p, c_i32]),
    "evc_plm_set_precision": (ctypes.c_int, [c_void_p, c_i32]),
    "evc_plm_set_seq_chunk": (ctypes.c_int, [c_void_p, c_i64]),
    "evc_plm_tc_bytes": (ctypes.c_int, [c_i64, c_i32, c_i32, c_i32, c_i64, c_i32, c_void_p]),
    "evc_plm_tc_bytes_alphabet": (ctypes.c_int, [c_i64, c_i32, c_i32, c_i32, c_i64, c_i32, c_void_p]),
    "evc_plm_device_bytes": (c_i64, [c_void_p]),
    "evc_plm_copy_onehot": (ctypes.c_int, [c_void_p, c_void_p, c_i64]),
    "evc_plm_copy_stage": (ctypes.c_int, [c_void_p, c_i32, c_void_p, c_i64]),
    "evc_fit_workspace_bytes": (c_i64, [c_i64, c_i32]),
    "evc_plm_set_host_history": (ctypes.c_int, [c_void_p, c_i32]),
    "evc_fit_workspace_split_bytes": (ctypes.c_int, [c_i64, c_i32, c_i32, c_void_p, c_void_p]),
    "evc_plm_host_bytes": (ctypes.c_int, [c_void_p, c_void_p, c_void_p]),
    "evc_fit_default_params": (None, [c_void_p]),
    "evc_plm_fit": (ctypes.c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                   c_void_p]),
    "evc_plm_fit_checkpointed": (ctypes.c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                                c_void_p, c_void_p, c_f64, c_void_p, c_void_p, c_void_p]),
    "evc_plm_fit_prepare": (ctypes.c_int, [c_void_p, c_i32]),
    "evc_plm_fit_vector": (ctypes.c_int, [c_void_p, c_i32, c_i32, c_void_p]),
    "evc_plm_pack_fx": (ctypes.c_int, [c_void_p, c_void_p, c_void_p]),
    "evc_plm_unpack_fx": (ctypes.c_int, [c_void_p, c_void_p, c_void_p]),
    "evc_plm_set_profiling": (ctypes.c_int, [c_void_p, c_i32]),
    "evc_plm_last_stage_ms": (ctypes.c_int, [c_void_p, c_void_p]),
    "evc_plm_add_regulariser": (ctypes.c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_f32, c_f32, c_void_p]),
    "evc_plm_eval_host": (ctypes.c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_f32, c_f32]),
    "evc_plm_weighted_counts": (ctypes.c_int, [c_void_p, c_void_p, c_void_p, c_void_p]),
    "evc_vec_dot": (ctypes.c_int, [c_void_p, c_void_p, c_i64, c_void_p, c_void_p]),
    "evc_vec_axpby": (ctypes.c_int, [c_void_p, c_void_p, c_f32, c_f32, c_i64, c_void_p]),
    "evc_vec_copy": (ctypes.c_int, [c_void_p, c_void_p, c_i64, c_void_p]),
    "evc_vec_sub": (ctypes.c_int, [c_void_p, c_void_p, c_void_p, c_i64, c_void_p]),
    "evc_vec_checksum": (ctypes.c_int, [c_void_p, c_i64, c_void_p, c_void_p]),
    "evc_lbfgs_direction": (ctypes.c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                           c_i64, c_i32, c_i32, c_i32, c_void_p]),
    "evc_lbfgs_update_pair": (ctypes.c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                             c_void_p, c_void_p, c_i64, c_void_p]),
    "evc_ec_scores": (ctypes.c_int, [c_void_p, c_void_p, c_void_p, c_i32, c_i32, c_void_p, c_void_p, c_void_p, c_void_p]),
    "evc_plm_energies": (ctypes.c_int, [c_void_p, c_void_p, c_void_p, c_void_p]),
    "evc_fn_scores": (ctypes.c_int, [c_void_p, c_i32, c_i32, c_void_p, c_void_p]),
    "evc_sampler_create": (ctypes.c_int, [c_void_p, c_void_p, c_i32, c_i32, c_void_p, c_i64, c_i64, ctypes.c_uint64,
                                          c_i32]),
    "evc_sampler_run": (ctypes.c_int, [c_void_p, c_i32, c_f32, c_void_p, c_void_p]),
    "evc_sampler_codes": (ctypes.c_int, [c_void_p, c_void_p, c_void_p]),
    "evc_sampler_set_model": (ctypes.c_int, [c_void_p, c_void_p, c_void_p]),
    "evc_sampler_anneal": (ctypes.c_int, [c_void_p, c_void_p, c_i32, c_void_p, c_void_p, c_void_p]),
    "evc_sampler_create_conditional": (ctypes.c_int, [c_void_p, c_void_p, c_i32, c_i32, c_void_p, c_i32, c_void_p,
                                                      c_void_p, c_i64, c_i64, ctypes.c_uint64, c_i32]),
    "evc_sampler_conditional_fields": (ctypes.c_int, [c_void_p, c_void_p, c_void_p]),
    "evc_sampler_set_ladder": (ctypes.c_int, [c_void_p, c_void_p, c_i32, c_i64]),
    "evc_sampler_temper": (ctypes.c_int, [c_void_p, c_i32, c_void_p, c_void_p, c_void_p]),
    "evc_sampler_ladder_state": (ctypes.c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "evc_sampler_record_best": (ctypes.c_int, [c_void_p, c_void_p]),
    "evc_sampler_best": (ctypes.c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "evc_sampler_descend": (ctypes.c_int, [c_void_p, c_i32, c_void_p, c_void_p, c_void_p]),
    "evc_code_counts": (ctypes.c_int, [c_void_p, c_i64, c_i32, c_i32, c_void_p, c_void_p]),
    "evc_bm_update": (ctypes.c_int, [c_void_p, c_void_p, c_i64, c_void_p, c_i64, c_i32, c_f64, c_f64, c_f64, c_void_p,
                                     c_void_p]),
    "evc_sampler_destroy": (None, [c_void_p]),
}

_lib = None


def load():
    """Load libevcplm.so and bind every symbol of the C ABI (no device needed)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise EngineUnavailableError(
            "CUDA engine library not built: %s is missing. There is no CPU fallback; "
            "build it with evcouplings_b200/csrc/build.sh (nvcc, sm_90a)." % LIB_PATH)
    try:
        lib = ctypes.CDLL(LIB_PATH)
    except OSError as e:
        raise EngineUnavailableError("cannot load %s: %s" % (LIB_PATH, e))
    for name, (restype, argtypes) in PROTOTYPES.items():
        try:
            fn = getattr(lib, name)
        except AttributeError:
            raise EngineUnavailableError("%s does not export %s" % (LIB_PATH, name))
        fn.restype = restype
        fn.argtypes = argtypes
    if lib.evc_abi_version() != ABI_VERSION:
        raise EngineUnavailableError("libevcplm ABI version mismatch")
    _lib = lib
    return lib


def check(rc, what=""):
    if rc != 0:
        msg = load().evc_last_error()
        raise EngineError("%s failed: %s" % (what or "libevcplm call", msg.decode() if msg else "unknown error"))


def require_device():
    """Raise unless at least one CUDA device is usable through the library."""
    lib = load()
    n = lib.evc_device_count()
    if n <= 0:
        raise EngineUnavailableError(
            "libevcplm found no CUDA device; the PLM engine has no CPU fallback")
    return n
