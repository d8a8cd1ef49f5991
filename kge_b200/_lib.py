"""ctypes binding of libb200kge.so (the C ABI declared in include/b200kge.h).

The library is built in-tree by kge_b200.build (nvcc, sm_90a).  There is NO CPU fallback: if the
shared object is missing or no sm_90 device is present, calls raise.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libb200kge.so")

# enums (include/b200kge.h)
MODELS = {"complex": 0, "distmult": 1, "simple": 2, "cp": 3, "rescal": 4, "transe": 5, "rotate": 6}
SP_, _PO = 0, 1
PREC = {"auto": 0, "fp32": 1, "3xtf32": 2, "tf32": 3, "tf32+bf16x2": 4, "f16x3": 5}
LOSS = {"bce": 1, "kl": 2, "bce_mean": 3, "bce_self_adversarial": 4, "margin_ranking": 5, "soft_margin": 6, "se": 7}
ERR_INVALID, ERR_UNSUPPORTED, ERR_CUDA, ERR_WORKSPACE, ERR_NO_DEVICE = -1, -2, -3, -4, -5


class Rows(C.Structure):
    _fields_ = [("base", C.c_void_p), ("idx", C.c_void_p), ("rows", C.c_int64), ("ld", C.c_int64),
                ("dim", C.c_int32)]


class Labels(C.Structure):
    _fields_ = [("idx", C.c_void_p), ("dense", C.c_void_p), ("ldl", C.c_int64)]


class Dropout(C.Structure):
    """b200kge_dropout_t: rates and mask key of one sub-batch (layout: include/b200kge.h)."""
    _fields_ = [("p_ent", C.c_float), ("p_rel", C.c_float), ("seed", C.c_uint64), ("call", C.c_uint64),
                ("row_base", C.c_int64)]


# every symbol include/b200kge.h declares, with its signature
_RP = C.POINTER(Rows)
_DP = C.POINTER(Dropout)
SIGNATURES = {
    "b200kge_version": (C.c_int, []),
    "b200kge_last_error": (C.c_char_p, []),
    "b200kge_device_ok": (C.c_int, []),
    "b200kge_launch_count": (C.c_int64, [C.c_int]),
    "b200kge_profile_enable": (C.c_int, [C.c_int]),
    "b200kge_profile_last_ms": (C.c_int, [C.POINTER(C.c_float)]),
    "b200kge_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int64, C.c_int64, C.c_int32, C.c_int]),
    "b200kge_score_spo": (C.c_int, [C.c_int, C.c_float, _RP, _RP, _RP, C.c_int64, C.c_void_p, C.c_void_p]),
    "b200kge_score_1vsN": (C.c_int, [C.c_int, C.c_int, C.c_float, C.c_int, _RP, _RP, _RP, C.c_int64,
                                     C.c_void_p, C.c_int64, C.c_void_p, C.c_size_t, C.c_void_p]),
    "b200kge_score_sp_po": (C.c_int, [C.c_int, C.c_float, C.c_int, _RP, _RP, _RP, _RP, C.c_int64,
                                      C.c_void_p, C.c_int64, C.c_void_p, C.c_size_t, C.c_void_p]),
    "b200kge_score_sp_po_bcast": (C.c_int, [C.c_int, C.c_float, C.c_int, _RP, _RP, _RP, _RP, C.c_int64, C.c_void_p,
                                            C.c_void_p, C.c_int, C.c_int64, C.c_int64, C.c_void_p, C.c_size_t,
                                            C.c_void_p]),
    "b200kge_score_1vsN_loss": (C.c_int, [C.c_int, C.c_int, C.c_float, C.c_int, _RP, _RP, _RP, C.c_int64,
                                          C.POINTER(Labels), C.c_int, C.c_float, C.c_void_p, C.c_void_p,
                                          C.c_void_p, C.c_size_t, C.c_void_p]),
    "b200kge_score_1vsN_rank": (C.c_int, [C.c_int, C.c_int, C.c_float, C.c_int, _RP, _RP, _RP, C.c_int64,
                                          C.c_void_p, C.c_void_p, C.c_int64, C.c_float, C.c_float,
                                          C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "b200kge_rank_sp_po": (C.c_int, [C.c_int, C.c_float, C.c_int, _RP, _RP, _RP, _RP, C.c_int64, C.c_void_p, C.c_void_p,
                                     C.c_int64, C.c_float, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t,
                                     C.c_void_p]),
    "b200kge_rank_sp_po_csr": (C.c_int, [C.c_int, C.c_float, C.c_int, _RP, _RP, _RP, _RP, C.c_int64, C.c_void_p,
                                         C.c_void_p, C.c_void_p, C.c_void_p, C.c_float, C.c_float, C.c_void_p,
                                         C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "b200kge_rank_sp_po_eval": (C.c_int, [C.c_int, C.c_float, C.c_int, _RP, _RP, C.c_int64, C.c_void_p, C.c_void_p,
                                          C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                          C.c_void_p, C.c_void_p, C.c_float, C.c_float, C.c_void_p, C.c_void_p,
                                          C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "b200kge_shard_gather_rows":(C.c_int, [_RP, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p]),
    "b200kge_loss_dense": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.POINTER(Labels), C.c_int,
                                     C.c_float, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "b200kge_rank_dense": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p,
                                     C.c_int64, C.c_float, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p]),
    "b200kge_ns_score": (C.c_int, [C.c_int, C.c_float, _RP, _RP, _RP, _RP, C.c_int, C.c_void_p, C.c_int64,
                                   C.c_int64, C.c_int, C.c_void_p, C.c_int64, C.c_void_p]),
    "b200kge_sample_uniform": (C.c_int, [C.c_uint64, C.c_uint64, C.c_int64, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p]),
    "b200kge_sample_uniform_filtered": (C.c_int, [C.c_uint64, C.c_uint64, C.c_int64, C.c_int64, C.c_int64, C.c_void_p,
                                                  C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p,
                                                  C.c_void_p]),
    "b200kge_filter_index_build": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_void_p,
                                             C.c_void_p, C.c_void_p, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "b200kge_sample_frequency": (C.c_int, [C.c_uint64, C.c_uint64, C.c_int64, C.c_void_p, C.c_int64, C.c_int64,
                                           C.c_void_p, C.c_void_p]),
    "b200kge_sample_frequency_filtered": (C.c_int, [C.c_uint64, C.c_uint64, C.c_int64, C.c_int64, C.c_int64, C.c_void_p,
                                                    C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p,
                                                    C.c_void_p, C.c_void_p, C.c_void_p]),
    "b200kge_frequency_cdf_build": (C.c_int, [C.c_void_p, C.c_int64, C.c_double, C.c_void_p]),
    "b200kge_frequency_filter_build": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p,
                                                 C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "b200kge_train_1vsall_forward": (C.c_int, [C.c_int, C.c_float, C.c_int, _RP, _RP, C.c_int64, C.c_void_p,
                                               C.c_int64, C.c_int, C.c_float, _DP, C.c_void_p, C.c_void_p,
                                               C.c_size_t, C.c_void_p]),
    "b200kge_train_1vsall_backward": (C.c_int, [C.c_int, C.c_float, _RP, _RP, C.c_int64, C.c_void_p, C.c_int64,
                                                C.c_int, C.c_float, _DP, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64,
                                                C.c_void_p, C.c_size_t, C.c_void_p]),
    "b200kge_train_1vsall_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int64, C.c_int64, C.c_int32, C.c_int]),
    "b200kge_train_1vsall_forward_host": (C.c_int, [C.c_int, C.c_float, C.c_int, _RP, _RP, C.c_void_p,
                                                    C.c_int64, C.c_int, C.c_float, C.c_void_p, C.c_void_p,
                                                    C.c_size_t, C.c_void_p]),
    "b200kge_kvsall_index_build": (C.c_int, [C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                             C.c_void_p, C.c_void_p, C.POINTER(C.c_int64)]),
    "b200kge_kvsall_lookup": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64,
                                        C.c_int64, C.c_void_p, C.c_void_p]),
    "b200kge_kvsall_gather": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64,
                                        C.c_void_p, C.c_void_p, C.c_void_p]),
    # experimental (not validated on hardware yet)
    "b200kge_gemm_nt_workspace_bytes": (C.c_size_t, [C.c_int64, C.c_int64, C.c_int64]),
    "b200kge_gemm_nt": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_int64,
                                    C.c_void_p, C.c_int64, C.c_void_p, C.c_size_t, C.c_void_p]),
    "b200kge_score_1vsN_backward_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int64, C.c_int64, C.c_int32]),
    "b200kge_score_1vsN_backward": (C.c_int, [C.c_int, C.c_int, C.c_float, _RP, _RP, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p,
                                              C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p,
                                              C.c_size_t, C.c_void_p]),
    "b200kge_score_1vsN_loss_csr_backward": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_float, _RP, _RP, C.c_void_p,
                                                       C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_float,
                                                       C.c_int, C.c_float, C.c_int64, _DP, C.c_void_p, C.c_int64,
                                                       C.c_void_p, C.c_int64, C.c_void_p, C.c_size_t, C.c_void_p]),
    "b200kge_score_1vsN_loss_csr_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int64, C.c_int64, C.c_int32, C.c_int64]),
    "b200kge_score_1vsN_loss_csr": (C.c_int, [C.c_int, C.c_int, C.c_float, C.c_int, _RP, _RP, _RP, C.c_int64,
                                                C.c_void_p, C.c_void_p, C.c_int64, C.c_float, C.c_int, C.c_float,
                                                C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "b200kge_ns_backward_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int64, C.c_int64, C.c_int32, C.c_int]),
    "b200kge_ns_backward": (C.c_int, [C.c_int, C.c_float, _RP, _RP, C.c_void_p, C.c_int, C.c_void_p, C.c_int64,
                                      C.c_int64, C.c_int, _DP, C.c_void_p, C.c_int64, C.c_float, C.c_int64, C.c_void_p,
                                      C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_size_t, C.c_void_p]),
    "b200kge_ns_backward_sparse_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int64, C.c_int64, C.c_int32, C.c_int64,
                                                                 C.c_int64, C.c_int]),
    "b200kge_ns_backward_sparse": (C.c_int, [C.c_int, C.c_float, _RP, _RP, C.c_void_p, C.c_int, C.c_void_p, C.c_int64,
                                             C.c_int64, C.c_int, _DP, C.c_void_p, C.c_int64, C.c_float, C.c_int64,
                                             C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64,
                                             C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64,
                                             C.c_void_p, C.c_size_t, C.c_void_p]),
    "b200kge_ns_p_backward_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int64, C.c_int64, C.c_int32, C.c_int64,
                                                            C.c_int64]),
    "b200kge_ns_p_backward": (C.c_int, [C.c_int, C.c_float, _RP, _RP, C.c_void_p, C.c_void_p, C.c_int64, C.c_int64,
                                        C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64,
                                        C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p,
                                        C.c_size_t, C.c_void_p]),
    "b200kge_ns_shared_score_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int64, C.c_int64, C.c_int32]),
    "b200kge_ns_shared_score": (C.c_int, [C.c_int, C.c_float, C.c_int, _RP, _RP, C.c_void_p, C.c_int, C.c_void_p,
                                          C.c_int64, C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int, C.c_void_p,
                                          C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_size_t, C.c_void_p]),
    "b200kge_ns_shared_backward_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int64, C.c_int64, C.c_int32, C.c_int64,
                                                                 C.c_int64]),
    "b200kge_ns_shared_backward": (C.c_int, [C.c_int, C.c_float, _RP, _RP, C.c_void_p, C.c_int, C.c_void_p, C.c_int64,
                                             C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int, C.c_void_p,
                                             C.c_int64, C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_void_p,
                                             C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                             C.c_int64, C.c_void_p, C.c_size_t, C.c_void_p]),
    "b200kge_optim_step_workspace_bytes": (C.c_size_t, [C.c_int64, C.c_int64, C.c_int64, C.c_int]),
    "b200kge_adagrad_step": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p, C.c_int64,
                                       C.c_int, C.c_int, C.c_float, C.c_float, C.c_float, C.c_void_p, C.c_size_t,
                                       C.c_void_p]),
    "b200kge_sparse_adam_step": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_void_p,
                                           C.c_void_p, C.c_int64, C.c_int, C.c_float, C.c_float, C.c_float, C.c_float,
                                           C.c_void_p, C.c_size_t, C.c_void_p]),
    "b200kge_ns_loss_workspace_bytes": (C.c_size_t, [C.c_int64]),
    "b200kge_ns_loss": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_void_p, C.c_int, C.c_float, C.c_float,
                                  C.c_float, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_size_t,
                                  C.c_void_p]),
    "b200kge_lookup_penalty": (C.c_int, [_RP, C.c_void_p, C.c_float, C.c_int, C.c_float, C.c_void_p, C.c_void_p,
                                           C.c_size_t, C.c_void_p]),
    "b200kge_normalize_rows": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.c_float, C.c_void_p]),
    "b200kge_dropout_mask": (C.c_int, [C.c_float, C.c_uint64, C.c_uint64, C.c_int, C.c_int64, C.c_int64, C.c_int32,
                                       C.c_void_p, C.c_void_p]),
    "b200kge_score_1vsN_loss_csr_dropout_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int64, C.c_int64, C.c_int32,
                                                                         C.c_int64]),
    "b200kge_score_1vsN_loss_csr_dropout": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_float, C.c_int, _RP, _RP,
                                                      C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p,
                                                      C.c_int64, C.c_float, C.c_int, C.c_float, _DP, C.c_void_p,
                                                      C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "b200kge_ns_score_dropout": (C.c_int, [C.c_int, C.c_float, _RP, _RP, C.c_void_p, C.c_int, C.c_void_p, C.c_int64,
                                           C.c_int64, C.c_int, _DP, C.c_void_p, C.c_int64, C.c_void_p]),
    "b200kge_score_so_loss_csr_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int64, C.c_int64, C.c_int32, C.c_int64,
                                                               C.c_int]),
    "b200kge_score_so_loss_csr": (C.c_int, [C.c_int, C.c_float, C.c_int, _RP, _RP, C.c_void_p, C.c_void_p, C.c_int64,
                                            C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_float, _DP, C.c_void_p,
                                            C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "b200kge_score_so_loss_csr_backward": (C.c_int, [C.c_int, C.c_float, _RP, _RP, C.c_void_p, C.c_void_p, C.c_int64,
                                                     C.c_void_p, C.c_void_p, C.c_int, C.c_float, C.c_int64, _DP,
                                                     C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p,
                                                     C.c_size_t, C.c_void_p]),
}

#: the most relations b200kge_ns_p_backward serves (B200KGE_NS_P_MAX_RELATIONS)
NS_P_MAX_RELATIONS = 4096

#: negative-sampling scoring implementations of the dropout entry points (B200KGE_NS_*); "all" draws like "batch"
NS_IMPL = {"triple": 0, "batch": 1, "all": 1}

_lib = None


class B200KgeError(RuntimeError):
    pass


def load() -> C.CDLL:
    """Loads libb200kge.so (raises if it has not been built: no silent fallback)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise B200KgeError(
                f"{LIB_PATH} not found: build it with `python -m kge_b200.build` "
                "(kge_b200 has no CPU / PyTorch fallback)"
            )
        lib = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(lib, name)  # AttributeError if the symbol is missing
            fn.restype = res
            fn.argtypes = args
        _lib = lib
    return _lib


def check(rc: int) -> None:
    if rc == 0:
        return
    msg = load().b200kge_last_error().decode("utf-8", "replace")
    if rc in (ERR_INVALID,):
        raise ValueError(msg)
    if rc == ERR_UNSUPPORTED:
        raise NotImplementedError(msg)
    # includes the literal "CUDA out of memory" when allocation failed (LibKGE train.py:384-413)
    raise B200KgeError(msg)
