"""ctypes binding of libb200hotpath.so (include/b200_hotpath.h).

The product path has no CPU fallback: if the library is missing or a call fails this module
raises.  `lib()` loads lazily so that CPU-only tooling (config parsing, the oracle, the gloo
tests) can import the package without a GPU.
"""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path

_PKG = Path(__file__).resolve().parent
LIB_PATH = _PKG / "libb200hotpath.so"

_vp, _i, _ll, _f, _sz = C.c_void_p, C.c_int, C.c_longlong, C.c_float, C.c_size_t

# name -> (restype, argtypes); mirrors include/b200_hotpath.h one to one
SIGNATURES = {
    "b200_version": (_i, []),
    "b200_last_error": (C.c_char_p, []),
    "b200_device_ok": (_i, []),
    "b200_launch_count": (C.c_ulonglong, []),
    "b200_tensor_map_cache_stats": (None, [C.POINTER(C.c_ulonglong), C.POINTER(C.c_ulonglong)]),
    "b200_gemm_bf16": (_i, [_i, _i, _i, _i, _i, _i, _vp, _ll, _ll, _vp, _ll, _ll, _vp, _ll, _ll,
                            _vp, _ll, _ll, _i, _f, _f, _vp, _vp, _i, _vp]),
    "b200_newton_schulz_workspace_bytes": (_sz, [_i, _i, _i, _i]),
    "b200_newton_schulz": (_i, [_vp, _vp, _i, _i, _i, _i, _f, _f, _f, _vp, _vp, _vp, _sz, _vp]),
    "b200_newton_schulz_allgather": (_i, [_vp, _vp, _i, _i, _i, _i, _f, _f, _f, _vp, _vp, _vp, _sz, _vp, _i, _vp]),
    "b200_reduce_workspace_bytes": (_sz, [_i]),
    "b200_muon_momentum": (_i, [_vp, _i, _vp, _vp, _vp, _ll, _i, _f, _i, _f, _vp, _sz, _vp]),
    "b200_shampoo_stats": (_i, [_vp, _vp, _ll, _ll, _vp, _vp, _i, _i, _i, _f, _f, _vp]),
    "b200_shampoo_root_workspace_bytes": (_sz, [_i, _i]),
    "b200_shampoo_root": (_i, [_vp, _vp, _vp, _vp, _i, _i, _f, _f, _i, _vp, _sz, _vp]),
    "b200_shampoo_root_newton_workspace_bytes": (_sz, [_i, _i]),
    "b200_shampoo_root_newton": (_i, [_vp, _vp, _vp, _vp, _i, _i, _f, _i, _f, _vp, _vp, _vp, _sz, _vp]),
    "b200_shampoo_precond_workspace_bytes": (_sz, [_i, _i, _i]),
    "b200_shampoo_precond": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _ll, _ll, _vp, _ll, _ll, _i, _i, _i, _f, _vp,
                                  _sz, _vp]),
    "b200_shampoo_graft_workspace_bytes": (_sz, [_i]),
    "b200_shampoo_graft": (_i, [_vp, _vp, _vp, _vp, _ll, _i, _f, _vp, _sz, _vp]),
    "b200_ns_scales": (_i, [_vp, _vp, _vp, _i, _f, _vp]),
    "b200_axpy_update": (_i, [_vp, _vp, _vp, _i, _ll, _f, _vp]),
    "b200_sgd_momentum": (_i, [_vp, _vp, _vp, _i, _vp, _ll, _f, _i, _f, _f, _vp]),
    "b200_adamw": (_i, [_vp, _vp, _vp, _i, _vp, _vp, _ll, _f, _f, _f, _f, _f, _f, _f, _f, _vp]),
    "b200_adam_direction": (_i, [_vp, _vp, _i, _vp, _vp, _ll, _f, _f, _f, _f, _f, _f, _f, _vp]),
    "b200_lion": (_i, [_vp, _vp, _vp, _i, _vp, _vp, _ll, _f, _f, _f, _f, _f, _vp, _f, _f, _i, _vp]),
    "b200_sgd": (_i, [_vp, _vp, _vp, _i, _vp, _vp, _ll, _f, _f, _f, _i, _f, _f, _vp, _f, _f, _i, _vp]),
    "b200_clip_accum": (_i, [_vp, _i, _vp, _ll, _f, _f, _i, _vp]),
    "b200_sumsq": (_i, [_vp, _i, _vp, _ll, _i, _i, _vp, _sz, _vp]),
    "b200_split_bf16": (_i, [_vp, _ll, _vp, _vp, _ll, _i, _i, _f, _f, _vp]),
    "b200_ema_split": (_i, [_vp, _i, _vp, _vp, _vp, _vp, _ll, _f, _f, _f, _f, _vp]),
    "b200_graft_update": (_i, [_vp, _vp, _vp, _vp, _ll, _i, _vp, _vp, _f, _vp]),
    "b200_rmsnorm_fwd": (_i, [_vp, _vp, _vp, _vp, _i, _i, _f, _i, _vp]),
    "b200_rmsnorm_bwd_workspace_bytes": (_sz, [_i, _i]),
    "b200_rmsnorm_bwd": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _vp, _sz, _vp]),
    "b200_rmsnorm_bwd_partial_rows": (_i, [_i, _i]),
    "b200_add_rmsnorm_fwd": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _f, _i, _vp]),
    "b200_add_rmsnorm_bwd": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _vp, _sz, _vp]),
    "b200_rope": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp]),
    "b200_rope_pos": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp]),
    "b200_mlp_gateup_glu_fwd": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _vp]),
    "b200_mlp_down_glu_bwd": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _vp]),
    "b200_embedding_bwd_workspace_bytes": (_sz, [_i, _i]),
    "b200_embedding_bwd": (_i, [_vp, _vp, _vp, _i, _ll, _i, _i, _vp, _sz, _vp]),
    "b200_glu_fwd": (_i, [_vp, _vp, _vp, _ll, _vp]),
    "b200_glu_bwd": (_i, [_vp, _vp, _vp, _vp, _vp, _ll, _vp]),
    "b200_ce_fwd": (_i, [_vp, _ll, _vp, _i, _i, _ll, _vp, _vp, _vp]),
    "b200_ce_bwd": (_i, [_vp, _ll, _vp, _i, _i, _ll, _vp, _vp, _vp]),
    "b200_attn_fwd": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _f, _i, _vp]),
    "b200_attn_bwd_workspace_bytes": (_sz, [_i, _i, _i, _i, _i]),
    "b200_attn_bwd": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _f, _i,
                           _vp, _sz, _vp]),
    "b200_attn_bwd_strided": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _f, _i, _i, _vp, _sz, _vp]),
    "b200_attn_fwd_doc": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _f, _vp]),
    "b200_attn_bwd_doc_workspace_bytes": (_sz, [_i, _i, _i, _i, _i]),
    "b200_attn_bwd_doc": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _f, _i, _vp, _sz,
                               _vp]),
    "b200_attn_fwd_window": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _f, _vp]),
    "b200_attn_bwd_window_workspace_bytes": (_sz, [_i, _i, _i, _i, _i]),
    "b200_attn_bwd_window": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _vp, _vp, _vp, _i, _i, _i, _i, _i, _f, _i,
                                  _vp, _sz, _vp]),
    "b200_attn_fwd_prefix": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _f, _vp]),
    "b200_attn_bwd_prefix_workspace_bytes": (_sz, [_i, _i, _i, _i, _i]),
    "b200_attn_bwd_prefix": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _f, _i, _vp,
                                  _sz, _vp]),
    "b200_attn_fwd_dropout": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i, _vp, _i, _i, _i, _i, _i, _f, _i, _f, C.c_uint64,
                                   _vp]),
    "b200_attn_bwd_dropout_workspace_bytes": (_sz, [_i, _i, _i, _i, _i]),
    "b200_attn_bwd_dropout": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _f,
                                   _i, _f, C.c_uint64, _i, _vp, _sz, _vp]),
    "b200_attn_fwd_alibi": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i, _vp, _i, _i, _i, _i, _i, _f, _vp]),
    "b200_attn_bwd_alibi": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _f,
                                 _i, _vp, _sz, _vp]),
    "b200_attn_decode_alibi": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i, _vp, _i, _i, _i, _i, _i, _f, _i, _vp, _sz,
                                    _vp]),
    "b200_attn_decode_window": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _f, _i, _vp, _sz, _vp]),
    "b200_attn_decode_workspace_bytes": (_sz, [_i, _i, _i, _i]),
    "b200_attn_decode": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _f, _i, _vp, _sz, _vp]),
    "b200_kv_append": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp]),
    "b200_rope_half": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp]),
    "b200_mlp_gateup_silu_fwd": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _vp]),
    "b200_mlp_down_silu_bwd": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _vp]),
    "b200_silu_glu_fwd": (_i, [_vp, _vp, _vp, _ll, _vp]),
    "b200_silu_glu_bwd": (_i, [_vp, _vp, _vp, _vp, _vp, _ll, _vp]),
    "b200_kv_append_half": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp]),
    "b200_kv_quantize": (_i, [_vp, _vp, _i, _i, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _vp]),
    "b200_kv_append_quant": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i,
                                  _i, _vp]),
    "b200_attn_fwd_cached": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _vp, _i, _i, _i, _i, _i, _i, _f, _vp]),
    "b200_kv_dequantize": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _vp]),
    "b200_attn_decode_ring": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _vp, _i, _i, _i, _i, _i, _f, _vp, _sz, _vp]),
    "b200_attn_fwd_ring": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _vp, _i, _i, _i, _i, _i, _i, _f, _vp]),
    "b200_kv_append_ring": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp]),
    "b200_attn_decode_quant": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _vp, _i, _i, _i, _i, _i, _i, _i, _f,
                                    _i, _vp, _sz, _vp]),
    "b200_attn_decode_beam": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _vp, _i, _i, _i, _i, _i, _i, _i,
                                   _i, _f, _i, _vp, _sz, _vp]),
    "b200_attn_decode_beam_workspace_bytes": (_sz, [_i, _i, _i, _i, _i]),
    "b200_attn_decode_beam_pack": (_i, [_i, _i, _i]),
    "b200_attn_decode_multi": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _vp, _i, _i, _i, _i, _i, _i, _f, _i, _vp,
                                    _sz, _vp]),
    "b200_attn_decode_multi_workspace_bytes": (_sz, [_i, _i, _i, _i, _i]),
    "b200_kv_append_beam": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _vp]),
    "b200_kv_beam_fork": (_i, [_vp, _i, _vp, _i, _i, _i, _i, _vp]),
    "b200_moe_route_workspace_bytes": (_sz, [_i, _i, _i]),
    "b200_moe_max_tiles": (_i, [_i, _i, _i]),
    "b200_moe_route": (_i, [_vp, _vp, _i, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
    "b200_moe_permute": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp, _vp]),
    "b200_moe_gemm": (_i, [_i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp]),
    "b200_moe_wgrad": (_i, [_vp, _ll, _vp, _ll, _vp, _i, _i, _i, _i, _vp, _vp, _vp]),
    "b200_moe_combine_fwd": (_i, [_vp, _vp, _vp, _i, _i, _i, _vp, _vp]),
    "b200_moe_combine_bwd": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp, _vp, _vp,
                                  _vp]),
    "b200_moe_unpermute": (_i, [_vp, _vp, _vp, _i, _i, _i, _vp, _vp]),
}



class NsGroup(C.Structure):
    """b200_ns_group (include/b200_hotpath.h)"""
    _fields_ = [("x_in", _vp), ("x_out", _vp), ("batch", _i), ("rows", _i), ("cols", _i), ("inv_norm", _vp),
                ("inv_norm_sq", _vp), ("peer_out", C.POINTER(_vp)), ("n_peers", _i)]


class GemmProblem(C.Structure):
    """b200_gemm_problem (include/b200_hotpath.h)"""
    _fields_ = [("a_mn", _i), ("b_mn", _i), ("M", _i), ("N", _i), ("K", _i), ("batch", _i),
                ("A", _vp), ("lda", _ll), ("strideA", _ll), ("B", _vp), ("ldb", _ll), ("strideB", _ll),
                ("C", _vp), ("ldc", _ll), ("strideC", _ll), ("D", _vp), ("ldd", _ll), ("strideD", _ll),
                ("alpha", _f), ("beta", _f), ("alpha_vec", _vp), ("beta_vec", _vp), ("symmetric", _i),
                ("k_splits", _i), ("splitk_ws", _vp), ("peer_D", C.POINTER(_vp)), ("n_peers", _i)]


class DwJob(C.Structure):
    """b200_dw_job (include/b200_hotpath.h)"""
    _fields_ = [("partials", _vp), ("dw", _vp), ("n_partials", _i), ("dw_is_bf16", _i), ("accumulate", _i),
                ("reserved", _i)]


SIGNATURES["b200_rmsnorm_dw_reduce"] = (_i, [C.POINTER(DwJob), _i, _i, _vp])
SIGNATURES["b200_gemm_grouped"] = (_i, [C.POINTER(GemmProblem), _i, _vp])
SIGNATURES["b200_newton_schulz_multi_workspace_bytes"] = (_sz, [C.POINTER(NsGroup), _i, _i])
SIGNATURES["b200_newton_schulz_multi"] = (_i, [C.POINTER(NsGroup), _i, _i, _f, _f, _f, _vp, _sz, _vp])

_lib = None


class B200Error(RuntimeError):
    pass


def lib() -> C.CDLL:
    """Load the C-ABI library (once). Raises if it has not been built."""
    global _lib
    if _lib is None:
        path = Path(os.environ.get("B200_HOTPATH_LIB", LIB_PATH))
        if not path.exists():
            raise B200Error(
                f"{path} not found: run `python __graft_entry__.py` (nvcc, sm_90a) first. "
                "There is no CPU fallback for the hot path.")
        handle = C.CDLL(str(path))
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(handle, name)  # AttributeError if the symbol is not exported
            fn.restype = res
            fn.argtypes = args
        _lib = handle
    return _lib


def check(rc: int, what: str) -> None:
    if rc != 0:
        msg = lib().b200_last_error()
        raise B200Error(f"{what} failed (rc={rc}): {msg.decode() if msg else '?'}")


def require_device() -> None:
    """Fail loudly when the CUDA path cannot run (no GPU / not an sm_90 part)."""
    import torch
    if not torch.cuda.is_available():
        raise B200Error("CUDA device required: the hot path has no CPU fallback")
    if not lib().b200_device_ok():
        raise B200Error("the current CUDA device is not compute capability 9.0 (H100)")
