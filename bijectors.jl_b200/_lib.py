"""ctypes binding of libb2b.so (include/b2b.h).  There is NO fallback: if the CUDA library is missing the
import fails loudly, and every entry point needs a CUDA device at call time."""
from __future__ import annotations

import ctypes
import os
from ctypes import POINTER, c_char_p, c_double, c_float, c_int, c_int32, c_int64, c_size_t, c_uint64, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "csrc", "libb2b.so")

B2B_OK = 0
B2B_EINVAL, B2B_EUNSUPPORTED, B2B_EWORKSPACE, B2B_ENONCCL = -1, -2, -3, -4
PLANAR, RADIAL, RQS, COUPLING_AFFINE, BATCHNORM, PERMUTE, STACKED_EW, MVNORMAL_DIAG = 1, 2, 3, 4, 5, 6, 7, 8
EW_IDENTITY, EW_EXP, EW_LOG, EW_SHIFT, EW_SCALE, EW_LEAKY_RELU, EW_LOGIT, EW_TRUNCATED = 0, 1, 2, 3, 4, 5, 6, 7
MAX_CHAIN = 24


class B2BError(RuntimeError):
    """Raised for every non-zero status of the C ABI (mirrors the reference's error(...) sites)."""

    def __init__(self, status: int, where: str = ""):
        self.status = status
        msg = lib().b2b_status_string(status).decode()
        super().__init__(f"{where}: {msg} (status {status})" if where else f"{msg} (status {status})")


class LayerDesc(ctypes.Structure):
    """b2b_layer_desc (include/b2b.h)."""

    _fields_ = [
        ("kind", c_int32),
        ("inverse", c_int32),
        ("n0", c_int32),
        ("n1", c_int32),
        ("n2", c_int32),
        ("n3", c_int32),
        ("f0", c_float),
        ("f1", c_float),
        ("p0", c_void_p),
        ("p1", c_void_p),
        ("p2", c_void_p),
        ("p3", c_void_p),
        ("i0", c_void_p),
        ("i1", c_void_p),
    ]


class LayerDesc64(ctypes.Structure):
    """b2b_layer_desc_f64 (include/b2b.h): the same fields with double parameters."""

    _fields_ = [
        ("kind", c_int32),
        ("inverse", c_int32),
        ("n0", c_int32),
        ("n1", c_int32),
        ("n2", c_int32),
        ("n3", c_int32),
        ("f0", c_double),
        ("f1", c_double),
        ("p0", c_void_p),
        ("p1", c_void_p),
        ("p2", c_void_p),
        ("p3", c_void_p),
        ("i0", c_void_p),
        ("i1", c_void_p),
    ]


# name -> (restype, argtypes); every symbol include/b2b.h declares
_F32P = c_void_p
_SIGS = {
    "b2b_version": (c_int, []),
    "b2b_status_string": (c_char_p, [c_int]),
    "b2b_chain_run_f32": (c_int, [POINTER(LayerDesc), c_int32, c_void_p, c_void_p, c_void_p, c_void_p, c_int32,
                                  c_int64, c_int64, c_int64, c_int, c_void_p, c_size_t, c_void_p]),
    "b2b_chain_workspace_bytes": (c_size_t, [POINTER(LayerDesc), c_int32, c_int32, c_int64, c_int, c_int]),
    "b2b_last_launch_count": (c_int, []),
    "b2b_set_kernel_variant": (c_int, [c_int]),
    "b2b_planar_fwd_f32": (c_int, [_F32P] * 6 + [c_int32, c_int64, c_int64, c_int64, c_int, c_void_p]),
    "b2b_planar_inv_f32": (c_int, [_F32P] * 6 + [c_int32, c_int64, c_int64, c_int64, c_int, c_void_p]),
    "b2b_planar_chain_hostparams_f32": (c_int, [_F32P] * 3 + [c_int32, c_int] + [_F32P] * 3 +
                                        [c_int32, c_int64, c_int64, c_int64, c_int, c_void_p]),
    "b2b_planar_chain_vjp_workspace_bytes": (c_size_t, [c_int32, c_int32, c_int64]),
    "b2b_planar_chain_vjp_f32": (c_int, [POINTER(LayerDesc), c_int32] + [c_void_p] * 7 +
                                 [c_int32, c_int64, c_int64, c_int64, c_int64, c_void_p, c_size_t, c_void_p]),
    "b2b_radial_chain_vjp_workspace_bytes": (c_size_t, [c_int32, c_int32]),
    "b2b_radial_chain_vjp_f32": (c_int, [POINTER(LayerDesc), c_int32] + [c_void_p] * 7 +
                                 [c_int32, c_int64, c_int64, c_int64, c_int64, c_void_p, c_size_t, c_void_p]),
    "b2b_coupling_affine_vjp_workspace_bytes": (c_size_t, [c_int32, c_int32]),
    "b2b_coupling_affine_vjp_f32": (c_int, [POINTER(LayerDesc)] + [c_void_p] * 6 +
                                    [c_int32, c_int64, c_int64, c_int64, c_int64, c_void_p, c_size_t, c_void_p]),
    "b2b_batchnorm_eval_vjp_workspace_bytes": (c_size_t, [c_int32]),
    "b2b_batchnorm_eval_vjp_f32": (c_int, [POINTER(LayerDesc)] + [c_void_p] * 6 +
                                   [c_int32, c_int64, c_int64, c_int64, c_int64, c_void_p, c_size_t, c_void_p]),
    "b2b_rqs_vjp_workspace_bytes": (c_size_t, [c_int32, c_int32]),
    "b2b_rqs_vjp_f32": (c_int, [POINTER(LayerDesc)] + [c_void_p] * 7 +
                        [c_int32, c_int64, c_int64, c_int64, c_int64, c_void_p, c_size_t, c_void_p]),
    "b2b_radial_fwd_f32": (c_int, [_F32P] * 6 + [c_int32, c_int64, c_int64, c_int64, c_int, c_void_p]),
    "b2b_radial_inv_f32": (c_int, [_F32P] * 6 + [c_int32, c_int64, c_int64, c_int64, c_int, c_void_p]),
    "b2b_rqs_fwd_f32": (c_int, [_F32P] * 6 + [c_int32, c_int32, c_int64, c_int64, c_int64, c_int, c_void_p]),
    "b2b_rqs_inv_f32": (c_int, [_F32P] * 6 + [c_int32, c_int32, c_int64, c_int64, c_int64, c_int, c_void_p]),
    "b2b_coupling_affine_fwd_f32": (c_int, [_F32P] * 3 + [c_void_p, c_int32, c_int32, c_void_p, c_int32, c_int32, _F32P,
                                            _F32P, c_int32, c_int64, c_int64, c_int64, c_int, c_void_p, c_size_t,
                                            c_void_p]),
    "b2b_coupling_affine_inv_f32": (c_int, [_F32P] * 3 + [c_void_p, c_int32, c_int32, c_void_p, c_int32, c_int32, _F32P,
                                            _F32P, c_int32, c_int64, c_int64, c_int64, c_int, c_void_p, c_size_t,
                                            c_void_p]),
    "b2b_coupling_workspace_bytes": (c_size_t, [c_int32, c_int32]),
    "b2b_batchnorm_eval_fwd_f32": (c_int, [_F32P] * 7 + [c_float, c_int32, c_int64, c_int64, c_int64, c_int, c_void_p]),
    "b2b_batchnorm_eval_inv_f32": (c_int, [_F32P] * 7 + [c_float, c_int32, c_int64, c_int64, c_int64, c_int, c_void_p]),
    "b2b_batchnorm_train_fwd_f32": (c_int, [_F32P] * 7 + [c_float, c_float, c_int32, c_int64, c_int64, c_int64, c_int, c_void_p,
                                            c_void_p, c_size_t, c_void_p]),
    "b2b_batchnorm_train_workspace_bytes": (c_size_t, [c_int32]),
    "b2b_permute_rows_f32": (c_int, [_F32P] * 3 + [c_void_p, c_int, c_int32, c_int64, c_int64, c_int64, c_int, c_void_p]),
    "b2b_stacked_elementwise_f32": (c_int, [_F32P] * 3 + [c_void_p, _F32P, _F32P, c_int, c_int32, c_int64, c_int64, c_int64,
                                            c_int, c_void_p]),
    "b2b_mvnormal_diag_logpdf_f32": (c_int, [_F32P] * 5 + [c_void_p, c_int32, c_int64, c_int64, c_void_p, c_size_t,
                                             c_void_p]),
    "b2b_chain_workspace_bytes_f64": (c_size_t, [c_int32, c_int]),
    "b2b_chain_run_f64": (c_int, [POINTER(LayerDesc64), c_int32, c_void_p, c_void_p, c_void_p, c_void_p, c_int32, c_int64,
                                  c_int64, c_int64, c_int, c_void_p, c_size_t, c_void_p]),
    "b2b_randn_f32": (c_int, [_F32P] * 3 + [c_uint64, c_uint64, c_int64, c_int32, c_int64, c_int64, c_void_p]),
    "b2b_chain_sample_f32": (c_int, [POINTER(LayerDesc), c_int32, _F32P, _F32P, c_uint64, c_uint64, c_int64, _F32P, _F32P,
                                     c_int32, c_int64, c_int64, c_void_p, c_size_t, c_void_p]),
    "b2b_host_ctx_create": (c_int, [POINTER(c_void_p), c_int32, c_int64, c_int32]),
    "b2b_host_ctx_destroy": (c_int, [c_void_p]),
    "b2b_host_ctx_wait_stream": (c_int, [c_void_p, c_void_p]),
    "b2b_chain_run_host_f32": (c_int, [c_void_p, POINTER(LayerDesc), c_int32, c_void_p, c_void_p, c_void_p,
                                       POINTER(c_double), c_int32, c_int64]),
    "b2b_host_register": (c_int, [c_void_p, c_size_t]),
    "b2b_host_unregister": (c_int, [c_void_p]),
    "b2b_numa_bind_to_device": (c_int, [c_int32, POINTER(c_int32), POINTER(c_int32)]),
    "b2b_device_numa_node": (c_int, [c_int32, POINTER(c_int32)]),
    "b2b_comm_unique_id": (c_int, [c_void_p]),
    "b2b_comm_init_rank": (c_int, [POINTER(c_void_p), c_int, c_int, c_void_p]),
    "b2b_allreduce_sum_f64": (c_int, [c_void_p, c_void_p, c_int32, c_void_p]),
    "b2b_comm_destroy": (c_int, [c_void_p]),
    "b2b_comm_init_all": (c_int, [POINTER(c_void_p), c_int, POINTER(c_int)]),
    "b2b_allreduce_sum_f64_all": (c_int, [c_void_p, POINTER(c_void_p), c_int32, POINTER(c_void_p)]),
    "b2b_workspace_bytes": (c_size_t, [POINTER(LayerDesc), c_int32, c_int64]),
}

_lib = None


def lib() -> ctypes.CDLL:
    """Load libb2b.so (once).  Raises ImportError -- never falls back -- when it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(nvcc, sm_90a).  bijectors.jl_b200 has no CPU fallback."
            )
        handle = ctypes.CDLL(LIB_PATH, mode=ctypes.RTLD_GLOBAL)
        for name, (res, args) in _SIGS.items():
            fn = getattr(handle, name)  # AttributeError if the library does not export a declared symbol
            fn.restype = res
            fn.argtypes = args
        _lib = handle
    return _lib


def exported_symbols():
    return sorted(_SIGS)


def check(status: int, where: str = "") -> None:
    if status != 0:
        raise B2BError(status, where)
