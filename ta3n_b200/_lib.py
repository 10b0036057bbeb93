"""ctypes binding of libta3n_sm90.so (the C ABI in include/ta3n_b200.h).

There is no CPU fallback: if the shared library is missing this module raises, and every
wrapper refuses tensors that are not CUDA fp32 contiguous.
"""
from __future__ import annotations

import ctypes as C
import os
import threading

from . import build as _build

ABI_VERSION = 5     # TA3N_ABI_VERSION of include/ta3n_b200.h that SIGNATURES mirrors

TA3N_GEMM_FP32_SIMT = 0
TA3N_GEMM_TF32_TCGEN05 = 1
TA3N_GEMM_TF32X3_TCGEN05 = 2


class RelationTable(C.Structure):
    _fields_ = [("num_frames", C.c_int), ("n_scales", C.c_int),
                ("scale_size", C.POINTER(C.c_int)), ("rel_count", C.POINTER(C.c_int)),
                ("frames", C.POINTER(C.c_int))]


class Dropout(C.Structure):
    _fields_ = [("p", C.c_float), ("keep", C.c_void_p), ("seed", C.c_uint64), ("step_dev", C.c_void_p)]


class StepDesc(C.Structure):
    """ta3n_step_desc of include/ta3n_b200.h (same field order)."""
    _fields_ = (
        [(n, C.c_int) for n in ("Bs", "Bt", "T", "D", "F", "H", "C", "use_attn", "loss_flags")] +
        [("gamma", C.c_float), ("domain_weight", C.c_float * 2), ("class_weight", C.c_void_p),
         ("beta_dev", C.c_void_p), ("tab", C.POINTER(RelationTable)),
         ("x_src", C.c_void_p), ("x_tgt", C.c_void_p), ("labels", C.c_void_p), ("valid_rows", C.c_void_p),
         ("drop_i", Dropout), ("drop_v", Dropout)] +
        [(n, C.c_void_p) for n in ("W_sh", "b_sh", "W1f", "b1f", "W2f", "b2f")] +
        [(n, C.POINTER(C.c_void_p)) for n in ("W_trn_host", "b_trn_host", "W1r_host", "b1r_host", "W2r_host",
                                              "b2r_host")] +
        [(n, C.c_void_p) for n in ("Wc", "bc", "W1v", "b1v", "W2v", "b2v")] +
        [(n, C.c_void_p) for n in ("dW_sh", "db_sh", "dW1f", "db1f", "dW2f", "db2f")] +
        [(n, C.POINTER(C.c_void_p)) for n in ("dW_trn_host", "db_trn_host", "dW1r_host", "db1r_host", "dW2r_host",
                                              "db2r_host")] +
        [(n, C.c_void_p) for n in ("dWc", "dbc", "dW1v", "db1v", "dW2v", "db2v")] +
        [(n, C.c_void_p) for n in ("feat", "hid_f", "pred_frame", "act", "feat_rel", "hid_r", "pred_rel", "attn",
                                   "feat_video", "dropped", "pred_video", "hid_v", "pred_dom", "loss",
                                   "step_counter", "workspace")] +
        [("workspace_bytes", C.c_size_t)])


_VP, _I, _F, _SZ = C.c_void_p, C.c_int, C.c_float, C.c_size_t
_IP = C.POINTER(C.c_int)
_PP = C.POINTER(C.c_void_p)
_TAB = C.POINTER(RelationTable)
_DRP = C.POINTER(Dropout)

# name -> (restype, argtypes); mirrors include/ta3n_b200.h one to one
SIGNATURES = {
    "ta3n_abi_version": (_I, []),
    "ta3n_last_error": (C.c_char_p, []),
    "ta3n_launch_count": (C.c_uint64, []),
    "ta3n_reset_launch_count": (None, []),
    "ta3n_set_gemm_engine": (_I, [_I]),
    "ta3n_get_gemm_engine": (_I, []),
    "ta3n_set_forward_scratch": (_I, [_VP, _SZ]),
    "ta3n_plan_forward_splits": (_I, [_I, _IP, _IP, _IP, _I, _SZ, _IP, C.POINTER(C.c_double)]),
    "ta3n_timing_enable": (None, [_I]),
    "ta3n_timing_report": (_SZ, [C.c_char_p, _SZ]),
    "ta3n_shared_fc_fwd": (_I, [_VP, _I, _VP, _I, _I, _VP, _VP, _I, _DRP, _VP, _VP]),
    "ta3n_shared_fc_bwd_workspace_bytes": (_SZ, [_I, _I, _I]),
    "ta3n_shared_fc_bwd": (_I, [_VP, _I, _VP, _I, _I, _I, _VP, _VP, _VP, _F, _VP, _VP, _VP, _SZ, _VP]),
    "ta3n_disc_fwd": (_I, [_VP, _I, _I, _I, _VP, _VP, _VP, _VP, _VP, _VP, _VP]),
    "ta3n_disc_bwd_workspace_bytes": (_SZ, [_I, _I, _I]),
    "ta3n_disc_bwd": (_I, [_VP, _I, _I, _I, _VP, _VP, _VP, _VP, _F, _VP, _I, _VP, _VP, _VP, _VP, _VP, _SZ, _VP]),
    "ta3n_grl_bwd": (_I, [_VP, _F, _VP, _SZ, _VP]),
    "ta3n_frame_attn_fwd": (_I, [_VP, _VP, _I, _I, _VP, _VP]),
    "ta3n_frame_attn_bwd": (_I, [_VP, _VP, _I, _I, _VP, _VP, _VP]),
    "ta3n_segment_mean_fwd": (_I, [_VP, _I, _I, _I, _VP, _VP]),
    "ta3n_segment_mean_bwd": (_I, [_VP, _I, _I, _I, _VP, _VP]),
    "ta3n_trn_fwd": (_I, [_VP, _I, _I, _I, _TAB, _PP, _PP, _I, _VP, _VP, _VP]),
    "ta3n_trn_bwd_workspace_bytes": (_SZ, [_I, _I, _I, _TAB]),
    "ta3n_trn_bwd": (_I, [_VP, _I, _I, _I, _TAB, _PP, _I, _VP, _VP, _PP, _PP, _VP, _I, _VP, _SZ, _VP]),
    "ta3n_relattn_fwd": (_I, [_VP, _I, _I, _I, _PP, _PP, _PP, _PP, _I, _VP, _VP, _VP, _VP, _VP]),
    "ta3n_relattn_bwd_workspace_bytes": (_SZ, [_I, _I, _I]),
    "ta3n_relattn_bwd": (_I, [_VP, _I, _I, _I, _PP, _PP, _I, _VP, _VP, _VP, _VP, _VP, _VP, _F, _VP,
                              _PP, _PP, _PP, _PP, _VP, _SZ, _VP]),
    "ta3n_general_attn_fwd": (_I, [_VP, _I, _I, _I, _VP, _VP, _VP, _VP, _VP, _VP, _VP, _VP]),
    "ta3n_general_attn_bwd_workspace_bytes": (_SZ, [_I, _I, _I]),
    "ta3n_general_attn_bwd": (_I, [_VP, _I, _I, _I, _VP, _VP, _VP, _VP, _VP, _VP, _VP, _VP, _VP, _VP, _VP, _VP, _SZ, _VP]),
    "ta3n_video_head_fwd": (_I, [_VP, _I, _I, _I, _VP, _VP, _DRP, _VP, _VP, _VP]),
    "ta3n_video_head_bwd_workspace_bytes": (_SZ, [_I, _I, _I]),
    "ta3n_video_head_bwd": (_I, [_VP, _I, _I, _I, _VP, _DRP, _VP, _VP, _VP, _F, _VP, _VP, _VP, _VP, _SZ, _VP]),
    "ta3n_fwd_batch_begin": (_I, []),
    "ta3n_fwd_batch_workspace_bytes": (_SZ, []),
    "ta3n_fwd_batch_flush": (_I, [_VP, _SZ, _VP]),
    "ta3n_wgrad_defer_begin": (_I, []),
    "ta3n_wgrad_defer_workspace_bytes": (_SZ, []),
    "ta3n_wgrad_defer_flush": (_I, [_VP, _SZ, _VP]),
    "ta3n_loss_workspace_bytes": (_SZ, [_I]),
    "ta3n_loss_fwd_bwd": (_I, [_VP, _VP, _VP, _VP, _VP, _I, _I, _I, _I, _I, _F, _I, _VP, _VP, _VP, _VP, _VP, _VP,
                               _VP, _SZ, _VP]),
    "ta3n_counter_inc": (_I, [_VP, _VP]),
    "ta3n_ce_loss_fwd_bwd": (_I, [_VP, _VP, _I, _I, _VP, _VP, _VP, _VP]),
    "ta3n_mcd_loss_fwd_bwd": (_I, [_VP, _VP, _I, _I, _VP, _VP, _VP, _VP, _VP, _VP]),
    "ta3n_accumulate": (_I, [_VP, _VP, C.c_longlong, _VP]),
    "ta3n_gather_batch": (_I, [_VP, C.c_longlong, _VP, _VP, C.c_longlong, _I, _VP, _VP,
                               _VP, C.c_longlong, _VP, C.c_longlong, _I, _VP, C.c_longlong, _VP, _VP, _VP]),
    "ta3n_gather_rows": (_I, [_VP, C.c_longlong, _VP, _VP, C.c_longlong, _I, _VP, _VP, C.c_longlong, _VP, _VP, _VP]),
    "ta3n_eval_workspace_bytes": (_SZ, [_I]),
    "ta3n_eval_head": (_I, [_VP, _I, _I, _I, _VP, _VP, _VP, _VP, _VP, _I, _IP, _VP, _I, C.c_longlong, _VP,
                            _VP, _VP, _VP, _VP, C.c_longlong, _VP, _SZ, _VP]),
    "ta3n_step_workspace_bytes": (_SZ, [C.POINTER(StepDesc)]),
    "ta3n_step_run_phased": (_I, [C.POINTER(StepDesc), _VP]),
    "ta3n_allreduce_flag_bytes": (_SZ, [_I]),
    "ta3n_allreduce_mean": (_I, [_PP, _VP, _PP, _VP, _I, _I, C.c_longlong, _VP]),
    "ta3n_sgd_workspace_bytes": (_SZ, []),
    "ta3n_sgd_nesterov_step": (_I, [_VP, _VP, _VP, C.c_longlong, _VP, _F, _F, _F, _VP, _SZ, _VP, _VP]),
    "ta3n_sgd_nesterov_step_masked": (_I, [_VP, _VP, _VP, C.c_longlong, _VP, _F, _F, _F, _VP, _SZ, _VP, _VP, _VP]),
    "ta3n_gemm_tn": (_I, [_VP, _VP, _VP, _I, _I, _I, _VP]),
    "ta3n_gemm_ex": (_I, [_VP, _I, _I, _VP, _I, _I, _VP, _I, _I, _I, _I, _VP, _SZ, _VP]),
}

_lock = threading.Lock()
_lib = None


class Ta3nError(RuntimeError):
    pass


def lib_path() -> str:
    return os.environ.get("TA3N_LIB", _build.LIB_PATH)


def load() -> C.CDLL:
    """Load the shared library (once).  Raises if it has not been built: no fallback."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is None:
            path = lib_path()
            if not os.path.exists(path):
                raise Ta3nError(
                    f"{path} is missing: build it with `python -m ta3n_b200.build` "
                    "(or __graft_entry__.build()). ta3n_b200 has no CPU / PyTorch fallback.")
            lib = C.CDLL(path)
            for name, (res, args) in SIGNATURES.items():
                fn = getattr(lib, name)   # AttributeError if the .so does not export the symbol
                fn.restype = res
                fn.argtypes = args
            if lib.ta3n_abi_version() != ABI_VERSION:
                raise Ta3nError("libta3n_sm90.so ABI version mismatch")
            _lib = lib
    return _lib


def check(rc: int) -> None:
    if rc != 0:
        msg = load().ta3n_last_error()
        raise Ta3nError(f"libta3n_sm90 error {rc}: {msg.decode() if msg else '?'}")


def ptr_array(ptrs):
    arr = (C.c_void_p * len(ptrs))(*ptrs)
    return arr


def set_gemm_engine(engine) -> None:
    """'tf32x3' (wgmma, error-compensated tf32: fp32-grade forward; the library default), 'tf32' (plain wgmma
    tf32) or 'fp32' (exact SIMT tiles)."""
    code = {"fp32": TA3N_GEMM_FP32_SIMT, "tf32": TA3N_GEMM_TF32_TCGEN05, "tf32x3": TA3N_GEMM_TF32X3_TCGEN05}.get(engine, engine)
    check(load().ta3n_set_gemm_engine(int(code)))


def get_gemm_engine() -> str:
    return {0: "fp32", 1: "tf32", 2: "tf32x3"}[load().ta3n_get_gemm_engine()]


def plan_forward_splits(shapes, sms: int = 132, scratch_bytes: int = 48 << 20):
    """Split-K factors the tf32x3 engine's balanced planner picks for one forward launch of GEMMs [(M, N, K), ...]
    (host-only, C ABI ta3n_plan_forward_splits).  Returns (ksplit list, unsplit makespan, chosen makespan)."""
    n = len(shapes)
    arr = lambda col: (C.c_int * n)(*[int(s[col]) for s in shapes])
    ks, span = (C.c_int * n)(), (C.c_double * 2)()
    check(load().ta3n_plan_forward_splits(n, arr(0), arr(1), arr(2), int(sms), int(scratch_bytes), ks, span))
    return list(ks), span[0], span[1]


def launch_count() -> int:
    return int(load().ta3n_launch_count())


def reset_launch_count() -> None:
    load().ta3n_reset_launch_count()


def timing_enable(on: bool) -> None:
    load().ta3n_timing_enable(int(bool(on)))


def timing_report() -> dict:
    """{label: (count, total_ms)} of the launches recorded since timing was enabled (synchronises)."""
    buf = C.create_string_buffer(1 << 16)
    load().ta3n_timing_report(buf, len(buf))
    out = {}
    for line in buf.value.decode().splitlines():
        label, count, ms = line.split()
        out[label] = (int(count), float(ms))
    return out
