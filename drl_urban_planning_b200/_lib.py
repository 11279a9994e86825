"""ctypes binding of libupb200.so (include/upb200.h).  There is no CPU fallback: if the library is missing
or a call fails, this raises."""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

HERE = os.path.dirname(os.path.abspath(__file__))
# UPB_LIB selects another build of the same ABI (bench.py --tiles bf16 -> libupb200_bf16.so, the labelled non-parity variant)
LIB_PATH = os.environ.get("UPB_LIB") or os.path.join(HERE, "libupb200.so")

UPB_NUM_PARAMS = 13729
UPB_GRAD_STRIDE = 13760
UPB_STAT_OFFSET = 13732
UPB_STAT_COUNT = 28

UPB_MLP_NUM_PARAMS = 10257           # rl-mlp ablation model (include/upb200.h)
UPB_MLP_GRAD_STRIDE = 10288
UPB_MLP_STAT_OFFSET = 10260

CLIP_REFERENCE, CLIP_ALWAYS, CLIP_NEVER = 0, 1, 2


class UpbError(RuntimeError):
    pass


class Config(C.Structure):
    _fields_ = [
        ("device", C.c_int32), ("n_cap", C.c_int32), ("e_cap", C.c_int32), ("max_graphs", C.c_int32),
        ("lr", C.c_float), ("beta1", C.c_float), ("beta2", C.c_float), ("adam_eps", C.c_float),
        ("clip_epsilon", C.c_float), ("value_pred_coef", C.c_float), ("entropy_coef", C.c_float),
        ("clip_mode", C.c_int32), ("grid_limit", C.c_int32),
    ]


_lib: Optional[C.CDLL] = None

_VP = C.c_void_p
_PROTOS = {
    "upb_abi_version": (C.c_int, []),
    "upb_last_error": (C.c_char_p, []),
    "upb_num_params": (C.c_int, []),
    "upb_param_slot": (C.c_int, [C.c_int, C.POINTER(C.c_char_p), C.POINTER(C.c_int), C.POINTER(C.c_int),
                                 C.POINTER(C.c_int)]),
    "upb_pack_measure": (C.c_int, [C.c_int, _VP, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_uint64)]),
    "upb_pack_fill": (C.c_int, [C.c_int, _VP, C.c_int, C.c_int, C.c_int, _VP, C.c_uint64]),
    "upb_pack_plan_create": (C.c_int, [C.c_int, _VP, C.c_int, C.c_int, C.c_int, C.POINTER(_VP), C.POINTER(C.c_uint64)]),
    "upb_pack_plan_fill": (C.c_int, [_VP, _VP, C.c_int, C.c_int, C.c_int, _VP, C.c_uint64, _VP]),
    "upb_pack_plan_destroy": (None, [_VP]),
    "upb_blob_info": (C.c_int, [_VP, C.c_uint64, C.POINTER(C.c_int), _VP]),
    "upb_create": (C.c_int, [C.POINTER(Config), C.POINTER(_VP)]),
    "upb_destroy": (None, [_VP]),
    "upb_forward": (C.c_int, [_VP, _VP, _VP, C.c_int, _VP, _VP, _VP, _VP, _VP, _VP, _VP]),
    "upb_ppo_grad": (C.c_int, [_VP, _VP, _VP, C.c_int, _VP, _VP, _VP, _VP, _VP, _VP, C.c_float, C.c_float,
                               _VP, _VP]),
    "upb_apply": (C.c_int, [_VP, _VP, _VP, _VP]),
    "upb_ppo_step": (C.c_int, [_VP, _VP, _VP, C.c_int, _VP, _VP, _VP, _VP, _VP, _VP, C.c_float, C.c_float,
                               _VP, _VP]),
    "upb_read_losses": (C.c_int, [_VP, _VP, C.POINTER(C.c_float), _VP]),
    "upb_gae": (C.c_int, [_VP, _VP, _VP, _VP, C.c_int, C.c_float, C.c_float, _VP, _VP, _VP]),
    "upb_get_opt_state": (C.c_int, [_VP, _VP, _VP, _VP]),
    "upb_set_opt_state": (C.c_int, [_VP, _VP, _VP, _VP]),
    "upb_rearm_clip": (C.c_int, [_VP]),
    "upb_profile_enable": (C.c_int, [_VP, C.c_int]),
    "upb_profile_read": (C.c_int, [_VP, C.POINTER(C.c_double), C.POINTER(C.c_int)]),
    "upb_grid_size": (C.c_int, [_VP]),
    "upb_set_stamp_buffer": (C.c_int, [_VP, _VP]),
    "upb_launch_count": (C.c_int64, [_VP]),
    "upb_select_action": (C.c_int, [_VP, _VP, _VP, C.c_int, _VP, _VP, _VP, _VP]),
    "upb_mlp_forward": (C.c_int, [_VP, _VP, _VP, C.c_int, _VP, _VP, _VP, _VP, _VP, _VP, _VP]),
    "upb_mlp_select_action": (C.c_int, [_VP, _VP, _VP, C.c_int, _VP, _VP, _VP, _VP]),
    "upb_mlp_ppo_grad": (C.c_int, [_VP, _VP, _VP, C.c_int, _VP, _VP, _VP, _VP, _VP, _VP, C.c_float, C.c_float,
                                   _VP, _VP]),
    "upb_mlp_apply": (C.c_int, [_VP, _VP, _VP, _VP]),
    "upb_mlp_ppo_step": (C.c_int, [_VP, _VP, _VP, C.c_int, _VP, _VP, _VP, _VP, _VP, _VP, C.c_float, C.c_float,
                                   _VP, _VP]),
    "upb_mlp_next_step_fused": (C.c_int, [_VP]),
    "upb_mlp_rearm_clip": (C.c_int, [_VP]),
    "upb_mlp_read_losses": (C.c_int, [_VP, _VP, C.POINTER(C.c_float), _VP]),
    "upb_mlp_get_opt_state": (C.c_int, [_VP, _VP, _VP, _VP]),
    "upb_mlp_set_opt_state": (C.c_int, [_VP, _VP, _VP, _VP]),
    "upb_peer_export": (C.c_int, [_VP, _VP]),
    "upb_peer_connect": (C.c_int, [_VP, C.c_int, C.c_int, _VP]),
    "upb_next_step_fused": (C.c_int, [_VP]),
    "upb_peer_timeouts": (C.c_int, [_VP, C.POINTER(C.c_int64)]),
}
EXPORTED_SYMBOLS = tuple(_PROTOS)
UPB_PEER_HANDLE_BYTES = 64


def lib() -> C.CDLL:
    """The loaded library; raises UpbError with build instructions if it does not exist."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise UpbError(
                f"{LIB_PATH} not found: build it with `python -m drl_urban_planning_b200.build` "
                "(nvcc, sm_90a).  There is no CPU fallback for the update path.")
        handle = C.CDLL(LIB_PATH)
        for name, (res, args) in _PROTOS.items():
            fn = getattr(handle, name)
            fn.restype = res
            fn.argtypes = args
        if handle.upb_abi_version() != 1:
            raise UpbError("libupb200.so ABI version mismatch; rebuild")
        _lib = handle
    return _lib


def check(rc: int, what: str = "") -> None:
    if rc != 0:
        msg = lib().upb_last_error()
        raise UpbError(f"{what or 'upb call'} failed ({rc}): {msg.decode() if msg else '?'}")


def param_slots():
    """[(name, offset, rows, cols)] as the C side sees the flat parameter vector."""
    out = []
    L = lib()
    i = 0
    while True:
        name, off, rows, cols = C.c_char_p(), C.c_int(), C.c_int(), C.c_int()
        if L.upb_param_slot(i, C.byref(name), C.byref(off), C.byref(rows), C.byref(cols)) != 0:
            break
        out.append((name.value.decode(), off.value, rows.value, cols.value))
        i += 1
    return out
