"""ctypes binding of libhb200.so (the C ABI declared in include/hb200.h).

There is no fallback: if the shared library is missing or a call fails, this raises.
"""
from __future__ import annotations

import ctypes
import os
from typing import Optional

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libhb200.so")

_C = {
    "p": ctypes.c_void_p,
    "i": ctypes.c_int,
    "l": ctypes.c_longlong,
    "f": ctypes.c_float,
    "d": ctypes.c_double,
    "z": ctypes.c_size_t,
    "s": ctypes.c_char_p,
}

# name -> (restype code, argtype codes); mirrors include/hb200.h one to one
SIGNATURES = {
    "hb200_last_error": ("s", ""),
    "hb200_version": ("i", ""),
    "hb200_launch_count": ("l", ""),
    "hb200_gae_adv": ("i", "ppppppp" + "iii" + "ff" + "ii" + "p"),
    "hb200_ver_gae": ("i", "ppppp" + "iii" + "dd" + "i" + "pp" + "i" + "p"),
    "hb200_adv_normalize": ("i", "plppip"),
    "hb200_ppo_loss_workspace_bytes": ("z", "iii"),
    "hb200_ppo_loss": ("i", "ppppppppppp" + "iii" + "fff" + "ii" + "ppp" + "ppppp" + "ppp"),
    "hb200_gaussian_act": ("i", "ppppppp" + "iiii" + "ff" + "ppp" + "p"),
    "hb200_gaussian_ppo_loss_workspace_bytes": ("z", "iii"),
    "hb200_gaussian_ppo_loss": ("i", "pppppp" + "pppppp" + "iiii" + "ff" + "fff" + "ii" + "ppp" + "pppppp" + "pp" + "p"),
    "hb200_clip_adam_workspace_bytes": ("z", "l"),
    "hb200_grad_sqnorm": ("i", "plfppp"),
    "hb200_clip_adam": ("i", "pppp" + "l" + "fffffff" + "l" + "pppp"),
    "hb200_prep_stats": ("i", "ppp" + "iiiii" + "f" + "pp"),
    "hb200_prep_finalize": ("i", "ppppp" + "ili" + "p"),
    "hb200_prep_apply": ("i", "ppp" + "iiiii" + "f" + "ppp" + "i" + "p"),
    "hb200_conv_fwd": ("i", "pppp" + "i" + "pp"),
    "hb200_conv_bias_act_fwd": ("i", "pppp" + "i" + "pp"),
    "hb200_prep_plain": ("i", "ppp" + "iiiii" + "pp"),
    "hb200_relu_bias_bwd": ("i", "pppp" + "li" + "p"),
    "hb200_bf16_hwc_to_f32_chw": ("i", "pp" + "iii" + "p"),
    "hb200_conv_dgrad": ("i", "pppppp"),
    "hb200_conv_wgrad": ("i", "ppppp"),
    "hb200_pack_conv_weight": ("i", "ppp" + "iiiii" + "p"),
    "hb200_unpack_conv_wgrad": ("i", "pp" + "iiiii" + "p"),
    "hb200_packed_weight_elems": ("z", "iiii"),
    "hb200_conv_s2_supported": ("i", "iiiii"),
    "hb200_conv_s2_wgrad_supported": ("i", "iiii"),
    "hb200_conv_s2_wgrad": ("i", "ppp" + "iiiii" + "p"),
    "hb200_unpack_s2_wgrad": ("i", "pp" + "ii" + "p"),
    "hb200_conv_s2_fwd": ("i", "pppp" + "pipi" + "iiiiii" + "p"),
    "hb200_conv_s2_dgrad": ("i", "ppppp" + "iiiiii" + "p"),
    "hb200_conv_halo_supported": ("i", "iiiii"),
    "hb200_conv_halo_wgrad_supported": ("i", "iiiii"),
    "hb200_pack_halo_weight": ("i", "pp" + "iiiiii" + "p"),
    "hb200_conv_halo": ("i", "ppppp" + "iiiiiiii" + "p"),
    "hb200_conv_halo_wgrad": ("i", "ppp" + "iiiiii" + "p"),
    "hb200_unpack_stem_wgrad": ("i", "pp" + "ii" + "p"),
    "hb200_umma_gemm_probe": ("i", "ppp" + "iiii" + "p"),
    "hb200_gn_apply": ("i", "pppppp" + "iiiii" + "f" + "i" + "p"),
    "hb200_gn_residual_relu": ("i", "pppppppppp" + "iiii" + "f" + "p"),
    "hb200_gn_relu_maxpool": ("i", "ppppppp" + "iiiii" + "f" + "p"),
    "hb200_maxpool_bwd": ("i", "ppp" + "iiii" + "p"),
    "hb200_gn_bwd_reduce": ("i", "ppppppppp" + "iiii" + "f" + "i" + "p"),
    "hb200_gn_bwd_apply": ("i", "ppppppppp" + "iiii" + "f" + "i" + "p"),
    "hb200_gn_bwd": ("i", "pppppppppp" + "iiii" + "f" + "i" + "p"),
    "hb200_gn_se_residual_relu": ("i", "pppppppp" + "pppp" + "ppppp" + "iiiii" + "f" + "p"),
    "hb200_gn_se_bwd": ("i", "pppppppppp" + "pppppp" + "iiiii" + "f" + "p"),
    "hb200_tma_halo_probe": ("i", "pp" + "iiiiiiiiii" + "p"),
    "hb200_gn_relu_maxpool_bwd_supported": ("i", "iiii"),
    "hb200_gn_relu_maxpool_bwd": ("i", "ppppppppp" + "iiiii" + "f" + "p"),
    "hb200_sgemm": ("i", "pll" + "pll" + "pl" + "p" + "iii" + "f" + "ii" + "p"),
    "hb200_tgemm": ("i", "pll" + "pll" + "pl" + "p" + "iii" + "ii" + "p"),
    "hb200_transpose_f32": ("i", "plpl" + "ii" + "p"),
    "hb200_f16_to_bf16": ("i", "pplp"),
    "hb200_bf16_to_f32": ("i", "pplp"),
    "hb200_f32_to_bf16": ("i", "pplp"),
    "hb200_lstm_step_fwd": ("i", "ppppplplppp" + "ii" + "p"),
    "hb200_lstm_step_bwd": ("i", "ppppppl" + "ppppp" + "ii" + "p"),
    "hb200_lstm_seq_fwd": ("i", "ppppplplppp" + "iii" + "pp"),
    "hb200_lstm_seq_bwd": ("i", "pppplppp" + "iii" + "pp"),
    "hb200_lstm_seq_bwd_chunk": ("i", "pppplppp" + "iii" + "pp" + "ii" + "p"),
    "hb200_gru_seq_fwd": ("i", "ppppplpp" + "iii" + "pp"),
    "hb200_gru_seq_bwd": ("i", "pppplpppp" + "iii" + "pp"),
    "hb200_rnn_shift_mask": ("i", "pplpp" + "iii" + "p"),
    "hb200_colsum": ("i", "plplii" + "p"),
    "hb200_relu_bwd": ("i", "pplll" + "i" + "p"),
    "hb200_gather_rows": ("i", "pppil" + "p"),
    "hb200_gather_rows_pad": ("i", "plppl" + "ii" + "p"),
    "hb200_f32_chw_to_bf16_hwc": ("i", "pp" + "iii" + "p"),
    "hb200_heads_fwd": ("i", "ppppp" + "iii" + "pp" + "p"),
    "hb200_heads_act": ("i", "pppppp" + "iii" + "pppp" + "p"),
    "hb200_embed_fwd": ("i", "pppppppp" + "iii" + "p"),
    "hb200_embed_bwd": ("i", "ppppp" + "iiii" + "ppp" + "p"),
    "hb200_sensor_linear_fwd": ("i", "pipii" + "ppp" + "iii" + "p"),
    "hb200_sensor_linear_bwd": ("i", "pipii" + "p" + "iii" + "pp" + "p"),
    "hb200_index_embed_fwd": ("i", "pppii" + "pip" + "ii" + "p"),
    "hb200_index_embed_bwd": ("i", "pppiii" + "p" + "ii" + "p" + "p"),
    "hb200_prev_action_linear_fwd": ("i", "ppii" + "ppp" + "ii" + "p"),
    "hb200_prev_action_linear_bwd": ("i", "ppii" + "p" + "ii" + "pp" + "p"),
    "hb200_prep_generic": ("i", "pppp" + "i" + "p" + "iii" + "pppp" + "p"),
    "hb200_obs_resample": ("i", "ppp" + "ii" + "p"),
    "hb200_obs_project": ("i", "pppppp" + "ii" + "p"),
}


class Hb200Error(RuntimeError):
    pass


class ConvShape(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int) for n in
                ("batch", "hi", "wi", "ci", "ho", "wo", "co", "kh", "kw", "stride", "pad")]


_lib: Optional[ctypes.CDLL] = None


def load() -> ctypes.CDLL:
    """Load libhb200.so, declaring every prototype.  Raises if it is not built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise Hb200Error(
            f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(there is no CPU / PyTorch fallback for the hot path)"
        )
    lib = ctypes.CDLL(LIB_PATH)
    missing = []
    for name, (res, args) in SIGNATURES.items():
        try:
            fn = getattr(lib, name)
        except AttributeError:
            missing.append(name)
            continue
        fn.restype = _C[res]
        fn.argtypes = [_C[c] for c in args]
    if missing:
        raise Hb200Error(f"{LIB_PATH} lacks symbols declared in include/hb200.h: {missing}")
    _lib = lib
    return lib


def exported_symbols():
    return sorted(SIGNATURES)


def ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    if t is None:
        return None
    return t.data_ptr()


def stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def check(rc: int, what: str = "") -> None:
    if rc != 0:
        msg = load().hb200_last_error().decode("utf-8", "replace")
        raise Hb200Error(f"{what} failed (rc={rc}): {msg}")


def call(name: str, *args) -> None:
    """Invoke an int-returning entry point, appending the current CUDA stream."""
    lib = load()
    rc = getattr(lib, name)(*args, stream())
    check(rc, name)
