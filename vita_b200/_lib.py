"""ctypes binding of libvita_b200.so (the C ABI declared in include/vita_b200.h).

There is deliberately no fallback: if the shared library is missing or a launch fails, the call raises.
"""
from __future__ import annotations

import ctypes
import os
from ctypes import c_char_p, c_float, c_int, c_int64, c_void_p
from pathlib import Path

_PKG = Path(__file__).resolve().parent
LIB_PATH = _PKG / "lib" / "libvita_b200.so"

P = c_void_p
I64 = c_int64

# name -> (restype, argtypes); mirrors include/vita_b200.h one to one.
SIGNATURES = {
    "vita_version": (c_int, []),
    "vita_last_error": (c_char_p, []),
    "vita_num_sms": (c_int, []),
    "vita_launch_count": (I64, [c_int]),
    "vita_set_option": (c_int, [ctypes.c_char_p, I64]),
    "vita_get_option": (I64, [ctypes.c_char_p]),
    "vita_gemm_bf16": (c_int, [P, I64, P, P, I64, I64, I64, I64, P, c_int, P, P, I64, P]),
    "vita_rmsnorm": (c_int, [P, P, P, I64, I64, c_float, P]),
    "vita_layernorm": (c_int, [P, P, P, P, I64, I64, c_float, c_int, c_float, P]),
    "vita_row_copy": (c_int, [P, P, P, P, I64, I64, P]),
    "vita_rope_kv_write": (c_int, [P, P, P, P, P, P, I64, I64, I64, I64, P]),
    "vita_gemm_qkv_rope": (c_int, [P, I64, P, P, I64, I64, I64, I64, I64, P, P, P, P, P, P]),
    "vita_gemm_qkv_rope_fp8": (c_int, [P, I64, P, P, I64, I64, I64, I64, I64, P, P, P, P, P, c_float, c_float, P]),
    "vita_attention_fwd": (c_int, [P, P, P, P, P, P, P, P, I64, I64, I64, I64, I64, I64, I64, P, c_int, I64, c_float, P]),
    "vita_attention_prefill_paged": (c_int, [P, I64, P, P, I64, P, I64, P, P, P, I64, P, I64, I64, I64, I64, I64, I64,
                                             c_float, P]),
    "vita_kv_fp8_stage_pages": (c_int, [P, P, P, I64, P, P, I64, P, P, I64, I64, I64, c_float, c_float, P]),
    "vita_decode_attention_workspace_bytes": (I64, [I64, I64, I64]),
    "vita_decode_attention_merge": (c_int, [I64, I64, I64]),
    "vita_decode_attention": (c_int, [P, P, P, P, P, P, P, I64, I64, I64, I64, I64, I64, I64, c_float, I64, P]),
    "vita_decode_attention_fp8": (c_int, [P, P, P, P, P, P, P, I64, I64, I64, I64, I64, I64, I64, c_float, I64,
                                          c_float, c_float, P]),
    "vita_decode_slots": (c_int, [P, P, P, I64, I64, I64, P]),
    "vita_argmax_rows": (c_int, [P, P, I64, I64, P]),
    "vita_sample_rows": (c_int, [P, I64, I64, I64, P, P, P, P, P, P, P, I64, I64, P]),
    "vita_sample_rows_logprobs": (c_int, [P, I64, I64, I64, P, P, P, P, P, P, P, P, I64, I64, P, P, P, P, I64, I64,
                                          I64, P]),
    "vita_sample_rows_logsoftmax": (c_int, [P, I64, I64, I64, P, P, P, P, P, P, P, P, I64, I64, P, P, P, P, I64, I64,
                                            I64, P]),
    "vita_sample_rows_streams": (c_int, [P, I64, I64, I64, P, P, P, P, P, P, P, P, P, I64, I64, P, P, P, P, I64, I64,
                                         I64, I64, P]),
    "vita_kv_copy_pages": (c_int, [P, I64, P, I64, I64, I64, P]),
    "vita_page_digest": (c_int, [P, I64, I64, I64, I64, P, P]),
    "vita_moe_router": (c_int, [P, P, P, P, P, P, I64, I64, I64, c_float, P]),
    "vita_moe_align": (c_int, [P, P, P, P, P, P, P, I64, I64, P]),
    "vita_moe_gemm_down_ep": (c_int, [P, P, P, P, P, P, I64, I64, I64, I64, I64, P]),
    "vita_ep_signal": (c_int, [P, I64, I64, I64, I64, P]),
    "vita_ep_wait": (c_int, [P, I64, I64, I64, I64, P]),
    "vita_ep_push": (c_int, [P, P, P, I64, I64, I64, P]),
    "vita_ep_reduce_norm_gather": (c_int, [P, P, P, P, P, I64, I64, I64, I64, I64, I64, c_float, I64, P]),
    "vita_moe_gemm_gate_up_silu": (c_int, [P, P, P, P, I64, I64, I64, I64, P]),
    "vita_moe_gemm_down": (c_int, [P, P, P, P, P, I64, I64, I64, I64, P]),
    "vita_moe_combine": (c_int, [P, P, P, P, P, I64, I64, c_float, P]),
    "vita_moe_route_scatter": (c_int, [P, P, P, P, P, P, P, P, P, I64, I64, I64, I64, c_float, P]),
    "vita_moe_gemm_gate_up_silu_slots": (c_int, [P, P, P, P, I64, I64, I64, I64, I64, P]),
    "vita_moe_gemm_down_slots": (c_int, [P, P, P, P, P, I64, I64, I64, I64, I64, P]),
    "vita_vit_im2col": (c_int, [P, P, I64, I64, I64, I64, I64, P]),
    "vita_vit_assemble": (c_int, [P, P, P, P, I64, I64, I64, P]),
    "vita_vit_pixel_shuffle": (c_int, [P, P, I64, I64, I64, c_float, P]),
    "vita_image_resample_u8": (c_int, [P, P, I64, I64, I64, c_int, I64, P, P, I64, P]),
    "vita_image_tiles_lut": (c_int, [P, P, P, I64, I64, I64, I64, P]),
    "vita_fbank": (c_int, [P, I64, P, P, P, P, I64, I64, I64, c_float, P]),
    "vita_whale_conv1": (c_int, [P, P, P, P, P, P, I64, I64, I64, I64, P]),
    "vita_whale_im2col2": (c_int, [P, P, I64, I64, I64, I64, P]),
    "vita_whale_qk_prep": (c_int, [P, P, P, P, P, P, I64, I64, I64, I64, P]),
    "vita_whale_adapter_im2col": (c_int, [P, P, P, I64, I64, I64, I64, P]),
    "vita_decode_embed": (c_int, [P, P, P, I64, P, P, P, P, I64, I64, I64, I64, P, P]),
    "vita_chain_begin": (c_int, [P, I64]),
    "vita_chain_end": (c_int, []),
    "vita_decode_router": (c_int, [P, P, P, P, P, P, I64, I64, I64, c_float, P]),
    "vita_decode_tc_workspace_bytes": (I64, [I64, I64]),
    "vita_decode_tc_qkv_rope": (c_int, [P, P, P, P, P, P, P, P, P, P, I64, I64, I64, I64, I64, I64, I64, I64, c_float, P]),
    "vita_decode_tc_qkv_rope_fp8": (c_int, [P, P, P, P, P, P, P, P, P, P, I64, I64, I64, I64, I64, I64, I64, I64,
                                            c_float, c_float, c_float, P]),
    "vita_decode_tc_oproj": (c_int, [P, P, P, P, I64, I64, I64, I64, P]),
    "vita_decode_tc_moe_gate_up": (c_int, [P, P, P, P, P, P, P, P, I64, I64, I64, I64, I64, c_float, P, I64, P]),
    "vita_decode_tc_moe_down": (c_int, [P, P, P, P, P, P, I64, I64, I64, I64, I64, P, I64, P]),
    "vita_tc_lm_head_argmax": (c_int, [P, I64, P, P, P, P, P, I64, I64, I64, I64, c_float, P]),
}


class VitaB200Error(RuntimeError):
    pass


_lib = None


def load() -> ctypes.CDLL:
    """dlopen the library and attach the prototypes.  Raises if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    path = Path(os.environ.get("VITA_B200_LIB", LIB_PATH))
    if not path.exists():
        raise VitaB200Error(
            f"{path} not found: build it with `python -m vita_b200.build` (nvcc, sm_90a). "
            "There is no CPU or PyTorch fallback for the vita_b200 kernels.")
    lib = ctypes.CDLL(str(path))
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is missing
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def call(name: str, *args) -> None:
    """Call an int-returning entry point and raise on a non-zero status."""
    lib = load()
    rc = getattr(lib, name)(*args)
    if rc != 0:
        msg = lib.vita_last_error()
        raise VitaB200Error(f"{name} failed (code {rc}): {msg.decode() if msg else ''}")
