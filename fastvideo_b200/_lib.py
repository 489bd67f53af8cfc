"""ctypes binding of libfvb200.so (the C ABI declared in include/fvb200.h).

There is deliberately no fallback: if the library is missing or a call fails, we raise.
"""
from __future__ import annotations

import ctypes
from ctypes import c_int, c_int64, c_void_p, c_char_p, c_float, POINTER
from pathlib import Path

_PKG = Path(__file__).resolve().parent
LIB_PATH = _PKG / "libfvb200.so"


class FvbError(RuntimeError):
    pass


_lib = None


def lib() -> ctypes.CDLL:
    global _lib
    if _lib is None:
        if not LIB_PATH.exists():
            raise FvbError(f"{LIB_PATH} is missing: run `python -m fastvideo_b200.build` "
                           "(there is no CPU/eager fallback for the CUDA path)")
        _lib = ctypes.CDLL(str(LIB_PATH))
        _lib.fvb_last_error.restype = c_char_p
        _lib.fvb_abi_version.restype = c_int
        _lib.fvb_attention_blocklist_workspace_bytes.restype = c_int64
    return _lib


LAUNCHES = 0  # kernels launched through the C ABI by this process (every fvb_* compute call launches one)


def check(code: int) -> None:
    global LAUNCHES
    LAUNCHES += 1
    if code != 0:
        msg = lib().fvb_last_error().decode(errors="replace")
        raise FvbError(f"libfvb200 error {code}: {msg}")


def ptr(t) -> c_void_p:
    """Device (or host) pointer of a torch tensor, or NULL for None."""
    return c_void_p(0 if t is None else t.data_ptr())


def stream_ptr() -> c_void_p:
    import torch
    return c_void_p(torch.cuda.current_stream().cuda_stream)
