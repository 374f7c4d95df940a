"""ctypes binding of libsurya_b200.so.

The product path has NO fallback: if the library is missing, or the process has no CUDA device when a kernel
is requested, we raise.  (`load(require_cuda=False)` exists so CPU-only tests can check that the library
loads and exports every symbol that include/surya_b200.h declares.)
"""
from __future__ import annotations

import ctypes
import re
from ctypes import c_char_p, c_float, c_int, c_longlong, c_void_p
from pathlib import Path

_PKG = Path(__file__).resolve().parent
_LIB_PATH = _PKG / "lib" / "libsurya_b200.so"
_HEADER = _PKG.parent / "include" / "surya_b200.h"
_lib = None


class SuryaB200Error(RuntimeError):
    pass


def header_symbols() -> list[str]:
    """Function names declared in include/surya_b200.h."""
    text = _HEADER.read_text()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(sb_[a-z0-9_]+)\s*\(", text)))


def lib_path() -> Path:
    return _LIB_PATH


def load(require_cuda: bool = True) -> ctypes.CDLL:
    global _lib
    if _lib is None:
        if not _LIB_PATH.exists():
            raise SuryaB200Error(
                f"{_LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                "(surya_b200 has no CPU or PyTorch fallback path)"
            )
        lib = ctypes.CDLL(str(_LIB_PATH))
        lib.sb_last_error.restype = c_char_p
        lib.sb_launch_count.restype = c_longlong
        _lib = lib
    if require_cuda:
        import torch

        if not torch.cuda.is_available():
            raise SuryaB200Error("surya_b200 kernels need a CUDA device (sm_90a); none is visible")
    return _lib


def check(rc: int, what: str = "") -> None:
    if rc != 0:
        msg = load(False).sb_last_error()
        raise SuryaB200Error(f"{what} failed rc={rc}: {msg.decode() if msg else ''}")


def launch_count() -> int:
    return int(load(False).sb_launch_count())


def ptr(t) -> c_void_p:
    """Device (or host) pointer of a torch tensor / None."""
    if t is None:
        return c_void_p(0)
    return c_void_p(t.data_ptr())


def stream_ptr() -> c_void_p:
    import torch

    return c_void_p(torch.cuda.current_stream().cuda_stream)


__all__ = [
    "SuryaB200Error", "load", "check", "ptr", "stream_ptr", "launch_count", "header_symbols", "lib_path",
    "c_int", "c_float", "c_void_p", "c_longlong",
]
