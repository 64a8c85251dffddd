"""ctypes binding of libgsplat_b200.so (the C ABI declared in include/gsplat_b200.h).

Every entry point's restype and argtypes are read from the header when this module is imported, so the prototypes
the compiler checks against the definitions are the only copy of the signatures.  The library is the only compute
path: if it cannot be loaded this module raises -- there is no PyTorch / CPU fallback (tests would otherwise pass on
a silent eager path).
"""
from __future__ import annotations

import ctypes
import os
import re
from typing import Optional

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libgsplat_b200.so")
HEADER_PATH = os.path.normpath(os.path.join(_HERE, os.pardir, "include", "gsplat_b200.h"))

_lib = None


class GsplatB200Error(RuntimeError):
    pass


class FThetaParams(ctypes.Structure):
    """gsb200_ftheta_params of include/gsplat_b200.h: the FTheta camera parameters of the 3DGUT entry points."""

    _fields_ = [
        ("reference_poly", ctypes.c_int),
        ("pixeldist_to_angle_poly", ctypes.c_float * 6),
        ("angle_to_pixeldist_poly", ctypes.c_float * 6),
        ("max_angle", ctypes.c_float),
        ("linear_cde", ctypes.c_float * 3),
    ]


# The C types the header passes by value.  Any pointer is passed as c_void_p; any other type is refused, so that a
# new one (a double, a uint16_t) cannot be bound as an integer of the wrong width.
_BY_VALUE = {
    "int64_t": ctypes.c_int64,
    "uint32_t": ctypes.c_uint32,
    "int": ctypes.c_int,
    "float": ctypes.c_float,
    "size_t": ctypes.c_size_t,
}
_PROTOTYPE = re.compile(r"^\s*((?:const\s+)?\w+\s*\*?)\s*(gsb200_\w+)\s*\(([^)]*)\)\s*;", re.M)


def _parse_header(text: str) -> dict:
    """{name: (restype, [argtypes])} of every gsb200_* prototype in the header text."""

    def ctype(decl: str, fn: str, what: str):
        if "*" in decl:
            return ctypes.c_void_p
        base = next((w for w in decl.split() if w != "const"), "")
        if base not in _BY_VALUE:
            raise GsplatB200Error(f"gsplat_b200.h: {fn}: {what} `{decl}` has a C type the binding does not map")
        return _BY_VALUE[base]

    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    out = {}
    for m in _PROTOTYPE.finditer(text):
        ret, name, params = m.group(1).strip(), m.group(2), m.group(3).strip()
        plist = [] if params in ("", "void") else [p.strip() for p in params.split(",")]
        res = ctypes.c_char_p if re.fullmatch(r"const\s+char\s*\*", ret) else ctype(ret, name, "return type")
        out[name] = (res, [ctype(p, name, "parameter") for p in plist])
    return out


def _read_header() -> str:
    try:
        with open(HEADER_PATH) as f:
            return f.read()
    except OSError as e:
        raise GsplatB200Error(f"{HEADER_PATH} cannot be read ({e.strerror}): the binding takes its signatures from it") from e


_SIGNATURES = _parse_header(_read_header())
EXPORTED_SYMBOLS = tuple(_SIGNATURES)


def lib():
    """The loaded library; raises if it has not been built (python -m gsplat_b200.build)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise GsplatB200Error(
                f"{LIB_PATH} is missing: build it with `python -m gsplat_b200.build` "
                "(nvcc, sm_90a). gsplat_b200 has no CPU / PyTorch fallback."
            )
        L = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in _SIGNATURES.items():
            fn = getattr(L, name)  # AttributeError if the .so does not export what the header declares
            fn.restype, fn.argtypes = res, args
        _lib = L
    return _lib


def check(rc: int, what: str) -> None:
    if rc == 0:
        return
    L = lib()
    msg = L.gsb200_error_string(rc).decode()
    if rc == -3:
        msg += ": " + L.gsb200_last_cuda_error().decode()
    text = f"{what}: {msg}"
    if rc in (-1, -2):
        raise ValueError(text)  # reference: TORCH_CHECK_VALUE -> ValueError
    raise GsplatB200Error(text)


def ptr(t: Optional[torch.Tensor]):
    return None if t is None else t.data_ptr()


def stream(device_index: Optional[int] = None) -> int:
    """Raw handle of torch's current stream on a device (default: the current device).  The private getter is the one
    torch's own code generators use; it skips the Stream object torch.cuda.current_stream() builds (3 us a call, a dozen
    calls per step)."""
    if device_index is None:
        device_index = torch._C._cuda_getDevice()
    return torch._C._cuda_getCurrentRawStream(device_index)


def require_cuda(*tensors: Optional[torch.Tensor]) -> torch.device:
    dev = None
    for t in tensors:
        if t is None:
            continue
        if not t.is_cuda:
            raise GsplatB200Error(
                "gsplat_b200 operators run only on CUDA tensors (sm_90a kernels; there is no CPU fallback)"
            )
        if dev is None:
            dev = t.device
        elif t.device != dev:
            raise ValueError("all tensors must be on the same CUDA device")
    if dev is None:
        raise ValueError("no tensor arguments")
    return dev


def f32c(t: Optional[torch.Tensor], name: str) -> Optional[torch.Tensor]:
    """contiguous float32 view/copy of t (the reference wrappers call .contiguous() too)."""
    if t is None:
        return None
    if t.dtype != torch.float32:
        raise TypeError(f"{name}: expected float32, got {t.dtype} (gsplat_b200 computes in fp32 only)")
    return t.contiguous()


def bits_for_count(count: int) -> int:
    return int(lib().gsb200_bits_for_count(int(count)))
