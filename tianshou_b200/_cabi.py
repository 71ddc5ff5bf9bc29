"""ctypes binding of ``libts_b200.so`` (the C ABI declared in ``include/ts_b200.h``).

The library is the product: if it cannot be loaded, every device entry point raises -- there is
no CPU fallback (the numpy/C oracle under ``oracle/`` is test infrastructure and is never imported
from here).  torch is used only as plumbing: device memory, the current CUDA stream.
"""
from __future__ import annotations

import ctypes as C
import os
import re
from typing import Any, NamedTuple

import numpy as np
import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libts_b200.so")
HEADER_PATH = os.path.join(os.path.dirname(_HERE), "include", "ts_b200.h")


class ExtensionMissingError(RuntimeError):
    pass


class HeaderError(ValueError):
    """A declaration of the C header that the binding has no rule for."""


# The header is the only definition of the ABI: every prototype, struct layout and TS_* constant below is parsed from it.
# Scalars and ts_stream_t bind by name; a pointer to a header struct binds as POINTER(struct), T** and void* const* as
# POINTER(c_void_p), every other pointer as c_void_p (const char* returns as c_char_p).  Any other type raises, so a
# header edit never binds silently as something else.
_SCALARS = {"int": C.c_int, "int32_t": C.c_int32, "int64_t": C.c_int64, "uint64_t": C.c_uint64, "size_t": C.c_size_t,
            "double": C.c_double, "float": C.c_float, "ts_stream_t": C.c_void_p}


class Abi(NamedTuple):
    functions: dict[str, tuple[Any, list[Any]]]       # name -> (restype, argtypes) of the product library
    diag_functions: dict[str, tuple[Any, list[Any]]]  # the `#ifdef TS_B200_DIAGNOSTICS` block (libts_b200_diag.so)
    structs: dict[str, type[C.Structure]]             # typedef name -> layout
    consts: dict[str, int]                            # every `#define TS_* <int>` and `enum { TS_* = <int> }`


def _ctype(decl: str, structs: dict[str, type[C.Structure]], where: str, ret: bool = False) -> Any:
    """ctypes type of one parameter or struct member (type and name) or, with ``ret``, of a return type."""
    tokens = [t for t in re.findall(r"\w+|\*", decl) if t != "const"]
    names, stars = [t for t in tokens if t != "*"], tokens.count("*")
    if not ret and len(names) > 1:
        names.pop()                                   # the parameter's name
    if len(names) == 1:
        base = names[0]
        if stars == 0 and base in _SCALARS:
            return _SCALARS[base]
        if stars == 0 and ret and base == "void":
            return None
        if stars == 1 and base in structs:
            return C.POINTER(structs[base])
        if stars == 1 and ret and base == "char":
            return C.c_char_p
        if stars == 1:
            return C.c_void_p
        if stars == 2:
            return C.POINTER(C.c_void_p)
    raise HeaderError(f"no ctypes rule for {decl.strip()!r} in: {' '.join(where.split())}")


def _functions(text: str, structs: dict[str, type[C.Structure]]) -> dict[str, tuple[Any, list[Any]]]:
    text = re.sub(r"^\s*#.*$", "", text, flags=re.M)      # preprocessor lines
    decl = re.compile(r"([A-Za-z_][\w\s*]*?)\b(ts_\w+)\s*\(([^()]*)\)\s*;")
    out = {}
    for m in decl.finditer(text):
        ret, name, params = m.groups()
        args = [] if params.strip() in ("", "void") else [_ctype(p, structs, m[0]) for p in params.split(",")]
        out[name] = (_ctype(ret, structs, m[0], ret=True), args)
    unread = re.search(r"[^;{}]*\bts_\w+\s*\([^;]*;?", decl.sub("", text))
    if unread:
        raise HeaderError(f"cannot read the declaration {' '.join(unread[0].split())!r}")
    return out


def parse_header(text: str) -> Abi:
    """The ABI declared by C header text in the dialect of include/ts_b200.h (no library needed)."""
    text = re.sub(r"/\*.*?\*/|//[^\n]*", " ", text, flags=re.S)
    consts = {k: int(v) for k, v in re.findall(r"^\s*#define\s+(TS_\w+)\s+(-?\d+)\s*$", text, flags=re.M)}
    for body in re.findall(r"\benum\s*\{(.*?)\}", text, flags=re.S):
        consts.update((k, int(v)) for k, v in re.findall(r"\b(TS_\w+)\s*=\s*(-?\d+)", body))
    structs: dict[str, type[C.Structure]] = {}
    for body, name in re.findall(r"typedef\s+struct\s*\w*\s*\{(.*?)\}\s*(\w+)\s*;", text, flags=re.S):
        fields = []
        for member in filter(str.strip, body.split(";")):
            first, *more = member.split(",")          # `int64_t a_w1, a_b1, ...;`
            ctype = _ctype(first, structs, member)
            names = [re.findall(r"\w+", first)[-1], *(n.strip() for n in more)]
            if not all(re.fullmatch(r"\w+", n) for n in names):
                raise HeaderError(f"cannot read the member {' '.join(member.split())!r} of {name}")
            fields += [(n, ctype) for n in names]
        structs[name] = type(name, (C.Structure,), {"_fields_": fields})
    diag = re.search(r"#ifdef\s+TS_B200_DIAGNOSTICS\b(.*?)#endif", text, flags=re.S)
    product = text.replace(diag[0], "") if diag else text
    return Abi(_functions(product, structs), _functions(diag[1] if diag else "", structs), structs, consts)


with open(HEADER_PATH) as _f:
    ABI = parse_header(_f.read())

TS_F32, TS_F64 = ABI.consts["TS_F32"], ABI.consts["TS_F64"]
AC_RELU, AC_CATEGORICAL = ABI.consts["TS_AC_RELU"], ABI.consts["TS_AC_CATEGORICAL"]
LOSS_PPO, LOSS_A2C = ABI.consts["TS_LOSS_PPO"], ABI.consts["TS_LOSS_A2C"]
OPT_ADAM, OPT_RMSPROP = ABI.consts["TS_OPT_ADAM"], ABI.consts["TS_OPT_RMSPROP"]
STATS_STRIDE = ABI.consts["TS_PPO_STATS_STRIDE"]
GRAD_EXTRA = ABI.consts["TS_PPO_GRAD_EXTRA"]
TS_PEER_HANDLE_BYTES = ABI.consts["TS_PEER_HANDLE_BYTES"]
ActorCriticDesc = ABI.structs["ts_actor_critic_desc"]
PPOHParams = ABI.structs["ts_ppo_hparams"]

DIAG_LIB_PATH = os.path.join(_HERE, "libts_b200_diag.so")
_lib: C.CDLL | None = None


def _bind(lib: C.CDLL, functions: dict[str, tuple[Any, list[Any]]]) -> C.CDLL:
    for name, (restype, argtypes) in functions.items():
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = restype, argtypes
    return lib


def use_diagnostics_library() -> C.CDLL:
    """Make the process-wide library the DIAGNOSTICS build (phase timeline, wgmma self-test); tools/ only."""
    global _lib
    if not os.path.exists(DIAG_LIB_PATH):
        raise ExtensionMissingError(f"{DIAG_LIB_PATH} not found: build it with `python -m tianshou_b200.csrc.build --diag`")
    _lib = None
    _lib = _bind(load_library(DIAG_LIB_PATH), ABI.diag_functions)
    return _lib


def load_library(path: str | None = None) -> C.CDLL:
    """dlopen the C-ABI library and attach the header's prototypes.  Raises ExtensionMissingError loudly."""
    global _lib
    if _lib is not None and path is None:
        return _lib
    p = path or LIB_PATH
    if not os.path.exists(p):
        raise ExtensionMissingError(
            f"{p} not found: build it with `python -m tianshou_b200.csrc.build` "
            "(nvcc, sm_90a).  tianshou_b200 has no CPU fallback."
        )
    lib = _bind(C.CDLL(p), ABI.functions)
    if path is None:
        _lib = lib
    return lib


def require_cuda() -> None:
    if not torch.cuda.is_available():
        raise ExtensionMissingError(
            "tianshou_b200 device path called without a CUDA device: there is no CPU fallback."
        )


def check(status: int, what: str) -> None:
    if status != 0:
        msg = load_library().ts_last_error().decode(errors="replace")
        raise RuntimeError(f"{what} failed (status {status}): {msg}")


def ptr(t: torch.Tensor | None) -> int | None:
    """Raw device pointer of a contiguous CUDA tensor (None -> NULL)."""
    if t is None:
        return None
    assert t.is_cuda, "device pointer requested for a host tensor"
    assert t.is_contiguous(), "kernels take dense tensors"
    return t.data_ptr()


def stream_ptr(device: torch.device | None = None) -> int:
    return torch.cuda.current_stream(device).cuda_stream


def call(name: str, *args: Any) -> None:
    lib = load_library()
    check(getattr(lib, name)(*args), name)


def launch_count() -> int:
    return int(load_library().ts_launch_count())


def reset_launch_count() -> None:
    load_library().ts_reset_launch_count()


def to_device(a: np.ndarray | torch.Tensor, device: torch.device, dtype: torch.dtype | None = None,
              non_blocking: bool = False) -> torch.Tensor:
    """numpy / tensor -> contiguous device tensor (bool arrays become uint8 views)."""
    if isinstance(a, np.ndarray):
        if a.dtype == np.bool_:
            a = a.view(np.uint8)
        t = torch.from_numpy(np.ascontiguousarray(a))
    else:
        t = a
        if t.dtype == torch.bool:
            t = t.view(torch.uint8)
    if dtype is not None and t.dtype != dtype:
        t = t.to(dtype)
    return t.to(device, non_blocking=non_blocking).contiguous()
