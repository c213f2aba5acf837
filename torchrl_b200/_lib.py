"""ctypes binding of libtorchrl_b200.so.

The C ABI is declared once, in include/torchrl_b200.h: ``load()`` reads every entry point's argument and return types
from that header, and ``call()`` checks each operand against its declaration before the launch.

There is NO fallback: if the shared object or the header is missing, a symbol is absent or a declaration uses a type
the binding does not know, ``load()`` raises.  ``load()`` only dlopens the library -- it needs libcudart's static
copy inside the .so but no GPU, so the symbol/ABI checks run on CPU boxes too.
"""
import ctypes
import os
import re

import torch

from . import build

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libtorchrl_b200.so")
HEADER_PATH = build.HEADER

_SCALARS = {"int": ctypes.c_int, "int64_t": ctypes.c_int64, "unsigned": ctypes.c_uint32, "uint64_t": ctypes.c_uint64,
            "float": ctypes.c_float, "double": ctypes.c_double}
_RESTYPES = {"int": ctypes.c_int, "int64_t": ctypes.c_int64, "char*": ctypes.c_char_p}
# the tensor dtype of each pointee type; void: no dtype check
_DTYPES = {"float": torch.float32, "double": torch.float64, "uint8_t": torch.uint8, "int": torch.int32,
           "int32_t": torch.int32, "unsigned": torch.int32, "int64_t": torch.int64, "uint64_t": torch.int64,
           "void": None}
_DECL = re.compile(r"^\s*([\w *]+?)\s*\b(trl_\w+)\s*\(([^)]*)\)\s*;", re.M)
_PARAM = re.compile(r"(.*?)(\w+)", re.S)

# name -> (restype, params), params: (name, ctypes type, pointee dtype or None, pointer depth) per parameter
SIGNATURES = {}
# name -> (function, parameter count, (index, dtype) of each pointer parameter (dtype None: not checked),
#         (index, element dtype) of each `T* const*` parameter)
_CALLS = {}
_lib = None


class NativeLibraryError(RuntimeError):
    pass


def _bare(ctype):
    return re.sub(r"\bconst\b|\s", "", ctype)


def parse_header(path):
    """SIGNATURES of every declaration `ret trl_name(type name, ...);` of the header, comments stripped."""
    if not os.path.exists(path):
        raise NativeLibraryError("%s not found: the binding reads the C ABI from it" % path)
    src = re.sub(r"/\*.*?\*/", "", open(path).read(), flags=re.S)
    sigs = {}
    for ret, name, params in _DECL.findall(src):
        decl = "%s(%s)" % (name, " ".join(params.split()))
        if _bare(ret) not in _RESTYPES:
            raise NativeLibraryError("%s: unsupported return type %r of %s" % (path, ret.strip(), decl))
        out = []
        for p in ([] if params.strip() == "void" else params.split(",")):
            ctype, pname = _PARAM.fullmatch(p.strip()).groups()
            t = _bare(ctype)
            base = t.rstrip("*")
            depth = len(t) - len(base)
            if base not in (_DTYPES if depth else _SCALARS):
                raise NativeLibraryError("%s: unsupported type %r in %s" % (path, ctype.strip(), decl))
            out.append((pname, ctypes.c_void_p if depth else _SCALARS[base], _DTYPES[base] if depth else None, depth))
        sigs[name] = (_RESTYPES[_bare(ret)], out)
    return sigs


def load():
    """dlopen the library once and type every entry point the header declares.  Raises if anything is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH) and os.environ.get("TORCHRL_B200_NO_AUTOBUILD") != "1":
        try:                                    # nvcc is part of the image: compile in-tree on first use
            build.build()
        except Exception as e:                  # noqa: BLE001
            raise NativeLibraryError("%s not found and the in-tree nvcc build failed (%s); there is no CPU "
                                     "fallback" % (LIB_PATH, e)) from e
    if not os.path.exists(LIB_PATH):
        raise NativeLibraryError(
            "%s not found: build it with `python -m torchrl_b200.build` (there is no CPU fallback)" % LIB_PATH)
    sigs = parse_header(HEADER_PATH)
    lib = ctypes.CDLL(LIB_PATH)
    for name, (restype, params) in sigs.items():
        try:
            fn = getattr(lib, name)
        except AttributeError as e:
            raise NativeLibraryError("symbol %s missing from %s" % (name, LIB_PATH)) from e
        fn.argtypes = [p[1] for p in params]
        fn.restype = restype
        ptrs = [(i, dtype, depth) for i, (_, _, dtype, depth) in enumerate(params) if depth]
        _CALLS[name] = (fn, len(params), tuple((i, dtype if depth == 1 else None) for i, dtype, depth in ptrs),
                        tuple((i, dtype) for i, dtype, depth in ptrs if depth == 2 and dtype is not None))
    SIGNATURES.update(sigs)
    _lib = lib
    return lib


def check(rc, name):
    if rc != 0:
        msg = load().trl_last_error()
        raise RuntimeError("%s failed (rc=%d): %s" % (name, rc, msg.decode() if msg else ""))


_LAUNCHES = 0


def launch_count():
    """Kernels launched through the C ABI so far (graph replays add their captured count)."""
    return _LAUNCHES


def add_launches(n):
    global _LAUNCHES
    _LAUNCHES += int(n)


def _reject(name, i, t, dtype):
    what = "%s: %s" % (name, SIGNATURES[name][1][i][0])
    if not t.is_cuda:
        raise ValueError("%s must be a CUDA tensor (torchrl_b200 has no CPU path)" % what)
    if t.dtype != dtype:
        raise TypeError("%s must be %s, got %s" % (what, dtype, t.dtype))
    raise ValueError("%s must be contiguous" % what)


def _ptr(t, dtype, name, i):
    if not (t.is_cuda and t.dtype is dtype and t.is_contiguous()):
        _reject(name, i, t, dtype)
    return t.data_ptr()


def call(name, *args, kernels=1):
    """Invoke a kernel-launching entry point, raise on error and count the `kernels` kernels it launched (the
    wrappers in ops.py know that number for each entry point and its arguments).

    The arguments are those of the header's declaration, exactly as many.  A tensor passed for a `T*` parameter must
    be a contiguous CUDA tensor of T's dtype (float32, float64, uint8, int32 for int / unsigned, int64 for int64_t /
    uint64_t); for `void*` and pointer-to-pointer parameters it passes its address unchecked.  A list passed for a
    `T* const*` parameter becomes a host array of its tensors' addresses (None: NULL), each checked against T.  None
    is NULL; ints, ctypes objects and ctypes arrays pass through unchanged."""
    global _LAUNCHES
    if _lib is None:
        load()
    fn, nparams, pointers, arrays = _CALLS[name]
    if len(args) != nparams:
        raise TypeError("%s takes %d arguments, got %d" % (name, nparams, len(args)))
    args = list(args)
    for i, dtype in pointers:          # the hot loop: _ptr's test inlined
        a = args[i]
        if isinstance(a, torch.Tensor):
            if dtype is not None and not (a.is_cuda and a.dtype is dtype and a.is_contiguous()):
                _reject(name, i, a, dtype)
            args[i] = a.data_ptr()
    for i, dtype in arrays:
        if isinstance(args[i], list):
            args[i] = (ctypes.c_void_p * len(args[i]))(*[None if t is None else _ptr(t, dtype, name, i)
                                                         for t in args[i]])
    rc = fn(*args)
    if rc != 0:
        check(rc, name)
    _LAUNCHES += kernels
