"""ctypes binding of the C-ABI library, read from its header (include/occ_b200.h).  There is NO fallback: if the library
or the header is missing or a call fails, a RuntimeError is raised -- the product path never routes through PyTorch
reference code or the oracle."""
import ctypes
import os
import re
from ctypes import c_double, c_float, c_int, c_longlong, c_size_t, c_uint, c_ulonglong, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "csrc", "libocc_b200.so")
HEADER_PATH = os.path.join(os.path.dirname(_HERE), "include", "occ_b200.h")
_lib = None

# the C types the header uses besides pointers (every pointer, occ_stream_t included, is a c_void_p)
_CTYPES = {"int": c_int, "unsigned int": c_uint, "long long": c_longlong, "unsigned long long": c_ulonglong,
           "size_t": c_size_t, "float": c_float, "double": c_double, "occ_stream_t": c_void_p}


def _ctype(decl, fn):
    """C type with its identifier removed ("const float* ", "unsigned int ") -> ctypes type"""
    if "*" in decl:
        return c_void_p
    t = _CTYPES.get(" ".join(w for w in decl.split() if w != "const"))
    if t is None:
        raise RuntimeError(f"occformer_b200: {fn}: no ctypes type for the C type '{decl.strip()}' of its declaration")
    return t


def signatures(path=HEADER_PATH):
    """name -> (restype, argtypes) of every occ_* function declared in the header"""
    if not os.path.exists(path):
        raise RuntimeError(f"occformer_b200: {path} is missing; the ctypes binding is read from it.")
    text = re.sub(r"/\*.*?\*/", " ", open(path).read(), flags=re.S)  # comments, also inside parameter lists
    text = re.sub(r"^\s*#.*$", "", text, flags=re.M)                 # preprocessor lines
    sigs = {}
    for stmt in text.split(";"):
        m = re.fullmatch(r"\s*([\w\s*]+?)\b(occ_\w+)\s*\((.*)\)\s*", stmt, re.S)
        if m:
            ret, name, params = m.groups()
            params = [] if params.strip() in ("", "void") else params.split(",")
            sigs[name] = (_ctype(ret, name), [_ctype(re.sub(r"\w+\s*$", "", p), name) for p in params])
    return sigs


def lib():
    """Load (once) and return the shared library with every function of the header bound; raise loudly if either is
    not there."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"occformer_b200: {LIB_PATH} is missing. Build it with `python -m occformer_b200.build` "
            "(or __graft_entry__.build()). There is no CPU / PyTorch fallback for the hot path.")
    l = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in signatures().items():
        fn = getattr(l, name)  # AttributeError if the library does not export a declared symbol
        fn.restype = res
        fn.argtypes = args
    _lib = l
    return l


def check(rc, what):
    if rc != 0:
        kind = "argument error" if rc < 0 else "cudaError"
        raise RuntimeError(f"occformer_b200: {what} failed with {kind} {rc}")
