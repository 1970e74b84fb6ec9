"""ctypes binding of the C-ABI library, read from its header (include/occ_b200.h).  There is NO fallback: if the library
or the header is missing or a call fails, a RuntimeError is raised -- the product path never routes through PyTorch
reference code or the oracle."""
import ctypes
import functools
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
# the types the header's pointers point to (ops._call matches a tensor's dtype against them)
_POINTEES = {"void", "float", "double", "int", "unsigned", "unsigned int", "unsigned char", "long long", "size_t"}


def _ctype(decl, fn):
    """C value type ("unsigned int ", "const int ") -> ctypes type"""
    t = _CTYPES.get(" ".join(w for w in decl.split() if w != "const"))
    if t is None:
        raise RuntimeError(f"occformer_b200: {fn}: no ctypes type for the C type '{decl.strip()}' of its declaration")
    return t


def _param(decl, fn):
    """one parameter ("const float* x") -> (ctypes type, name, pointee type without const ("float") or None)"""
    typ, name = re.fullmatch(r"\s*(.*?)\b(\w+)\s*", decl, re.S).groups()
    if "*" not in typ:
        return _ctype(typ, fn), name, None
    pointee = " ".join(w for w in typ.replace("*", " ", 1).split() if w != "const")
    if pointee not in _POINTEES:
        raise RuntimeError(f"occformer_b200: {fn}: unknown pointee type of its parameter '{decl.strip()}'")
    return c_void_p, name, pointee


def _declarations(path):
    """name -> (restype, [(argtype, parameter name, pointee type or None)]) of every occ_* function in the header"""
    if not os.path.exists(path):
        raise RuntimeError(f"occformer_b200: {path} is missing; the ctypes binding is read from it.")
    text = re.sub(r"/\*.*?\*/", " ", open(path).read(), flags=re.S)  # comments, also inside parameter lists
    text = re.sub(r"^\s*#.*$", "", text, flags=re.M)                 # preprocessor lines
    decls = {}
    for stmt in text.split(";"):
        m = re.fullmatch(r"\s*([\w\s*]+?)\b(occ_\w+)\s*\((.*)\)\s*", stmt, re.S)
        if m:
            ret, name, params = m.groups()
            params = [] if params.strip() in ("", "void") else params.split(",")
            decls[name] = (_ctype(ret, name), [_param(p, name) for p in params])
    return decls


def signatures(path=HEADER_PATH):
    """name -> (restype, argtypes) of every occ_* function declared in the header"""
    return {name: (res, [a for a, _, _ in ps]) for name, (res, ps) in _declarations(path).items()}


@functools.lru_cache(maxsize=None)
def parameters(path=HEADER_PATH):
    """name -> [(parameter name, pointee C type or None)] of every occ_* function declared in the header (read once)"""
    return {name: [(p, t) for _, p, t in ps] for name, (_, ps) in _declarations(path).items()}


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
