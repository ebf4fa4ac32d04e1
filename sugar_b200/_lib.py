"""ctypes binding of libsugar_b200.so.

The C header include/sugar_b200.h is the binding's only statement of the ABI: its structs, callback types, integer
SGR_* constants and SGR_API prototypes are read from it at import (parse_header) and exported here under their C names.

There is no CPU fallback: if the CUDA library is missing this module raises at import, and every
call raises on a non-zero status with the library's own message.
"""
import ctypes as C
import os
import re

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("SGR_LIB_PATH", os.path.join(_HERE, "lib", "libsugar_b200.so"))  # override: the stats build (scripts/blend_stats.py)
HEADER_PATH = os.path.join(os.path.dirname(_HERE), "include", "sugar_b200.h")

# sgr_struct_bytes(i) is the library's sizeof of _STRUCT_ORDER[i] (the index order of its switch)
_STRUCT_ORDER = ("SgrView", "SgrGaussians", "SgrBackwardPlan", "SgrFieldParams", "SgrSsimParams", "SgrDensifyGates",
                 "SgrDensifyColumn", "SgrAdamSegment", "SgrPeerPlan")

# The header's types by value; a pointer may point to one of these, to a header struct, or to _POINTEES.
_SCALARS = {"int32_t": C.c_int32, "int": C.c_int32, "int64_t": C.c_int64, "uint32_t": C.c_uint32,
            "uint64_t": C.c_uint64, "unsigned long long": C.c_ulonglong, "size_t": C.c_size_t, "float": C.c_float,
            "double": C.c_double}
_POINTEES = ("void", "char", "uint8_t")


class SgrError(RuntimeError):
    pass


def parse_header(text: str):
    """-> (names, prototypes) of the C header `text`.  names: its integer `#define SGR_*` constants, its structs as
    ctypes.Structure classes and its function-pointer typedefs as CFUNCTYPEs, by their C names; prototypes: every
    SGR_API function as name -> (restype, argtypes).  A pointer to a header struct is POINTER(struct), a returned
    `const char *` c_char_p, any other pointer c_void_p.  Raises SgrError naming any declaration it cannot map."""
    text = re.sub(r"/\*.*?\*/|//[^\n]*", " ", text, flags=re.S)
    names = {m[1]: int(m[2]) for m in
             re.finditer(r"^[ \t]*#[ \t]*define[ \t]+(SGR_\w+)[ \t]+\(?[ \t]*(-?\d+)[ \t]*\)?[ \t]*$", text, re.M)}
    text = re.sub(r"^[ \t]*#.*$", "", text, flags=re.M)   # the other preprocessor lines, SGR_API's definition among them
    structs = {s: type(s, (C.Structure,), {"__module__": __name__}) for s in re.findall(r"\bstruct\s+(\w+)", text)}
    callbacks = {}

    def ctype(spec, what, ret=False):
        base, stars = " ".join(w for w in re.findall(r"\w+", spec) if w != "const"), spec.count("*")
        if not stars and (base in _SCALARS or base in callbacks):
            return _SCALARS.get(base) or callbacks[base]
        if ret and (base, stars) in (("void", 0), ("char", 1)):
            return None if base == "void" else C.c_char_p
        if stars == 1 and base in structs:
            return C.POINTER(structs[base])
        if stars and (base in _SCALARS or base in structs or base in _POINTEES):
            return C.c_void_p
        raise SgrError(f"{HEADER_PATH}: {what}: no ctypes type for '{' '.join(spec.split())}'")

    def declarator(decl, what):   # 'const float *x' -> ('const float *', 'x', None); 'float w[11]' -> (.., 'w', 11)
        m = re.fullmatch(r"\s*(.*?)(\w+)\s*(?:\[(\d+)\])?\s*", decl, re.S)
        if m is None:
            raise SgrError(f"{HEADER_PATH}: {what}: cannot parse '{' '.join(decl.split())}'")
        return m[1], m[2], m[3] and int(m[3])

    def params(arglist, fn):
        if arglist.strip() in ("", "void"):
            return []
        return [ctype(declarator(a, fn)[0], f"{fn}({' '.join(a.split())})") for a in arglist.split(",")]

    for m in re.finditer(r"typedef\s+([^;{}()]+?)\(\s*\*\s*(\w+)\s*\)\s*\(([^()]*)\)\s*;", text):
        callbacks[m[2]] = C.CFUNCTYPE(ctype(m[1], m[2], ret=True), *params(m[3], m[2]))
    for m in re.finditer(r"\bstruct\s+(\w+)\s*\{([^{}]*)\}", text):
        fields = []
        for decl in filter(str.strip, m[2].split(";")):
            first, *more = decl.split(",")   # int32_t N, K, P;
            spec, name, n = declarator(first, m[1])
            for spec, name, n in [(spec, name, n)] + [declarator(spec.split("*")[0] + d, m[1]) for d in more]:
                t = ctype(spec, f"{m[1]}.{name}")
                fields.append((name, t * n if n else t))
        structs[m[1]]._fields_ = fields   # after the class exists: SgrPeerPlan is used by pointer before its body
    prototypes = {m[2]: (ctype(m[1], m[2], ret=True), params(m[3], m[2]))
                  for m in re.finditer(r"\bSGR_API\s+([^;{}()]*?)(\w+)\s*\(([^()]*)\)\s*;", text)}
    if len(prototypes) != len(re.findall(r"\bSGR_API\b", text)):
        raise SgrError(f"{HEADER_PATH}: an SGR_API declaration is not of the form `SGR_API <ret> <name>(<args>);`")
    return {**names, **structs, **callbacks}, prototypes


with open(HEADER_PATH) as _f:
    _names, PROTOTYPES = parse_header(_f.read())
globals().update(_names)
_structs = {n for n, t in _names.items() if isinstance(t, type) and issubclass(t, C.Structure)}
if _structs != set(_STRUCT_ORDER):
    raise SgrError(f"{HEADER_PATH}: structs {sorted(_structs ^ set(_STRUCT_ORDER))} are not both in the header and in "
                   "_lib._STRUCT_ORDER, the index order of sgr_struct_bytes")


def _load():
    if not os.path.exists(LIB_PATH):
        raise SgrError(
            f"{LIB_PATH} not found: build it with `python sugar_b200/build.py` (needs nvcc). "
            "sugar_b200 has no CPU or PyTorch fallback.")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in PROTOTYPES.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is missing
        fn.restype = res
        fn.argtypes = args
    return lib


lib = _load()
for _i, _n in enumerate(_STRUCT_ORDER):
    if lib.sgr_struct_bytes(_i) != C.sizeof(_names[_n]):   # a library built from another version of the header
        raise SgrError(f"{LIB_PATH}: struct {_n} is {lib.sgr_struct_bytes(_i)} bytes in the library, "
                       f"{C.sizeof(_names[_n])} in {HEADER_PATH} -- rebuild with `python sugar_b200/build.py`")


def check(status: int) -> None:
    if status != 0:
        raise SgrError(lib.sgr_last_error().decode(errors="replace") or f"libsugar_b200 error {status}")


# How the op wrappers pass tensors to the library.  Argument checks run first, so that they work on CPU tensors too.

def ptr(t):
    """Device pointer of an optional tensor: None or an empty tensor gives NULL."""
    return None if t is None or t.numel() == 0 else t.data_ptr()


def f32_ptr(t, name: str):
    """ptr() of an optional float32 CUDA tensor, checked (the rasterizer's arguments)."""
    if t is None or t.numel() == 0:
        return None
    if t.dtype != torch.float32:
        raise TypeError(f"{name} must be float32, got {t.dtype}")
    if not t.is_cuda:
        raise SgrError(f"{name} must be a CUDA tensor (sugar_b200 has no CPU path)")
    return t.data_ptr()


def stream(dev):
    """The current CUDA stream of `dev` as the library takes it."""
    return torch.cuda.current_stream(dev).cuda_stream


def scratch(nbytes: int, dev) -> torch.Tensor:
    """Device scratch of `nbytes`, the answer of one of the library's size queries."""
    return torch.empty(nbytes, dtype=torch.uint8, device=dev)


def require_cuda(module: str, *ts) -> None:
    for t in ts:
        if t is not None and not (torch.is_tensor(t) and t.is_cuda):
            raise SgrError(f"sugar_b200.{module} needs CUDA tensors: there is no CPU fallback")


def tensor(t, name: str, dtype, shape, device=None, ref: str = "verts", align: int = 0):
    """-> `t` as the kernel may read it: contiguous, and copied when `align` (bytes) is given and not met.
    Raises ValueError unless `t` is a `dtype` tensor of `shape` on `device` (when given; `ref` names the argument
    that fixed it).  `shape` entries are sizes, or names of free dimensions (str)."""
    want = ",".join(str(s) for s in shape)
    if not torch.is_tensor(t) or t.dtype != dtype or t.dim() != len(shape) or \
            any(isinstance(s, int) and t.shape[i] != s for i, s in enumerate(shape)):
        got = f"{t.dtype} {tuple(t.shape)}" if torch.is_tensor(t) else type(t).__name__
        raise ValueError(f"{name} must be {str(dtype).replace('torch.', '')} [{want}], got {got}")
    if device is not None and t.device != device:
        raise ValueError(f"{name} on {t.device}, {ref} on {device}")
    t = t.contiguous()
    if align and t.data_ptr() % align:
        t = t.clone()
    return t


def same_device(dev, ref: str = "verts", **ts) -> None:
    for name, t in ts.items():
        if t is not None and t.device != dev:
            raise ValueError(f"{name} on {t.device}, {ref} on {dev}")


def check_ids(*checks) -> None:
    """checks: (ids, lo, hi, what).  Raises ValueError naming each check with ids outside [lo, hi), after one host
    read for all of them."""
    checks = [c for c in checks if c[0].numel()]
    if not checks:
        return
    counts = torch.stack([((ids < lo) | (ids >= hi)).sum() for ids, lo, hi, _ in checks]).tolist()
    for n, (_, lo, hi, what) in zip(counts, checks):
        if n:
            raise ValueError(f"{n} {what} outside [{lo}, {hi})")


def profile(on: bool) -> None:
    check(lib.sgr_profile_enable(int(on)))


def profile_read():
    """-> {kernel name: (total_ms, launches)} since profiling was enabled / last read."""
    n = lib.sgr_num_kernel_kinds()
    ms = (C.c_float * n)()
    cnt = (C.c_int * n)()
    check(lib.sgr_profile_read(ms, cnt))
    return {lib.sgr_kernel_name(k).decode(): (float(ms[k]), int(cnt[k])) for k in range(n) if cnt[k]}


def profile_timeline(max_records: int = 4096):
    """-> [(kernel name, begin_ms, end_ms)] of every launch since profiling was enabled."""
    kinds = (C.c_int * max_records)()
    tb = (C.c_float * max_records)()
    te = (C.c_float * max_records)()
    n = lib.sgr_profile_timeline(max_records, kinds, tb, te)
    if n < 0:
        check(n)
    return [(lib.sgr_kernel_name(kinds[i]).decode(), float(tb[i]), float(te[i])) for i in range(n)]
