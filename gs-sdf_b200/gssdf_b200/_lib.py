"""ctypes binding of libgssdf_b200.so generated from include/gssdf_b200.h (the single source of truth).

The library is the product: if it is missing or fails to load this module raises -- there is no
CPU or PyTorch fallback anywhere in the package.
"""
import ctypes as C
import os
import re

_PKG = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(_PKG))
HEADER = os.path.join(ROOT, "include", "gssdf_b200.h")
SO_PATH = os.path.join(os.path.dirname(_PKG), "libgssdf_b200.so")

_SCALARS = {"uint8_t": C.c_uint8, "int32_t": C.c_int32, "int64_t": C.c_int64, "uint32_t": C.c_uint32, "float": C.c_float,
            "size_t": C.c_size_t, "int": C.c_int, "double": C.c_double}


def _strip_comments(src):
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return re.sub(r"//[^\n]*", "", src)


def parse_header(path=HEADER):
    """Returns ({struct_name: [(field, ctype)]}, {func_name: (restype, n_args)})."""
    src = _strip_comments(open(path).read())
    for m in re.finditer(r"#define\s+(GSSDF_\w+)\s+(\d+)\s*$", src, flags=re.M):  # integer macros used as array extents
        src = re.sub(r"\[" + m.group(1) + r"\]", "[" + m.group(2) + "]", src)
    structs = {}
    ctypes_structs = {}
    for m in re.finditer(r"typedef\s+struct\s+(\w+)\s*\{(.*?)\}\s*(\w+)\s*;", src, flags=re.S):
        name, body = m.group(3), m.group(2)
        fields = []
        for decl in body.split(";"):
            decl = " ".join(decl.split())
            if not decl:
                continue
            decl = decl.replace("const ", "")
            base, rest = decl.split(" ", 1)
            for item in rest.split(","):
                item = item.strip()
                arr = re.match(r"(\w+)\[(\d+)\]$", item)
                parr = re.match(r"\*\s*(\w+)\[(\d+)\]$", item)
                if parr:  # array of pointers
                    fields.append((parr.group(1), C.c_void_p * int(parr.group(2))))
                elif item.startswith("*"):
                    fields.append((item.lstrip("* "), C.c_void_p))
                elif arr:
                    fields.append((arr.group(1), (ctypes_structs.get(base) or _SCALARS[base]) * int(arr.group(2))))
                elif base in ctypes_structs:  # nested struct by value
                    fields.append((item, ctypes_structs[base]))
                else:
                    fields.append((item, _SCALARS[base]))
        structs[name] = fields
        ctypes_structs[name] = type(name, (C.Structure,), {"_fields_": fields})
    funcs = {}
    for m in re.finditer(r"^\s*(const char \*|int64_t|int32_t|int|size_t)\s*(gssdf_\w+)\s*\(([^)]*)\)\s*;", src, flags=re.M):
        ret, name, args = m.group(1).strip(), m.group(2), m.group(3)
        funcs[name] = (ret, args)
    return structs, funcs, ctypes_structs


_STRUCT_FIELDS, FUNCS, STRUCTS = parse_header()


def _argtypes(args):
    """ctypes argtypes of one prototype's parameter list: pointers, struct pointers and gssdf_stream_t -> c_void_p."""
    args = args.strip()
    if args in ("", "void"):
        return []
    out = []
    for item in args.split(","):
        item = " ".join(item.replace("const ", "").split())
        if "*" in item or item.startswith("gssdf_stream_t"):
            out.append(C.c_void_p)
        else:
            out.append(_SCALARS[item.split(" ")[0]])
    return out

_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(SO_PATH):
            raise RuntimeError(
                f"{SO_PATH} not found: build it with `python gs-sdf_b200/build.py` (nvcc, sm_90a). "
                "gssdf_b200 has no CPU/PyTorch fallback.")
        L = C.CDLL(SO_PATH)
        for name, (ret, _args) in FUNCS.items():
            fn = getattr(L, name)  # raises AttributeError if a declared symbol is not exported
            fn.restype = {"int": C.c_int, "int32_t": C.c_int32, "int64_t": C.c_int64, "size_t": C.c_size_t, "const char *": C.c_char_p}[ret]
            # typed arguments: an untyped Python int is passed as a 32-bit C int, which would truncate 64-bit handles
            # (cudaStream_t of a non-default stream, device pointers, int64 sizes)
            fn.argtypes = _argtypes(_args)
        m = re.search(r"#define\s+GSSDF_ABI_REVISION\s+(\d+)", open(HEADER).read())
        if m and L.gssdf_abi_revision() != int(m.group(1)):
            raise RuntimeError(f"{SO_PATH} was built against ABI revision {L.gssdf_abi_revision()}, the header says {m.group(1)}: "
                               "rebuild with `python gs-sdf_b200/build.py`")
        _lib = L
    return _lib


class GssdfError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"gssdf_b200 error {code}: {msg}")
        self.code = code


def check(rc):
    if rc != 0:
        msg = lib().gssdf_last_error().decode()
        if rc == -1:
            raise ValueError(f"gssdf_b200: {msg}")  # reference: TORCH_CHECK / std::invalid_argument
        raise GssdfError(rc, msg)


def make_args(struct_name, **kw):
    S = STRUCTS[struct_name]
    a = S()
    names = {f[0] for f in S._fields_}
    for k, v in kw.items():
        if k not in names:
            raise KeyError(f"{struct_name} has no field {k}")
        if hasattr(v, "data_ptr"):  # torch tensor
            v = v.data_ptr() if v.numel() > 0 else (v.data_ptr() or None)
        elif isinstance(v, (list, tuple)):
            v = type(getattr(a, k))(*v)
        setattr(a, k, v)
    return a
