"""ctypes binding of libreagent_b200.so, read from the C ABI in include/reagent_b200.h.

The header is the one description of the ABI.  At import, every `#define RB200_X value` becomes
the module attribute X (and ACT = {"relu": RB200_ACT_RELU, ...}), and every
`typedef struct rb200_foo_bar { ... } rb200_foo_bar_t;` becomes the ctypes.Structure FooBarT
(STRUCTS maps the C names to them).  lib() gives every rb200_* prototype its argtypes / restype
(FUNCTIONS).  A declaration outside the subset read here raises Rb200Error at import.

The product path has NO fallback: if the CUDA library is missing or a call fails this
module raises.  Build with `python -c "import __graft_entry__ as g; g.build()"` or
`reagent_b200/csrc/build.sh`.
"""
import ast
import ctypes as C
import operator
import os
import re


class Rb200Error(RuntimeError):
    pass


HEADER_PATH = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                           "include", "reagent_b200.h")

_SCALARS = {"int32_t": C.c_int32, "int64_t": C.c_int64, "uint32_t": C.c_uint32,
            "uint8_t": C.c_uint8, "int": C.c_int, "float": C.c_float, "double": C.c_double}
_POINTEES = ("void", "char", "unsigned char")  # types that appear only behind a pointer
_OPS = {ast.Add: operator.add, ast.Sub: operator.sub, ast.Mult: operator.mul}
_DECL = re.compile(r"(?:const\s+)?(unsigned\s+\w+|\w+)\s*(.*)", re.S)
_DECLARATOR = re.compile(r"((?:\*\s*(?:const\b\s*)?)*)(\w+)\s*(?:\[([^\[\]]+)\])?")
_STATEMENT = re.compile(r"\s*(typedef\s+struct\s+\w+\s*\{([^{}]*)\}\s*(\w+)|[^;{}]+?)\s*;")
_PROTOTYPE = re.compile(r"(.+?)\b(rb200_\w+)\s*\(([^()]*)\)")


def _value(expr, consts, what):
    """A number, or + - * over numbers and earlier RB200_* constants."""
    def ev(n):
        if isinstance(n, ast.Constant) and type(n.value) in (int, float):
            return n.value
        if isinstance(n, ast.Name) and n.id in consts:
            return consts[n.id]
        if isinstance(n, ast.UnaryOp) and isinstance(n.op, ast.USub):
            return -ev(n.operand)
        if isinstance(n, ast.BinOp) and type(n.op) in _OPS:
            return _OPS[type(n.op)](ev(n.left), ev(n.right))
        raise Rb200Error(f"reagent_b200.h: unsupported value {expr.strip()!r} in {what}")

    try:
        return ev(ast.parse(expr.strip(), mode="eval").body)
    except SyntaxError:
        raise Rb200Error(f"reagent_b200.h: unsupported value {expr.strip()!r} in {what}") from None


def _ctype(base, stars, structs, what):
    # Pointer rule, for fields and parameters alike: a pointer to an rb200 struct is a host
    # descriptor -- callers pass the struct or C.pointer(desc), and ctypes keeps it alive -- so it
    # becomes POINTER(struct).  rb200_feature_col_t* is a device array that callers assign as an
    # int; it and every other pointer become c_void_p.
    if stars == 0:
        t = _SCALARS.get(base) or structs.get(base)
    elif stars == 1 and base in structs and base != "rb200_feature_col_t":
        t = C.POINTER(structs[base])
    elif base in _SCALARS or base in structs or base in _POINTEES:
        t = C.c_void_p
    else:
        t = None
    if t is None:
        raise Rb200Error(f"reagent_b200.h: unsupported type {base + '*' * stars!r} in {what}")
    return t


def _declarations(decl, consts, structs, what):
    """[(name, ctype)] of one C declaration, `int32_t a, b[N]` or `const float* const* p`."""
    m = _DECL.fullmatch(decl.strip())
    if not m:
        raise Rb200Error(f"reagent_b200.h: cannot read {decl.strip()!r} in {what}")
    base, out = m.group(1), []
    for d in m.group(2).split(","):
        dm = _DECLARATOR.fullmatch(d.strip())
        if not dm:
            raise Rb200Error(f"reagent_b200.h: cannot read {decl.strip()!r} in {what}")
        t = _ctype(base, dm.group(1).count("*"), structs, what)
        if dm.group(3) is not None:
            t = t * _value(dm.group(3), consts, what)
        out.append((dm.group(2), t))
    return out


def read_header(text):
    """(constants, structs, functions) of the C header `text`: {"RB200_X": value},
    {"rb200_foo_t": ctypes.Structure} and {"rb200_f": (restype, argtypes)}."""
    text = re.sub(r"/\*.*?\*/|//[^\n]*", " ", text, flags=re.S)
    text = re.sub(r"^\s*#\s*ifdef\s+__cplusplus\b.*?^\s*#\s*endif\b", "", text, flags=re.S | re.M)
    consts = {}
    for m in re.finditer(r"^[ \t]*#[ \t]*define[ \t]+(RB200_\w+)(.*)$", text, re.M):
        if not m.group(2)[:1].isspace():  # a function-like macro or one without a value
            raise Rb200Error(f"reagent_b200.h: unsupported macro {m.group(0).strip()!r}")
        consts[m.group(1)] = _value(m.group(2), consts, m.group(1))
    text = re.sub(r"^[ \t]*#[^\n]*", "", text, flags=re.M)
    structs, functions, pos = {}, {}, 0
    while text[pos:].strip():
        m = _STATEMENT.match(text, pos)
        if not m:
            raise Rb200Error(f"reagent_b200.h: cannot read {' '.join(text[pos:].split())[:80]!r}")
        pos = m.end()
        if m.group(2) is not None:
            tname = m.group(3)
            short = re.fullmatch(r"rb200_(\w+)_t", tname)
            if not short:
                raise Rb200Error(f"reagent_b200.h: struct {tname!r} is not named rb200_*_t")
            fields = [f for s in m.group(2).split(";") if s.strip()
                      for f in _declarations(s, consts, structs, tname)]
            cls_name = "".join(w.capitalize() for w in short.group(1).split("_")) + "T"
            structs[tname] = type(cls_name, (C.Structure,), {"_fields_": fields})
            continue
        decl = " ".join(m.group(1).split())
        p = _PROTOTYPE.fullmatch(decl)
        if not p:
            raise Rb200Error(f"reagent_b200.h: cannot read {decl!r}")
        ret, name, params = p.group(1).strip(), p.group(2), p.group(3).strip()
        if ret in ("void", "const char*"):
            restype = None if ret == "void" else C.c_char_p
        else:
            [(_, restype)] = _declarations(ret + " _", consts, structs, name)
        argtypes = []
        for q in params.split(",") if params != "void" else []:
            [(_, t)] = _declarations(q, consts, structs, name)
            argtypes.append(t)
        functions[name] = (restype, argtypes)
    return consts, structs, functions


if not os.path.exists(HEADER_PATH):
    raise Rb200Error(f"{HEADER_PATH} not found: the binding is read from the C header")
with open(HEADER_PATH) as _f:
    _CONSTS, STRUCTS, FUNCTIONS = read_header(_f.read())
globals().update({k[len("RB200_"):]: v for k, v in _CONSTS.items()})
globals().update({cls.__name__: cls for cls in STRUCTS.values()})
ACT = {k[len("RB200_ACT_"):].lower(): v for k, v in _CONSTS.items() if k.startswith("RB200_ACT_")}


_LIB = None
# RB200_LIB selects another build of the SAME library (e.g. the profiling build with the
# clock64 timeline compiled in); there is no other implementation to fall back to.
LIB_PATH = os.environ.get("RB200_LIB") or os.path.join(
    os.path.dirname(os.path.abspath(__file__)), "libreagent_b200.so")


def lib():
    """Load (once) and return the shared library; raise loudly if it is missing."""
    global _LIB
    if _LIB is None:
        if not os.path.exists(LIB_PATH):
            raise Rb200Error(
                f"{LIB_PATH} not found: the CUDA extension is not built. "
                "Run reagent_b200/csrc/build.sh (there is no CPU fallback).")
        so = C.CDLL(LIB_PATH)
        for name, (restype, argtypes) in FUNCTIONS.items():
            f = getattr(so, name)
            f.restype, f.argtypes = restype, argtypes
        _LIB = so
    return _LIB


def check(rc, what=""):
    if rc != 0:
        msg = lib().rb200_last_error().decode("utf-8", "replace")
        raise Rb200Error(f"{what} failed (rc={rc}): {msg}")


def ptr(t, device=None):
    """Device pointer of a torch tensor (None -> NULL).  A host tensor -- or one on another
    GPU than `device` -- would reach the kernel as a wild pointer (illegal address, sticky
    context error), so it is refused here with a Python exception instead."""
    if t is None:
        return None
    if not t.is_cuda:
        raise Rb200Error("reagent_b200: a CPU tensor reached a CUDA entry point (call "
                         "trainer.cuda() / batch.cuda() first; there is no CPU path)")
    if device is not None and t.device != device:
        raise Rb200Error(f"reagent_b200: tensor on {t.device}, expected {device}")
    return t.data_ptr()


def on_device(t, device):
    """`t` on `device` (moved once if it was created elsewhere, e.g. trainer-owned constants
    of a trainer that was built from already-CUDA networks and never .cuda()'d)."""
    if t is None or (t.is_cuda and t.device == device):
        return t
    return t.to(device)


def cur_stream():
    import torch

    return torch.cuda.current_stream().cuda_stream


def require_current_device(device):
    """Launches go to the CURRENT device's stream; tensors elsewhere would be wild pointers
    there.  Multi-GPU callers run one process per GPU or wrap calls in torch.cuda.device()."""
    import torch

    if device.type != "cuda" or torch.cuda.current_device() != (device.index or 0):
        raise Rb200Error(f"reagent_b200: tensors live on {device} but the current CUDA device is "
                         f"cuda:{torch.cuda.current_device()} -- wrap the call in "
                         f"torch.cuda.device({device.index})")
