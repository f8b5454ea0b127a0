"""The C ABI against its ctypes binding (no GPU): reagent_b200/_lib.py reads
include/reagent_b200.h, and these tests hold what it read to the library that was built and to
the layout a C compiler gives the same header."""
import ctypes as C
import os
import re
import subprocess

import pytest

from reagent_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_every_struct_matches_the_library_and_the_c_compiler(tmp_path):
    """Every struct of the header: sizeof in the loaded library, and sizeof and every field's
    offsetof as gcc lays the header out, equal the ctypes binding's.  Sizes alone would miss a
    field the binding places wrongly inside a struct of the right size, which the kernel would
    then read as the wrong pointer."""
    assert len(_lib.STRUCTS) >= 22
    lib = _lib.lib()
    for name, cls in _lib.STRUCTS.items():
        assert lib.rb200_abi_sizeof(name.encode()) == C.sizeof(cls), name
    assert lib.rb200_abi_sizeof(b"no_such_struct") == -1

    want, lines = [], []
    for name, cls in _lib.STRUCTS.items():
        want.append(f"{name} {C.sizeof(cls)}")
        lines.append(f'  printf("{name} %zu\\n", sizeof({name}));')
        for field, _ in cls._fields_:
            want.append(f"{name}.{field} {getattr(cls, field).offset}")
            lines.append(f'  printf("{name}.{field} %zu\\n", offsetof({name}, {field}));')
    src = tmp_path / "layout.c"
    src.write_text("#include <stddef.h>\n#include <stdio.h>\n#include \"reagent_b200.h\"\n"
                   "int main(void) {\n" + "\n".join(lines) + "\n  return 0;\n}\n")
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-std=c11", "-I", os.path.join(ROOT, "include"),
                    str(src), "-o", str(exe)], check=True)
    got = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split("\n")
    assert got[:-1] == want


def test_c_abi_exports_every_declared_symbol():
    lib = _lib.lib()
    hdr = open(os.path.join(ROOT, "include", "reagent_b200.h")).read()
    names = set(re.findall(r"\b(rb200_[a-z0-9_]+)\s*\(", hdr))
    assert len(names) >= 20
    assert names == set(_lib.FUNCTIONS)
    for n in sorted(names):
        assert hasattr(lib, n), f"libreagent_b200.so does not export {n}"
        assert getattr(lib, n).argtypes is not None, n
    assert lib.rb200_version() >= 1


@pytest.mark.parametrize("snippet", [
    "typedef union rb200_u { int32_t a; float b; } rb200_u_t;",
    "typedef struct rb200_b { int32_t a : 3; } rb200_b_t;",
    "typedef struct rb200_c { size_t n; } rb200_c_t;",
    "typedef struct rb200_d { int32_t a[RB200_NOT_DEFINED]; } rb200_d_t;",
    "typedef struct rb200_e { struct { int32_t a; } inner; } rb200_e_t;",
    "int rb200_f(int32_t a, (int32_t b);",
    "int rb200_g(long a);",
    "#define RB200_H(x) (x)",
    "#define RB200_I \"text\"",
    "static int counter;",
])
def test_reader_refuses_what_it_cannot_bind(snippet):
    with pytest.raises(_lib.Rb200Error):
        _lib.read_header("#include <stdint.h>\n" + snippet + "\n")


# ---------------------------------------------------------------------------
# Fields appended to a struct go after every existing one, so a binding built against the
# shorter struct keeps its offsets.
# ---------------------------------------------------------------------------
def test_adam_args_new_fields_follow_every_existing_one():
    A = _lib.AdamArgsT
    names = [f[0] for f in A._fields_]
    assert names[-4:] == ["dp_max_blocks", "decoupled_weight_decay", "amsgrad", "max_exp_avg_sq"]
    # the fields that were there before keep their offsets (their struct was 208 bytes)
    assert A.dp_max_blocks.offset + 4 <= 208 <= A.decoupled_weight_decay.offset + 4
    a = A()
    assert (a.decoupled_weight_decay, a.amsgrad, a.max_exp_avg_sq) == (0, 0, None)


def test_head_structs_grow_by_sample_weight():
    for name, mirror in (("rb200_qrdqn_args_t", _lib.QrdqnArgsT), ("rb200_c51_args_t", _lib.C51ArgsT)):
        assert mirror._fields_[-1][0] == "sample_weight", name
        assert mirror.sample_weight.offset == C.sizeof(mirror) - 8, name


def test_ac_args_struct_grows_by_the_per_fields():
    names = [f[0] for f in _lib.AcArgsT._fields_]
    assert names[-2:] == ["sample_weight", "td_error_out"]
    assert _lib.AcArgsT.td_error_out.offset == C.sizeof(_lib.AcArgsT) - 8
    assert _lib.AcArgsT.sample_weight.offset == C.sizeof(_lib.AcArgsT) - 16


def test_grown_structs_match_their_mirrors():
    assert _lib.DqnArgsT.sample_weight.offset == C.sizeof(_lib.DqnArgsT) - 8
    assert _lib.AddArgsT.priority_from_max.offset > _lib.AddArgsT.rows.offset
