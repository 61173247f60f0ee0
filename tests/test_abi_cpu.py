"""The C ABI boundary, checked on the CPU: include/vmambair_b200.h against its ctypes mirrors in vmambair_b200/_lib.py.

A small C program generated from the mirrors is compiled against the header with the host compiler and prints what C says about
every mirrored typedef: its size and, looked up by the ctypes field names, every member's offset, size and scalar kind (nested
structs and array elements included).  A field the header does not have fails to compile and is reported as a mismatch.  The
constants Python hard-codes, and the parameter count of every declared function, are compared the same way.  Field order matters
only to the mirrors: every argument struct is built from keyword arguments naming its fields, which an ast walk over the Python
sources enforces."""
import ast
import ctypes as C
import functools
import os
import re
import subprocess
import tempfile

from vmambair_b200 import _lib, ops

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "vmambair_b200.h")
STRUCTS = [v for v in vars(_lib).values() if isinstance(v, type) and issubclass(v, C.Structure)]
MIRRORS = {getattr(v, "_c_name_", None): v for v in STRUCTS}
_FLOAT, _INT = (C.c_float, C.c_double), (C.c_int, C.c_long, C.c_longlong)


def _header_code():
    return re.sub(r"/\*.*?\*/", " ", open(HEADER).read(), flags=re.S)


def _kind(t):
    return "f" if t in _FLOAT else "i" if t in _INT else "o"


def _layout(t, path="", off=0):
    """(C member designator, offset, size, kind) of a value of ctypes type t at `path`, then of every member and array element 0
    inside it; path "" is the struct itself"""
    yield path, off, C.sizeof(t), _kind(t)
    if issubclass(t, C.Array):
        yield from _layout(t._type_, f"{path}[0]", off)
    elif issubclass(t, C.Structure):
        for name, ft in t._fields_:
            yield from _layout(ft, f"{path}.{name}" if path else name, off + getattr(t, name).offset)


def _constants():
    """every vmb_dtype value and VMB_CONV_* / VMB_PREP_MAX_JOBS macro of the header -> the value Python uses for it"""
    code = _header_code()
    enum = re.search(r"typedef\s+enum\s*\{([^}]*)\}\s*vmb_dtype\s*;", code).group(1)
    want = {n: getattr(_lib, "DT_" + n[4:]) for n in re.findall(r"\b(VMB_\w+)\s*=", enum)}
    want.update({n: getattr(ops, n[4:]) for n in re.findall(r"#define\s+(VMB_CONV_\w+)", code)})
    want["VMB_PREP_MAX_JOBS"] = len(_lib.PrepArgs().jobs)
    return want


@functools.lru_cache(maxsize=None)
def _c_values():
    """{(typedef, member designator): (offset, size, kind)} and {constant: value}, as the C compiler sees the header"""
    lines = ["#include <stddef.h>", "#include <stdio.h>", '#include "vmambair_b200.h"',
             '#define KIND(x) _Generic((x), float: "f", double: "f", int: "i", long: "i", long long: "i", default: "o")',
             "int main(void) {"]
    for cname, mirror in MIRRORS.items():
        lines.append(f'    printf("{cname}||0|%zu|o\\n", sizeof({cname}));')
        for path, _, _, _ in list(_layout(mirror))[1:]:
            m = f"(({cname}*)0)->{path}"
            lines.append(f'    printf("{cname}|{path}|%zu|%zu|%s\\n", offsetof({cname}, {path}), sizeof({m}), KIND({m}));')
    for name in _constants():
        lines.append(f'    printf("={name}|%lld\\n", (long long)({name}));')
    lines += ["    return 0;", "}"]
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "abi.c"), os.path.join(d, "abi")
        with open(src, "w") as f:
            f.write("\n".join(lines) + "\n")
        r = subprocess.run(["gcc", "-std=c11", "-I", os.path.dirname(HEADER), src, "-o", exe], capture_output=True, text=True)
        assert r.returncode == 0, f"the mirrors name members the header does not declare:\n{r.stderr}"
        out = subprocess.run([exe], capture_output=True, text=True, check=True).stdout
    layout, consts = {}, {}
    for line in out.splitlines():
        if line.startswith("="):
            name, v = line[1:].split("|")
            consts[name] = int(v)
        else:
            cname, path, off, size, kind = line.split("|")
            layout[(cname, path)] = (int(off), int(size), kind)
    return layout, consts


def test_every_header_struct_has_one_mirror():
    typedefs = re.findall(r"typedef\s+struct\s*\{[^{}]*\}\s*(vmb_\w+)\s*;", _header_code())
    names = [getattr(v, "_c_name_", None) for v in STRUCTS]
    assert None not in names, [v.__name__ for v in STRUCTS if not hasattr(v, "_c_name_")]
    assert len(names) == len(set(names)), "two mirrors name the same typedef"
    assert set(names) == set(typedefs), {"no mirror": set(typedefs) - set(names), "no such typedef": set(names) - set(typedefs)}


def test_mirror_layouts_match_the_header():
    """size of every mirror; offset, size and kind of every member (by name), nested structs and arrays included"""
    layout, _ = _c_values()
    bad = [(cname, path, (off, size, kind), layout[(cname, path)])
           for cname, mirror in MIRRORS.items() for path, off, size, kind in _layout(mirror)
           if layout[(cname, path)] != (off, size, kind)]
    assert not bad, "(typedef, member, ctypes (offset, size, kind), C (offset, size, kind)):\n" + "\n".join(map(str, bad))


def test_python_constants_match_the_header():
    _, consts = _c_values()
    want = _constants()
    assert {"VMB_F32", "VMB_BF16", "VMB_F16", "VMB_CONV_PLAIN", "VMB_CONV_ADD_NEAREST"} <= set(want)
    assert consts == want


def test_symbol_parameter_counts_match_the_prototypes():
    protos = dict(re.findall(r"\b(vmb_\w+)\s*\(([^()]*)\)\s*;", _header_code()))
    assert set(protos) == set(_lib.SYMBOLS)
    for name, (_, argtypes) in _lib.SYMBOLS.items():
        params = [] if protos[name].strip() == "void" else protos[name].split(",")
        assert len(argtypes) == len(params), (name, argtypes, protos[name])
        for t, p in zip(argtypes, params):  # a struct pointer points at the mirror of the struct the prototype names
            if hasattr(t, "_type_") and isinstance(t._type_, type) and issubclass(t._type_, C.Structure):
                assert re.search(rf"\b{t._type_._c_name_}\s*\*", p), (name, t._type_.__name__, p)


def _python_sources():
    for top in ("vmambair_b200", "tests", "tools"):
        for d, _, files in os.walk(os.path.join(ROOT, top)):
            yield from (os.path.join(d, f) for f in sorted(files) if f.endswith(".py"))
    yield os.path.join(ROOT, "__graft_entry__.py")


def test_structs_are_built_by_field_name():
    """_lib.<Mirror>(...) and a Mirror imported from _lib take keyword arguments only, each naming a field of that mirror: no value is
    placed by field order, and none is lost to a misspelt name (ctypes would keep it as a plain attribute, leaving the field zero)"""
    bad = []
    for path in _python_sources():
        tree = ast.parse(open(path).read(), path)
        imported = {a.asname or a.name: a.name for n in ast.walk(tree)
                    if isinstance(n, ast.ImportFrom) and (n.module or "").endswith("_lib") for a in n.names}
        for n in ast.walk(tree):
            if not isinstance(n, ast.Call):
                continue
            f = n.func
            via_lib = isinstance(f, ast.Attribute) and (getattr(f.value, "id", None) == "_lib" or getattr(f.value, "attr", None) == "_lib")
            name = f.attr if via_lib else imported.get(f.id) if isinstance(f, ast.Name) else None
            mirror = getattr(_lib, name, None) if name is not None else None
            if not (isinstance(mirror, type) and issubclass(mirror, C.Structure)):
                continue
            fields = {field for field, _ in mirror._fields_}
            unknown = [k.arg for k in n.keywords if k.arg not in fields]  # k.arg None: **mapping, whose names cannot be checked
            if n.args or unknown:
                bad.append(f"{os.path.relpath(path, ROOT)}:{n.lineno} {name}: {len(n.args)} positional, unknown fields {unknown}")
    assert not bad, "argument structs not built by field name:\n" + "\n".join(bad)
