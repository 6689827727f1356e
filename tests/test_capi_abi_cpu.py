"""CPU: the ctypes binding states the C ABI of include/svo_b200.h exactly.  capi.PROTOTYPES names every function the
header declares with its return and argument types, and every struct of the header has one ctypes mirror with the
same fields, offsets and size as the C compiler lays it out.  Neither the library build nor a GPU is needed: a wrong
prototype or mirror would pass arguments or read outputs at the wrong place without any error on the host."""
import ctypes as C
import os
import re
import subprocess

from rpg_svo_b200 import capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INCLUDE = os.path.join(ROOT, "include")


def _header() -> str:
    src = open(os.path.join(INCLUDE, "svo_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", " ", src, flags=re.S)
    src = re.sub(r"//[^\n]*", " ", src)
    return re.sub(r"^\s*#[^\n]*", " ", src, flags=re.M)


def _ctype(decl: str, is_return: bool):
    """The ctypes type the binding must use for one C type (a parameter's declaration without its name)."""
    decl = " ".join(decl.split())
    if "*" in decl:
        return C.c_char_p if is_return and decl.replace(" ", "") == "constchar*" else C.c_void_p
    return {"int": C.c_int, "double": C.c_double, "size_t": C.c_size_t, "uint64_t": C.c_uint64, "void": None}[decl]


def _prototypes():
    """[(name, return type, [argument types])] of the header, in its order."""
    out = []
    for ret, name, params in re.findall(r"([A-Za-z_][\w\s\*]*?)\s*\b(svo_b200_\w+)\s*\(([^()]*)\)\s*;", _header()):
        params = [p.strip() for p in params.split(",")]
        if params == ["void"]:
            params = []
        # drop each parameter's name: the type is what precedes the last identifier
        args = [_ctype(re.sub(r"\w+\s*$", "", p), False) for p in params]
        out.append((name, _ctype(ret, True), args))
    return out


def _structs():
    """{typedef name: [field names in order]} of every struct the header defines (not the opaque handles)."""
    out = {}
    for body, name in re.findall(r"typedef\s+struct\s*\w*\s*\{(.*?)\}\s*(\w+)\s*;", _header(), flags=re.S):
        fields = []
        for decl in filter(None, (d.strip() for d in body.split(";"))):
            for d in decl.split(","):
                fields.append(re.search(r"(\w+)\s*(\[[^\]]*\])?\s*$", d).group(1))
        out[name] = fields
    return out


def _mirror_name(typedef: str) -> str:
    return "".join(w.capitalize() for w in typedef[len("svo_b200_"):].split("_"))


def test_prototype_table_matches_the_header():
    header = _prototypes()
    assert len(header) >= 50
    assert [n for n, _, _ in capi.PROTOTYPES] == [n for n, _, _ in header], "names or order differ"
    for (name, ret, args), (_, want_ret, want_args) in zip(capi.PROTOTYPES, header):
        assert len(args) == len(want_args), f"{name}: {len(args)} arguments, the header declares {len(want_args)}"
        assert ret is want_ret, f"{name}: return type {ret}, the header's is {want_ret}"
        for i, (a, w) in enumerate(zip(args, want_args)):
            assert a is w, f"{name}: argument {i} is {a}, the header's is {w}"


def test_struct_mirrors_match_the_c_layout(tmp_path):
    structs = _structs()
    assert len(structs) >= 15
    mirrors = {_mirror_name(t): t for t in structs}
    defined = {k for k, v in vars(capi).items() if isinstance(v, type) and issubclass(v, C.Structure)}
    assert defined == set(mirrors), f"mirrors without a header struct: {defined - set(mirrors)}, " \
                                    f"header structs without a mirror: {set(mirrors) - defined}"
    lines = ["#include <stddef.h>", "#include <stdio.h>", '#include "svo_b200.h"', "int main(void) {"]
    for t, fields in structs.items():
        lines.append(f'  printf("{t} %zu\\n", sizeof({t}));')
        for f in fields:
            lines.append(f'  printf("{t}.{f} %zu %zu\\n", offsetof({t}, {f}), sizeof((({t}*)0)->{f}));')
    lines += ["  return 0;", "}"]
    src, exe = tmp_path / "layout.c", tmp_path / "layout"
    src.write_text("\n".join(lines) + "\n")
    subprocess.check_call(["gcc", "-std=c99", "-I", INCLUDE, "-o", str(exe), str(src)])
    layout = dict(line.split(" ", 1) for line in subprocess.check_output([str(exe)], text=True).splitlines())
    for mirror, t in mirrors.items():
        cls = getattr(capi, mirror)
        names = [n for n, _ in cls._fields_]
        assert names == structs[t], f"{mirror}: fields {names}, {t} has {structs[t]}"
        assert C.sizeof(cls) == int(layout[t]), f"{mirror}: {C.sizeof(cls)} bytes, {t} has {layout[t]}"
        for n in names:
            f = getattr(cls, n)
            assert f"{f.offset} {f.size}" == layout[f"{t}.{n}"], f"{mirror}.{n}: offset, size {f.offset} {f.size}, " \
                                                                 f"C has {layout[f'{t}.{n}']}"
