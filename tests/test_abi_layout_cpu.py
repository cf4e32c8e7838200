"""CPU test: every ctypes structure of emoportraits_b200/lib.py has exactly the layout of its C counterpart in
include/emoportraits_b200.h (size and the offset of every field, in declaration order).  A small C program is compiled
against the header and prints sizeof / offsetof; a mismatch would silently scramble kernel arguments on the GPU."""
import ctypes as C
import pathlib
import subprocess

ROOT = pathlib.Path(__file__).resolve().parents[1]

PAIRS = {
    "GridSample3dDesc": "emo_grid_sample3d_desc", "GridSample2dAffineDesc": "emo_grid_sample2d_affine_desc",
    "ResizeBilinearDesc": "emo_resize_bilinear_desc", "GnFinalizeDesc": "emo_gn_finalize_desc", "ApplyDesc": "emo_apply_desc",
    "GnHeadDesc": "emo_gn_head_desc", "ConvDesc": "emo_conv_desc", "ConvPlanInfo": "emo_conv_plan_info", "ConvDirectDesc": "emo_conv_direct_desc",
    "LinearDesc": "emo_linear_desc", "ResampleDesc": "emo_resample_desc", "PoseDesc": "emo_pose_desc",
}


def _c_name(f):
    return f[:-1] if f.endswith("_") and f[:-1] in ("in",) else f


def test_every_ctypes_structure_matches_the_header(tmp_path):
    from emoportraits_b200 import lib as L

    structs = {n: getattr(L, n) for n in PAIRS}
    # every Structure subclass defined in lib.py is covered
    defined = {n for n, v in vars(L).items() if isinstance(v, type) and issubclass(v, C.Structure) and v is not C.Structure}
    assert defined == set(PAIRS), defined ^ set(PAIRS)
    lines = ['#include <stddef.h>', '#include <stdio.h>', f'#include "{ROOT / "include" / "emoportraits_b200.h"}"', "int main(void) {"]
    for py, cn in PAIRS.items():
        lines.append(f'  printf("{py} sizeof %zu\\n", sizeof({cn}));')
        for fname, _ in structs[py]._fields_:
            lines.append(f'  printf("{py} {fname} %zu\\n", offsetof({cn}, {_c_name(fname)}));')
    lines += ["  return 0;", "}"]
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-std=c11", "-o", str(exe), str(src)], check=True)       # unknown field name -> compile error
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout
    got = {}
    for ln in out.splitlines():
        py, key, val = ln.split()
        got[(py, key)] = int(val)
    for py, st in structs.items():
        assert got[(py, "sizeof")] == C.sizeof(st), (py, got[(py, "sizeof")], C.sizeof(st))
        for fname, _ in st._fields_:
            assert got[(py, fname)] == getattr(st, fname).offset, (py, fname, got[(py, fname)], getattr(st, fname).offset)
    # and the header declares no field the binding lacks: count the members of each C struct
    import re

    hdr = (ROOT / "include" / "emoportraits_b200.h").read_text()
    for py, cn in PAIRS.items():
        body = hdr[:hdr.index("} " + cn + ";")]
        body = body[body.rindex("typedef struct"):]   # (emo_apply_desc carries a struct tag: emo_conv_desc.post points to it)
        body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
        decls = [d for d in body.split("{", 1)[1].split(";") if d.strip()]
        n_members = sum(len(d.split(",")) for d in decls)
        assert n_members == len(structs[py]._fields_), (py, n_members, len(structs[py]._fields_))


def test_ctypes_prototypes_match_the_header():
    """argument count and kind (pointer / int / long long / float / double) of every prototype in lib.SYMBOLS vs the header"""
    import re

    from emoportraits_b200 import lib as L

    hdr = re.sub(r"/\*.*?\*/", "", (ROOT / "include" / "emoportraits_b200.h").read_text(), flags=re.S)
    protos = dict(re.findall(r"\n\s*(?:const\s+char\s*\*|int)\s+(emo_\w+)\s*\(([^)]*)\)\s*;", hdr))
    assert set(protos) == set(L.SYMBOLS), set(protos) ^ set(L.SYMBOLS)

    def kind_c(arg):
        arg = arg.strip()
        if arg in ("void", ""):
            return None
        if "*" in arg:
            return "ptr"
        for k in ("long long", "double", "float", "int"):
            if re.search(rf"\b{k}\b", arg):
                return k
        raise AssertionError(arg)

    def kind_py(t):
        if t in (C.c_void_p, C.c_char_p) or (isinstance(t, type) and issubclass(t, C._Pointer)):
            return "ptr"
        return {C.c_longlong: "long long", C.c_double: "double", C.c_float: "float", C.c_int: "int"}[t]

    for name, (res, args) in L.SYMBOLS.items():
        want = [k for k in (kind_c(a) for a in protos[name].split(",")) if k is not None]
        got = [kind_py(t) for t in args]
        assert want == got, (name, want, got)
