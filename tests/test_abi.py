"""The C-ABI library loads (no GPU needed) and exports every symbol include/thb200.h declares; the ctypes
signature table covers exactly the declared functions.  No compute calls here."""
import os
import re

from theseus_b200 import _lib, build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    src = open(os.path.join(ROOT, "include", "thb200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(thb_[a-z0-9_]+)\s*\(", src)))


def test_library_builds_and_exports_declared_symbols():
    build.build(verbose=False)
    lib = _lib.load()
    names = _declared()
    assert len(names) >= 30
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/thb200.h but not exported by libthb200.so"
    assert sorted(_lib.SIGNATURES) == names
    assert lib.thb_version() >= 100
    assert lib.thb_compiled_arch() == 90
    # pure host-side query (no device access)
    ws = lib.thb_potrf_workspace_bytes(2, 130)  # L [2,256,256] + W [2,4,64,64] + flags/counters/tables
    assert ws % 256 == 0 and 2 * 256 * 256 * 8 + 2 * 4 * 64 * 64 * 8 < ws < 2 * 256 * 256 * 8 + 2 * 4 * 64 * 64 * 8 + 4096
    assert lib.thb_error_num_chunks(17) == 3


def test_header_is_plain_c99(tmp_path):
    """The drop-in boundary is a C ABI: include/thb200.h must compile as plain C (no C++-isms, no torch types)."""
    import shutil
    import subprocess
    gcc = shutil.which("gcc")
    if gcc is None:
        return
    src = tmp_path / "hdr.c"
    src.write_text('#include "thb200.h"\nint main(void) { thb_cost_group g; thb_sparse_lane_root r; (void)g; (void)r; return thb_version() > 0 ? 0 : 1; }\n')
    res = subprocess.run([gcc, "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", os.path.join(ROOT, "include"), "-fsyntax-only", str(src)],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr


def test_sass_is_hopper_and_uses_fp64_tensor_pipe():
    import shutil
    import subprocess
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        return
    out = subprocess.run([cuobjdump, "-lelf", _lib.lib_path()], capture_output=True, text=True).stdout
    assert "sm_90a" in out
    assert "sm_52" not in out and "sm_100" not in out  # sm_90a only: no multi-arch fat binary
    sass = subprocess.run([cuobjdump, "-sass", _lib.lib_path()], capture_output=True, text=True).stdout
    assert "chol_col_kernel" in sass and "DMMA" in sass and "LDGSTS" in sass


def test_product_does_not_import_oracle():
    pkg = os.path.join(ROOT, "theseus_b200")
    for dp, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".cpp")):
                txt = open(os.path.join(dp, f)).read()
                assert "import oracle" not in txt and "from oracle" not in txt, f


def test_ctypes_signatures_match_the_header_prototypes():
    """Every prototype of include/thb200.h parsed and compared with _lib.SIGNATURES argument by argument: count, struct-pointer types
    (a wrong POINTER(struct) makes ctypes refuse the call at run time -- on the GPU box), integer / floating scalar widths, return type."""
    import ctypes as C
    src = open(os.path.join(ROOT, "include", "thb200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    src = re.sub(r"typedef struct \w+ \{.*?\} \w+;", "", src, flags=re.S)
    structs = {"thb_cost_group": _lib.CostGroup, "thb_var_table": _lib.VarTable, "thb_gram_plan": _lib.GramPlan,
               "thb_sparse_plan": _lib.SparsePlanStruct, "thb_sparse_lane_plan": _lib.SparseLanePlanStruct,
               "thb_sparse_lane_root": _lib.SparseLaneRootStruct, "thb_sparse_lane_tiles": _lib.SparseLaneTilesStruct,
               "thb_sparse_lane_pieces": _lib.SparseLanePiecesStruct, "thb_front_plan": _lib.FrontPlanStruct}
    scalars = {"int64_t": C.c_int64, "int32_t": C.c_int32, "int": C.c_int32, "double": C.c_double, "float": C.c_float,
               "thb_stream_t": C.c_void_p, "uint8_t": C.c_uint8}
    protos = re.findall(r"\b(int64_t|int32_t|int|void|double)\s+(thb_[a-z0-9_]+)\s*\(([^)]*)\)\s*;", src)
    assert len(protos) == len(_lib.SIGNATURES), (len(protos), len(_lib.SIGNATURES))
    for ret, name, params in protos:
        res, args = _lib.SIGNATURES[name]
        assert res == {"int64_t": C.c_int64, "int32_t": C.c_int32, "int": C.c_int32, "void": None, "double": C.c_double}[ret], name
        plist = [p.strip() for p in params.split(",")] if params.strip() not in ("", "void") else []
        assert len(plist) == len(args), (name, len(plist), len(args))
        for i, (p, a) in enumerate(zip(plist, args)):
            ptype = re.sub(r"\s+\w+$", "", p).replace("const ", "").strip()    # drop the parameter name
            if ptype.endswith("*"):
                base = ptype.rstrip("*").strip()
                if base in structs:
                    assert a == C.POINTER(structs[base]), f"{name} argument {i}: header says {base}*, ctypes says {a}"
                elif base == "char":
                    assert a == C.c_char_p, f"{name} argument {i} ({p}): ctypes says {a}"
                elif base == "thb_symbolic*":      # thb_symbolic** out-parameter
                    assert a in (C.c_void_p, C.POINTER(C.c_void_p)), f"{name} argument {i} ({p}): ctypes says {a}"
                else:
                    assert a == C.c_void_p, f"{name} argument {i} ({p}): expected a raw pointer, ctypes says {a}"
            else:
                assert ptype in scalars, (name, p)
                assert a == scalars[ptype], f"{name} argument {i} ({p}): ctypes says {a}"
