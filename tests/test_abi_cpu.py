"""CPU-only checks of the drop-in boundary: libb200gs.so loads without a GPU, exports every entry point that
include/b200gs.h declares (and nothing in the header is missing from the ctypes table), and the argument validation /
error-reporting contract of the C ABI holds (bad arguments are rejected BEFORE any CUDA call: no compute here)."""
import ctypes
import os
import re

import pytest

from conftest import ROOT

HEADER = os.path.join(ROOT, "include", "b200gs.h")


@pytest.fixture(scope="module")
def lib():
    from b200gs import _lib
    if not os.path.exists(_lib.LIB_PATH):   # the driver normally runs __graft_entry__.build() first
        import __graft_entry__
        __graft_entry__.build()
    return _lib


def _declared_symbols():
    text = open(HEADER).read()
    return sorted(set(re.findall(r"B200GS_API\s+[\w\s\*]+?\b(b200gs_\w+)\s*\(", text)))


def test_header_symbols_are_exported_and_bound(lib):
    declared = _declared_symbols()
    assert len(declared) >= 20
    handle = lib.lib()
    for name in declared:
        assert hasattr(handle, name), f"{name} declared in include/b200gs.h but not exported by libb200gs.so"
    assert sorted(lib.EXPORTED_SYMBOLS) == declared, set(lib.EXPORTED_SYMBOLS) ^ set(declared)
    assert handle.b200gs_version() >= 100


def test_view_struct_layout_matches_header(lib):
    # 6 int32 + 10 float + 16 + 16 + 3 + 1 floats = 52 x 4 bytes; the kernel parameter block relies on this layout
    assert ctypes.sizeof(lib.B200gsView) == 208
    assert lib.B200gsView.viewmatrix.offset == 64 and lib.B200gsView.projmatrix.offset == 128 and lib.B200gsView.campos.offset == 192


def test_argument_validation_without_gpu(lib):
    L = lib.lib()
    v = lib.B200gsView()
    v.width, v.height, v.mode, v.sh_degree, v.sh_stride = 64, 64, 0, 3, 16
    # unsupported SH degree
    assert L.b200gs_sh_fwd(5, 36, 10, None, None, None, None) == -1
    assert b"degree" in L.b200gs_last_error()
    # bad mode
    v.mode = 7
    assert L.b200gs_project_fwd(ctypes.byref(v), 0, *([None] * 13), None) == -1
    assert b"mode" in L.b200gs_last_error()
    v.mode = 1
    # NULL pointers with n > 0
    assert L.b200gs_project_fwd(ctypes.byref(v), 5, *([None] * 13), None) == -1
    assert b"NULL" in L.b200gs_last_error() or b"must not be NULL" in L.b200gs_last_error()
    # sh_stride smaller than (degree+1)^2
    v.sh_stride = 4
    dummy = ctypes.c_void_p(16)
    assert L.b200gs_project_fwd(ctypes.byref(v), 5, dummy, dummy, dummy, dummy, *([dummy] * 9), None) == -1
    assert b"sh_stride" in L.b200gs_last_error()
    # unsupported channel count / bad image size in the blend entry points
    assert L.b200gs_blend_fwd(0, 0, 64, 3, *([None] * 7), None, 1, 1, None, None, None, None) == -1
    # [n,12] row buffers that are not 16-byte aligned (every other pointer is a non-NULL dummy)
    d16, d8 = ctypes.c_void_p(16), ctypes.c_void_p(8)
    assert L.b200gs_blend_fwd_rows(0, 64, 64, d16, d16, d8, d16, d16, 3, 1, d16, d16, d16, None) == -1
    assert b"aligned" in L.b200gs_last_error()
    for rows, v_rows in ((d8, d16), (d16, d8)):
        assert L.b200gs_blend_bwd_rows(0, 64, 64, d16, d16, rows, d16, d16, d16, d16, 3, 1, d16, 1.0, 1.0, v_rows, None) == -1
        assert b"aligned" in L.b200gs_last_error()
    assert L.b200gs_bin_count_rows(0, 64, 64, 1, d8, 1, d16, 1 << 20, d16, None, 0, None, None, 0) == -1
    assert b"aligned" in L.b200gs_last_error()
    # n = 0 is a valid no-op everywhere that takes a count
    v.sh_stride = 16
    assert L.b200gs_project_fwd(ctypes.byref(v), 0, *([None] * 13), None) == 0
    assert L.b200gs_sh_fwd(3, 16, 0, None, None, None, None) == 0


def test_no_fallback_when_library_missing(lib, monkeypatch):
    """The product path must fail loudly without the CUDA library — no torch / oracle fallback."""
    monkeypatch.setattr(lib, "_lib", None)
    monkeypatch.setattr(lib, "LIB_PATH", os.path.join(ROOT, "does", "not", "exist.so"))
    with pytest.raises(lib.B200gsError):
        lib.lib()


def test_product_does_not_import_oracle():
    pkg = os.path.join(ROOT, "gaussian-splatting-lightning_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith(".py"):
                src = open(os.path.join(dirpath, f)).read()
                assert "oracle" not in re.sub(r'"""[\s\S]*?"""|#.*', "", src), f"{f} references oracle/"


def test_every_python_call_site_passes_the_declared_number_of_arguments():
    """ctypes only reports a wrong argument count when the call runs, i.e. on the GPU box: check the call sites of the host code
    statically against the signature table (a call through *args / **kwargs is skipped)."""
    import ast
    import glob
    from b200gs import _lib
    sig = _lib._SIGNATURES
    pkg = os.path.join(ROOT, "gaussian-splatting-lightning_b200")
    files = glob.glob(os.path.join(pkg, "*.py")) + glob.glob(os.path.join(pkg, "compat", "*.py")) + [os.path.join(ROOT, "bench.py")] \
        + glob.glob(os.path.join(ROOT, "tests", "*.py")) + glob.glob(os.path.join(ROOT, "profiles", "tools", "*.py"))
    checked = 0
    for path in files:
        tree = ast.parse(open(path).read(), filename=path)
        for node in ast.walk(tree):
            if isinstance(node, ast.Call) and isinstance(node.func, ast.Attribute) and node.func.attr in sig:
                if any(isinstance(a, ast.Starred) for a in node.args) or node.keywords:
                    continue
                want = len(sig[node.func.attr][1])
                assert len(node.args) == want, f"{os.path.relpath(path, ROOT)}:{node.lineno}: {node.func.attr} called with {len(node.args)} arguments, declared {want}"
                checked += 1
    assert checked > 40


def test_every_entry_point_has_a_caller_outside_the_tests():
    """Every symbol of the ctypes table is reached from the package, bench.py or __graft_entry__.py: as an attribute of the library
    handle (`L.b200gs_x(...)`) or by name through getattr.  An entry point that only tests call is dead ABI: delete it with its
    prototype, wrapper and table entry."""
    import ast
    import glob
    from b200gs import _lib
    pkg = os.path.join(ROOT, "gaussian-splatting-lightning_b200")
    files = glob.glob(os.path.join(pkg, "**", "*.py"), recursive=True) + [os.path.join(ROOT, "bench.py"), os.path.join(ROOT, "__graft_entry__.py")]
    used = set()
    for path in files:
        for node in ast.walk(ast.parse(open(path).read(), filename=path)):
            if isinstance(node, ast.Attribute):
                used.add(node.attr)
            elif (isinstance(node, ast.Call) and isinstance(node.func, ast.Name) and node.func.id == "getattr" and len(node.args) >= 2
                  and isinstance(node.args[1], ast.Constant)):
                used.add(node.args[1].value)
    unused = sorted(set(_lib._SIGNATURES) - used)
    assert not unused, f"entry points without a caller in the package, bench.py or __graft_entry__.py: {unused}"


def test_header_prototypes_and_ctypes_table_agree_on_argument_counts(lib):
    """Every prototype of include/b200gs.h has as many parameters as its entry of the ctypes signature table (a drifted table only
    fails when the call runs, i.e. on the GPU box)."""
    text = re.sub(r"/\*.*?\*/", " ", open(HEADER).read(), flags=re.S)       # comments may contain commas and parentheses
    protos = re.findall(r"B200GS_API\s+[\w\s\*]+?\b(b200gs_\w+)\s*\(([^;]*?)\)\s*;", text, flags=re.S)
    assert len(protos) == len(lib.EXPORTED_SYMBOLS)
    for name, args in protos:
        args = args.strip()
        n = 0 if args in ("", "void") else len([a for a in args.split(",") if a.strip()])
        assert n == len(lib._SIGNATURES[name][1]), f"{name}: header has {n} parameters, ctypes table {len(lib._SIGNATURES[name][1])}"
