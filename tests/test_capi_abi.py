"""CPU test: the C-ABI shared library loads without a GPU and exports every symbol include/hybvio_b200.h declares."""
import ctypes
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    src = open(os.path.join(ROOT, "include", "hybvio_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(hv_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    from hybvio_b200 import capi
    assert os.path.exists(capi.LIB_PATH), "build the library first: make (or __graft_entry__.build())"
    lib = ctypes.CDLL(capi.LIB_PATH)
    syms = declared_symbols()
    assert len(syms) >= 50
    missing = [s for s in syms if not hasattr(lib, s)]
    assert not missing, f"declared in include/hybvio_b200.h but not exported: {missing}"


def test_no_cpu_fallback_without_gpu():
    """On a box without a GPU the context must fail loudly (HV_ERR_NO_DEVICE), never fall back to a CPU path."""
    import torch
    from hybvio_b200 import capi
    lib = capi.load()
    if torch.cuda.is_available():
        return
    h = ctypes.c_void_p()
    rc = lib.hv_ctx_create(0, ctypes.byref(h))
    assert rc == -2 and b"no CPU fallback" in lib.hv_last_error()


def test_version_string():
    from hybvio_b200 import capi
    assert b"sm_90a" in capi.load().hv_version()


def test_header_is_plain_c99(tmp_path):
    """The boundary is a C ABI: include/hybvio_b200.h must compile as C (no C++-isms, no torch / CUDA types)."""
    import subprocess
    src = tmp_path / "hdr.c"
    src.write_text('#include "hybvio_b200.h"\nint main(void) { hv_camera_model c; hv_visual_update_params p; hv_track_result r; hv_ekf_op o; '
                   '(void)c; (void)p; (void)r; (void)o; return 0; }\n')
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I" + os.path.join(root, "include"), "-fsyntax-only", str(src)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr


def test_ctypes_structs_match_the_header(tmp_path):
    """hybvio_b200/capi.py mirrors the structs of include/hybvio_b200.h by hand: sizes and field offsets must agree with what
    the C compiler lays out."""
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, root)
    from hybvio_b200 import capi
    pairs = {"hv_camera_model": capi.CameraModel, "hv_track_obs": capi.TrackObs, "hv_track_model": capi.TrackModel,
             "hv_visual_update_params": capi.VisualUpdateParams, "hv_track_result": capi.TrackResult, "hv_ekf_op": capi.EkfOp,
             "hv_ekf_params": capi.EkfParams, "hv_lk_job": capi.LkJob}
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "hybvio_b200.h"', 'int main(void) {']
    for cname, py in pairs.items():
        lines.append(f'printf("{cname} size %zu\\n", sizeof({cname}));')
        for fname, _ in py._fields_:
            lines.append(f'printf("{cname} {fname} %zu\\n", offsetof({cname}, {fname}));')
    lines += ['return 0; }']
    src, exe = tmp_path / "layout.c", tmp_path / "layout"
    src.write_text("\n".join(lines))
    subprocess.check_call(["gcc", "-std=c99", "-I" + os.path.join(root, "include"), str(src), "-o", str(exe)])
    out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout
    got = {}
    for ln in out.splitlines():
        a, b, c = ln.split()
        got[(a, b)] = int(c)
    for cname, py in pairs.items():
        assert got[(cname, "size")] == ctypes.sizeof(py), cname
        for fname, _ in py._fields_:
            assert got[(cname, fname)] == getattr(py, fname).offset, (cname, fname)


def _c_category(decl, is_return=False):
    d = decl.strip()
    if "*" in d or "[" in d:
        return "ptr"
    toks = re.sub(r"\bconst\b", "", d).split()
    if not is_return and len(toks) > 1:
        toks = toks[:-1]                                    # parameter name
    return {"int": "int", "unsigned": "int", "double": "f64", "float": "f32", "size_t": "size", "long long": "i64", "void": "void"}[" ".join(toks)]


def _ctypes_category(t):
    if t is None:
        return "void"
    table = {ctypes.c_int: "int", ctypes.c_uint: "int", ctypes.c_double: "f64", ctypes.c_float: "f32", ctypes.c_size_t: "size",
             ctypes.c_longlong: "i64", ctypes.c_void_p: "ptr", ctypes.c_char_p: "ptr"}
    if t in table:
        return table[t]
    assert issubclass(t, (ctypes._Pointer, ctypes.Array)) or hasattr(t, "from_param"), t
    return "ptr"


def test_ctypes_prototypes_match_the_header():
    """Every prototype of include/hybvio_b200.h against the argtypes / restype hybvio_b200/capi.py binds: same number of
    arguments, same class (pointer, int, double, float, size_t, long long) at every position. A mismatch only shows up as a
    crash or a garbage argument on the GPU box, so it is checked here."""
    from hybvio_b200 import capi
    lib = capi.load()
    src = open(os.path.join(ROOT, "include", "hybvio_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    src = re.sub(r"//[^\n]*", "", src)
    protos = re.findall(r"^\s*((?:const\s+)?(?:long long|[A-Za-z_]\w*)\s*\**)\s*(hv_\w+)\s*\(([^;{]*?)\)\s*;", src, flags=re.M)
    assert len(protos) >= 70
    assert sorted(p[1] for p in protos) == declared_symbols()
    bad = []
    for ret, name, args in protos:
        f = getattr(lib, name)
        want = [] if args.strip() in ("", "void") else [_c_category(a) for a in args.split(",")]
        if f.argtypes is None:
            if want:
                bad.append((name, "no argtypes", want))
            continue
        got = [_ctypes_category(t) for t in f.argtypes]
        if got != want:
            bad.append((name, got, want))
        # ctypes' default restype is c_int
        if _ctypes_category(f.restype) != _c_category(ret, is_return=True):
            bad.append((name, "restype", f.restype, ret))
    assert not bad, bad


_NULL_PROBE = r"""
import ctypes, sys
sys.path.insert(0, {root!r})
from hybvio_b200 import capi
lib = capi.load()
for name in {names!r}:
    f = getattr(lib, name)
    args = []
    for t in (f.argtypes or []):
        if t in (ctypes.c_int, ctypes.c_uint, ctypes.c_size_t, ctypes.c_longlong):
            args.append(0)
        elif t in (ctypes.c_double, ctypes.c_float):
            args.append(0.0)
        else:
            args.append(None)
    print(name, flush=True)
    r = f(*args)
    print(name, "->", r, flush=True)
print("probe complete")
"""


def test_every_entry_point_survives_null_arguments():
    """No exceptions and no crashes across the boundary: every function of the header called with NULL handles / NULL pointers / zeros
    (in a child process, so that a crash is a test failure with the function's name and not the end of the test run). Functions that
    return a status must not report success for a NULL handle (destroy / release of NULL are no-ops, like free)."""
    import subprocess
    import sys
    names = declared_symbols()
    r = subprocess.run([sys.executable, "-c", _NULL_PROBE.format(root=ROOT, names=names)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "probe complete" in r.stdout, "crashed in " + r.stdout.strip().splitlines()[-1] + "\n" + r.stderr[-500:]
    results = dict(l.split(" -> ") for l in r.stdout.splitlines() if " -> " in l)
    noop_ok = {"hv_ctx_destroy", "hv_ekf_destroy", "hv_pyr_release", "hv_ingest_destroy", "hv_device_count", "hv_ctx_launch_count", "hv_ekf_was_stationary"}
    wrong = [n for n, v in results.items() if v.lstrip("-").isdigit() and int(v) >= 0 and n not in noop_ok]
    assert not wrong, f"status 0 for NULL arguments: {wrong}"


def test_every_environment_switch_of_the_library_is_documented():
    """Every getenv("HV_...") of the library / adapters appears in INTEGRATION.md's table of switches."""
    import glob
    names = set()
    for pat in ("hybvio_b200/csrc/*.cu", "hybvio_b200/csrc/*.cuh", "hybvio_b200/host/*.cpp", "hybvio_b200/host/*.cu", "hybvio_b200/*.py"):
        for f in glob.glob(os.path.join(ROOT, pat)):
            src = open(f).read()
            names |= set(re.findall(r'getenv\("(HV_[A-Z0-9_]+)"\)', src))
            names |= set(re.findall(r'environ(?:\.get\(|\[)"(HV_[A-Z0-9_]+)"', src))
    for pat in ("hybvio_b200/host/*.hpp",):
        for f in glob.glob(os.path.join(ROOT, pat)):
            names |= set(re.findall(r'getenv\("(HV_[A-Z0-9_]+)"\)', open(f).read()))
    assert 1 <= len(names) <= 4, sorted(names)          # round 1 had 19; the A/Bs that have been settled are gone
    doc = open(os.path.join(ROOT, "INTEGRATION.md")).read()
    missing = sorted(n for n in names if n not in doc)
    assert not missing, f"not documented in INTEGRATION.md: {missing}"
