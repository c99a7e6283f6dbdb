"""CPU checks of the C-ABI boundary: the library builds, loads, and exports every symbol include/yb200.h declares."""
import ctypes
import os

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
    from yolov7_d2_b200 import build, capi

    if build.find_nvcc() is None and not os.path.exists(capi.LIB_PATH):
        pytest.skip("no nvcc and no prebuilt libyb200.so")
    build.build()
    names = capi.declared_symbols()
    assert len(names) >= 20 and "yb200_conv2d_fwd" in names and "yb200_postprocess_nms" in names
    lib = ctypes.CDLL(capi.LIB_PATH)
    for n in names:
        assert hasattr(lib, n), n
    assert lib.yb200_version() == 100


def test_argument_validation_without_gpu():
    """invalid arguments are rejected on the host before any CUDA call (no GPU needed)"""
    from yolov7_d2_b200 import capi

    L = capi.lib()
    a = capi.Act(0, 1, 8, 8, 16, 16, 0)
    assert L.yb200_conv2d_fwd(ctypes.byref(a), None, ctypes.byref(a), 3, 1, None, None, None) == -1
    assert b"null" in L.yb200_last_error()
    assert L.yb200_simota_workspace(0, 8400) < 0 and L.yb200_nms_workspace(4, 70000) < 0
    assert L.yb200_simota_workspace(64, 8400) > 0 and L.yb200_nms_workspace(64, 8400) > 0


def test_sass_contains_hopper_tensor_and_tma_instructions():
    import shutil
    import subprocess

    from yolov7_d2_b200 import capi

    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not available")
    sass = subprocess.run(["cuobjdump", "-sass", capi.LIB_PATH], capture_output=True, text=True).stdout
    assert "HGMMA" in sass and "UTMALDG" in sass, "wgmma / TMA instructions missing from the sm_90a build"


def test_attention_and_gemm_kernels_use_wgmma():
    """per kernel: the attention core, the convolution GEMM and the weight-gradient GEMM must themselves contain warpgroup MMA and TMA
    instructions (not just some other kernel of the library)"""
    import re
    import shutil
    import subprocess

    from yolov7_d2_b200 import capi

    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not available")
    sass = subprocess.run(["cuobjdump", "-sass", capi.LIB_PATH], capture_output=True, text=True).stdout
    funcs = {}
    for part in re.split(r"\n\s*Function : ", sass)[1:]:
        name, _, body = part.partition("\n")
        funcs[name.strip()] = body
    att = [b for n, b in funcs.items() if "attention_fwd_kernel" in n or "attention_bwd_kv_kernel" in n or "attention_bwd_q_kernel" in n]
    assert len(att) == 6, "attention kernels not found in the library"
    assert all("HGMMA" in b and "UTMALDG" in b and "MUFU.EX2" in b for b in att)
    conv = [b for n, b in funcs.items() if "conv_gemm_persistent_kernel" in n]
    assert conv and all("HGMMA" in b and "UTMALDG" in b for b in conv)
    wg = [b for n, b in funcs.items() if "wgrad_gemm_kernel" in n]
    assert wg and all("HGMMA" in b and "UTMALDG" in b for b in wg)
    # programmatic dependent launch: every kernel of the library waits for its predecessor (griddepcontrol.wait = ACQBULK) and releases its
    # dependents (launch_dependents = PREEXIT)
    missing = [n for n, b in funcs.items() if "ACQBULK" not in b or "PREEXIT" not in b]
    assert not missing, missing[:5]


def test_extended_entry_points_validate_arguments_without_gpu():
    from yolov7_d2_b200 import capi

    L = capi.lib()
    a = capi.Act(0, 1, 1, 8, 64, 64, 0)
    assert L.yb200_attention_fwd(ctypes.byref(a), ctypes.byref(a), ctypes.byref(a), None, ctypes.c_float(1.0), ctypes.byref(a), None, None) != 0
    assert L.yb200_layernorm_fwd(ctypes.byref(a), None, None, ctypes.c_float(1e-6), ctypes.byref(a), None, None) != 0
    assert L.yb200_sgd_step(None, None, None, ctypes.c_int64(0), None, None, None, 0, ctypes.c_float(0), ctypes.c_float(0), ctypes.c_float(0), 0, 0,
                            ctypes.c_float(1), None, ctypes.c_float(0), None) != 0
    assert b"null" in L.yb200_last_error() or b"sgd_step" in L.yb200_last_error()


def test_public_header_is_plain_c():
    """the drop-in boundary is a C ABI: include/yb200.h must compile as C99 without any C++ or torch type"""
    import shutil
    import subprocess
    import tempfile

    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    with tempfile.TemporaryDirectory() as td:
        src = os.path.join(td, "h.c")
        with open(src, "w") as fh:
            fh.write('#include "yb200.h"\nint main(void) { return 0; }\n')
        r = subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-fsyntax-only", "-I", os.path.join(ROOT, "include"), src], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr


def test_every_python_call_site_matches_the_header_arity():
    """ctypes does not check argument counts: compare every `.yb200_*( ... )` call in the repo with the prototype in include/yb200.h"""
    import glob
    import re

    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "yb200.h")).read(), flags=re.S)
    arity = {}
    for m in re.finditer(r"\b(yb200_[a-z0-9_]+)\s*\(([^;{]*?)\)\s*;", hdr, flags=re.S):
        args = m.group(2).strip()
        arity[m.group(1)] = 0 if args in ("", "void") else len(args.split(","))

    def count_args(src, i):
        depth, j, n, seen = 1, i, 0, False
        while depth > 0:
            c = src[j]
            if c in "([{":
                depth += 1
            elif c in ")]}":
                depth -= 1
            elif c == "," and depth == 1:
                n += 1
            if depth >= 1 and not c.isspace() and c != ")":
                seen = True
            j += 1
        return n + 1 if seen else 0

    bad = []
    files = [f for pat in ("*.py", "yolov7_d2_b200/*.py", "tests/*.py", "tools/*.py") for f in glob.glob(os.path.join(ROOT, pat))]
    assert len(files) > 20
    for f in files:
        src = open(f).read()
        for m in re.finditer(r"\.(yb200_[a-z0-9_]+)\(", src):
            name = m.group(1)
            if name in arity and count_args(src, m.end()) != arity[name]:
                bad.append((os.path.relpath(f, ROOT), name, count_args(src, m.end()), arity[name]))
    assert not bad, bad


def test_product_never_imports_the_oracle():
    """oracle/ is test infrastructure: the package must not import it, and bench.py only inside its baseline legs (the reference arm, the
    stock-PyTorch library bar and the cpu_baseline block) -- never on the measured product path"""
    import glob
    import re

    for f in glob.glob(os.path.join(ROOT, "yolov7_d2_b200", "*.py")):
        assert not re.search(r"^\s*(from|import)\s+oracle\b", open(f).read(), flags=re.M), f
    src = open(os.path.join(ROOT, "bench.py")).read()
    hits = [m.start() for m in re.finditer(r"^\s*from oracle\b", src, flags=re.M)]
    assert len(hits) == 3
    for h, fn in zip(hits[:2], ("def run_reference", "def library_bar")):  # inside the two baseline functions
        assert src.rfind(fn, 0, h) == src.rfind("\ndef ", 0, h) + 1, fn
    assert "no_cpu_baseline" in src[src.rfind("\n    if ", 0, hits[2]):hits[2]]  # third one inside the cpu_baseline block


def test_every_pdl_launched_kernel_waits_for_its_predecessor():
    """launch_k (csrc/host_common.cuh) gives kernels the programmatic-stream-serialization attribute: such a kernel may be scheduled while its
    predecessor is still running, so it MUST execute griddepcontrol.wait (pdl_sync) before touching global memory.  Static check over the sources."""
    import glob
    import re

    root = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "yolov7_d2_b200", "csrc")
    src = {f: open(f).read() for f in glob.glob(os.path.join(root, "*.cu*"))}
    names = set()
    for s in src.values():
        names.update(m.group(1) for m in re.finditer(r"launch_k\(\s*([A-Za-z_]\w*)", s))
        names.update(m.group(1) for m in re.finditer(r"launch_k_opt\([^,]+,\s*([A-Za-z_]\w*)", s))
    names -= {"void", "kernel"}  # the declarations of launch_k / launch_k_opt themselves
    assert len(names) >= 50
    for n in sorted(names):
        bodies = []
        for s in src.values():
            for m in re.finditer(r"__global__[^;{]*?\b" + n + r"\s*\(", s, re.S):
                i, depth = m.end(), 1
                while depth:
                    depth += (s[i] == "(") - (s[i] == ")")
                    i += 1
                j = s.index("{", i)
                if s[i:j].strip():
                    continue
                k, d = j + 1, 1
                while d:
                    d += (s[k] == "{") - (s[k] == "}")
                    k += 1
                bodies.append(s[j:k])
        assert bodies, f"definition of kernel {n} not found"
        assert all("pdl_sync()" in b for b in bodies), f"kernel {n} is launched through launch_k but never calls pdl_sync()"
