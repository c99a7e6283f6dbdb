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


# --- argument checks of every view-taking entry point ----------------------------------------------------------------------------------
# One row per failing call: (entry point, arguments, exact return code, name the message must contain, whether it must say "null").
# Views are _V(...) (ptr defaults to a fake 16-byte aligned address), other pointers _P; None is NULL.  Rows with two faults whose codes
# differ pin the order of the checks.  The table runs in a subprocess with the GPUs hidden: a call that wrongly passes validation then
# fails at its first CUDA call with -3 instead of launching on fake pointers.
_P = 0x10000


class _V:
    def __init__(self, n=2, h=8, w=8, c=64, pitch=None, off=0, ptr=_P):
        self.f = (ptr, n, h, w, c, c + off if pitch is None else pitch, off)


class _F(float):  # passed as a C float
    pass


class _I64(int):  # passed as an int64_t
    pass


def _capi_rows():
    I, U, C = -1, -2, -3
    v, v4 = _V(), _V(h=4, w=4)
    rows = []

    def row(fn, args, code, who=None, null=False):
        rows.append((fn, args, code, who or fn, null))

    # conv_api.cu: forward
    fwd = lambda x=v, w=_P, z=v, k=3, s=1, sm=None, sq=None: [x, w, z, k, s, sm, sq, None]
    row("conv2d_fwd", fwd(x=None), I, null=True)
    row("conv2d_fwd", fwd(x=None, s=3), I)
    row("conv2d_fwd", fwd(x=_V(n=0)), I)
    row("conv2d_fwd", fwd(z=_V(c=12)), I)
    row("conv2d_fwd", fwd(s=3), U)
    row("conv2d_fwd", fwd(s=2), I)  # output grid is not the input grid / 2
    row("conv2d_fwd", fwd(sm=_P), I)
    row("conv2d_fwd", fwd(sm=_P, s=3), U)
    row("conv2d_fwd", fwd(w=None), I, null=True)
    row("conv2d_fwd", fwd(k=5), U)
    row("conv2d_fwd", fwd(x=_V(c=8), z=_V(c=8)), U)  # input channels not a multiple of 16
    fold = lambda x=v, z=v, f=2: [x, _P, z, 3, 1, _P, _P, f, None]
    row("conv2d_fwd_fold", fold(f=0), I)
    row("conv2d_fwd_fold", fold(z=None), I)
    row("conv2d_fwd_fold", fold(z=_V(c=24), f=16), I)
    row("conv2d_fwd_fold", fold(x=None), I, who="conv2d_fwd", null=True)
    for fn in ("conv2d_bn_silu_fwd", "conv2d_affine_fwd"):
        ep = lambda x=v, w=_P, sc=_P, r=None, o=v, s=1: [x, w, sc, _P, r, o, 3, s, None]
        row(fn, ep(x=None), I, null=True)
        row(fn, ep(x=None, s=3), I)
        row(fn, ep(o=_V(pitch=60)), I)
        row(fn, ep(r=_V(c=64, pitch=32)), I)
        row(fn, ep(s=3), U)
        row(fn, ep(o=v4), I)
        row(fn, ep(r=_V(c=32)), I)
        row(fn, ep(r=_V(c=32), s=3), U)
        row(fn, ep(w=None), I, null=True)
    row("conv2d_bn_silu_fwd", [v, _P, None, _P, None, v, 3, 1, None], I, null=True)
    row("conv2d_bn_silu_fwd", [v, _P, _P, None, None, v, 3, 3, None], I)  # the null scale / shift is reported before the stride
    relu = lambda x=v, w=_P, o=v, k=3, s=1: [x, w, _P, o, k, s, None]
    row("conv2d_relu_fwd", relu(x=None), I, null=True)
    row("conv2d_relu_fwd", relu(o=None, s=3), I, null=True)
    row("conv2d_relu_fwd", relu(s=3), U)
    row("conv2d_relu_fwd", relu(s=2), I)
    row("conv2d_relu_fwd", relu(w=None), I, null=True)
    row("conv2d_relu_fwd", relu(w=None, k=5), I, null=True)
    row("conv2d_relu_fwd", relu(k=2), U)  # 2x2 kernels need stride 2
    row("linear_relu_fwd", [None, _P, _P, v, None], I, who="conv2d_relu_fwd", null=True)
    row("linear_relu_fwd", [v, _P, _P, v4, None], I, who="conv2d_relu_fwd")
    for fn, bias in (("conv1x1_nchw_f32", [_P]), ("conv1x1_nchw_f32_batched", [])):
        ep = lambda x=_V(h=16, w=16), w=_P, co=16, o=_P: [x, w] + bias + [co, o, None]
        row(fn, ep(x=None), I, null=True)
        row(fn, ep(x=_V(h=16, w=16, off=4)), I)
        row(fn, ep(o=None), I)
        row(fn, ep(co=0), I)
        row(fn, ep(co=129), I)
        row(fn, ep(x=_V(n=1, h=65536, w=32768)), U)
        row(fn, ep(x=_V(n=1, h=65536, w=32768), co=0), I)
        row(fn, ep(x=_V(h=16, w=16, c=8)), U)
        row(fn, ep(w=None), I, null=True)
    row("conv1x1_nchw_f32_batched", [_V(h=10, w=10), _P, 16, _P, None], U)  # a 128-pixel tile would span images
    row("conv1x1_nchw_f32_batched", [_V(h=10, w=10, c=8), _P, 16, _P, None], U)
    gelu = lambda x=v, u=None, h=v: [x, _P, _P, u, h, None]
    row("linear_gelu_fwd", gelu(x=None), I, null=True)
    row("linear_gelu_fwd", gelu(h=_V(c=0)), I)
    row("linear_gelu_fwd", gelu(u=_V(off=8, pitch=64)), I)
    row("linear_gelu_fwd", gelu(h=v4), I)
    row("linear_gelu_fwd", gelu(u=_V(pitch=128)), I)
    row("linear_gelu_fwd", [v, None, _P, None, v, None], I, null=True)
    for fn, split in (("conv1x1_bias_f32", []), ("conv1x1_bias_f32_split", [8, 2])):
        xs = _V(c=64, pitch=128) if split else v
        ep = lambda x=xs, sp=split, b=_P, co=85, at=64, ao=0, ct=85, cf=0: [x] + sp + [_P, b, co, _P, at, ao, ct, cf, None]
        row(fn, ep(x=None), I, null=True)
        row(fn, ep(b=None), I)
        row(fn, ep(co=129), I)
        row(fn, ep(ao=8), I)  # 8 + 64 anchors > 64
        row(fn, ep(cf=1), I)
        row(fn, ep(x=_V(c=8, pitch=128) if split else _V(c=8)), U)
    row("conv1x1_bias_f32_split", [xs, 0, 2, _P, _P, 85, _P, 64, 0, 85, 0, None], I)
    row("conv1x1_bias_f32_split", [xs, 8, 4, _P, _P, 85, _P, 64, 0, 85, 0, None], I)
    row("conv1x1_bias_f32_split", [_V(c=64, pitch=64), 8, 2, _P, _P, 85, _P, 64, 0, 85, 0, None], I)  # plane 1 beyond the pitch
    row("conv1x1_bias_f32_split", [xs, 8, 2, None, _P, 85, _P, 64, 0, 85, 0, None], I, null=True)
    spl = lambda x=_V(c=64, pitch=192), lo=64, pl=3, w=_P, z=_P, zp=64, s=1: [x, lo, pl, w, 64, 3, s, z, zp, 0, None]
    row("conv2d_fwd_split", spl(x=None), I, null=True)
    row("conv2d_fwd_split", spl(z=None), I)
    row("conv2d_fwd_split", spl(lo=0), I)
    row("conv2d_fwd_split", spl(zp=32), I)
    row("conv2d_fwd_split", spl(zp=32, s=3), I)
    row("conv2d_fwd_split", spl(s=3), U)
    row("conv2d_fwd_split", spl(pl=1), I)
    row("conv2d_fwd_split", spl(lo=96), I)  # plane 2 beyond the pitch
    row("conv2d_fwd_split", spl(w=None), I, null=True)
    # conv_api.cu: data and weight gradients
    dg = lambda dz=v, w=_P, dx=v, a=None, k=3, s=1: [dz, w, dx, a, k, s, None]
    row("conv2d_dgrad", dg(dz=None), I, null=True)
    row("conv2d_dgrad", dg(dx=_V(w=0)), I)
    row("conv2d_dgrad", dg(a=_V(c=64, pitch=32)), I)
    row("conv2d_dgrad", dg(w=None), I, null=True)
    row("conv2d_dgrad", dg(w=None, k=5), I, null=True)
    row("conv2d_dgrad", dg(k=5), U)
    row("conv2d_dgrad", dg(s=2), I)
    row("conv2d_dgrad", dg(a=_V(c=32)), I)
    row("conv2d_dgrad", dg(dz=_V(c=8)), U)
    row("conv2d_dgrad", dg(dz=_V(c=8), s=2), I)
    row("linear_dgrad_gelu", [v, _P, None, v, _P, None], I, null=True)
    row("linear_dgrad_gelu", [v, _P, v, _V(pitch=128), _P, None], I)
    row("linear_dgrad_gelu", [None, _P, v, v, _P, None], I, who="conv2d_dgrad", null=True)
    row("linear_dgrad_relu", [v, _P, v, None, _P, None], I, null=True)
    row("linear_dgrad_relu", [v, _P, _V(c=32), v, _P, None], I)
    row("linear_dgrad_relu", [v, None, v, v, _P, None], I, who="conv2d_dgrad", null=True)
    wgw = lambda x=v, dz=v, k=3, s=1: [x, dz, k, s]
    row("conv2d_wgrad_workspace", wgw(x=None), I, who="conv2d_wgrad", null=True)
    row("conv2d_wgrad_workspace", wgw(k=5), U, who="conv2d_wgrad")
    row("conv2d_wgrad_workspace", wgw(s=2), I, who="conv2d_wgrad")
    row("conv2d_wgrad_workspace", wgw(x=_V(c=24)), U, who="conv2d_wgrad")
    row("conv2d_wgrad_workspace", wgw(dz=_V(c=48, pitch=64)), U, who="conv2d_wgrad")  # 48 of a 64-channel pitch: boxes of 32 overshoot
    wg = lambda x=v, dz=v, cr=64, g=_P, ws=_P, nb=1 << 30: [x, dz, 3, 1, cr, g, 0, ws, _I64(nb), None]
    row("conv2d_wgrad", wg(dz=None), I, null=True)
    row("conv2d_wgrad", wg(g=None), I, null=True)
    row("conv2d_wgrad", wg(ws=None, x=_V(c=24)), U)
    row("conv2d_wgrad", wg(cr=0), I)
    row("conv2d_wgrad", wg(cr=65), I)
    row("conv2d_wgrad", wg(nb=16), I)
    wgg = lambda x=v, k=3, grp=4: [x, v, k, 1, 64, grp, _P, 0, _P, _I64(1 << 30), None]
    row("conv2d_wgrad_grouped", wgg(grp=1), I)
    row("conv2d_wgrad_grouped", wgg(grp=1, k=5), I)
    row("conv2d_wgrad_grouped", wgg(k=1), U)
    row("conv2d_wgrad_grouped", wgg(x=_V(c=64, pitch=128)), U)
    row("conv2d_wgrad_grouped", wgg(x=None), I, who="conv2d_wgrad", null=True)

    # elementwise.cu
    bna = lambda z=v, sc=_P, r=None, o=v, up=None: [z, sc, _P, r, o, up, None]
    row("bn_apply_silu", bna(z=None), I, null=True)
    row("bn_apply_silu", bna(o=_V(pitch=60)), I)
    row("bn_apply_silu", bna(r=_V(off=4)), I)
    row("bn_apply_silu", bna(up=_V(h=0)), I)
    row("bn_apply_silu", bna(sc=None), I, null=True)
    row("bn_apply_silu", bna(r=v4), I)
    row("bn_apply_silu", bna(up=v), I)
    row("bn_apply_silu", bna(z=_V(c=2056), o=_V(c=2056)), U)
    row("bn_apply_silu", bna(z=_V(c=2056), o=_V(c=2056), sc=None), I, null=True)
    row("bn_apply_silu", bna(z=_V(c=2056), o=_V(c=1024)), I)
    bnt = lambda z=v, sm=_P, rm=_P, rv=_P, o=v: [z, sm, _P, _I64(128), _P, _P, _F(1e-3), _F(0.03), rm, rv, _P, _P, _P, _P, None, o, None, None]
    row("bn_train_apply_silu", bnt(sm=None), I, null=True)
    row("bn_train_apply_silu", bnt(rv=None), I)
    row("bn_train_apply_silu", bnt(rm=None, rv=None, z=None), I, who="bn_apply_silu", null=True)
    row("bn_train_apply_silu", bnt(o=v4), I, who="bn_apply_silu")
    bwd = lambda z=v, da=v, da2=None, up=None, sc=_P, dz=v, dg=None: [z, da, da2, up, sc, _P, _P, _P, _P, _P, dz, dg, None, 0, None]
    row("bn_silu_bwd", bwd(da=None), I, null=True)
    row("bn_silu_bwd", bwd(dz=_V(c=4)), I)
    row("bn_silu_bwd", bwd(da2=_V(off=4, pitch=72)), I)
    row("bn_silu_bwd", bwd(up=_V(pitch=8)), I)
    row("bn_silu_bwd", bwd(sc=None), I, null=True)
    row("bn_silu_bwd", bwd(dg=_P), I, null=True)
    row("bn_silu_bwd", bwd(da2=v4), I)
    row("bn_silu_bwd", bwd(up=v), I)
    c2k = _V(c=2056)
    row("bn_silu_bwd", bwd(z=c2k, da=c2k, dz=c2k), U)
    row("bn_silu_bwd", bwd(z=c2k, da=c2k, dz=c2k, sc=None), I, null=True)
    spp = lambda x=v, o5=v, o13=v: [x, o5, v, o13, _P, None]
    row("spp_pool", spp(x=None), I, null=True)
    row("spp_pool", spp(o13=_V(c=60)), I)
    row("spp_pool", spp(o5=v4), I)
    sppb = lambda d0=v, am=_P, dx=v: [d0, v, v, v, am, _P, dx, None]
    row("spp_pool_bwd", sppb(dx=None), I, null=True)
    row("spp_pool_bwd", sppb(d0=_V(n=-1)), I)
    row("spp_pool_bwd", sppb(am=None), I, null=True)
    row("spp_pool_bwd", sppb(d0=v4), I)
    row("copy_view", [None, v, None], I, null=True)
    row("copy_view", [v, _V(c=8, pitch=64, off=60), None], I)
    row("copy_view", [v, v4, None], I)

    # convnext.cu
    dw = lambda x=v, w=_P, a=None, o=v: [x, w, _P, a, o, 0, None]
    row("dwconv7", dw(x=None), I, null=True)
    row("dwconv7", dw(x=_V(c=48)), I)  # channel slices of 32
    row("dwconv7", dw(o=_V(c=64, pitch=80)), I)
    row("dwconv7", dw(a=_V(c=4)), I)
    row("dwconv7", dw(w=None), I, null=True)
    row("dwconv7", dw(a=v4), I)
    row("dwconv7", dw(o=_V(c=32)), I)
    dww = lambda x=v, dy=v, g=_P: [x, dy, g, _P, 0, _P, None]
    row("dwconv7_wgrad", dww(dy=None), I, null=True)
    row("dwconv7_wgrad", dww(x=_V(c=48)), I)
    row("dwconv7_wgrad", dww(g=None), I)
    row("dwconv7_wgrad", dww(dy=v4), I)
    lnf = lambda x=v, g=_P, y=v: [x, g, _P, _F(1e-6), y, _P, None]
    row("layernorm_fwd", lnf(x=None), I, null=True)
    row("layernorm_fwd", lnf(y=_V(c=6)), I)  # channels in fours
    row("layernorm_fwd", lnf(g=None), I)
    row("layernorm_fwd", lnf(y=v4), I)
    lnb = lambda dy=v, st=_P, a=None, dx=v: [dy, v, st, _P, a, dx, _P, _P, 0, _P, None]
    row("layernorm_bwd", lnb(dx=None), I, null=True)
    row("layernorm_bwd", lnb(dy=_V(c=64, pitch=66)), I)
    row("layernorm_bwd", lnb(a=_V(off=4, pitch=64)), I)
    row("layernorm_bwd", lnb(st=None), I, null=True)
    row("layernorm_bwd", lnb(a=v4), I)
    row("colsum", [None, _F(1.0), _P, 0, _P, None], I, null=True)
    row("colsum", [_V(c=12), _F(1.0), _P, 0, _P, None], I)
    row("colsum", [v, _F(1.0), None, 0, _P, None], I, null=True)
    row("colsum", [_V(c=2056), _F(1.0), _P, 0, _P, None], U)
    row("colsum", [_V(c=2056), _F(1.0), None, 0, _P, None], I, null=True)
    pf = lambda im=_P, h=32, o=_V(n=2, h=8, w=8, c=48): [im, 0, 2, h, 32, o, None]
    row("patchify4", pf(o=None), I, null=True)
    row("patchify4", pf(o=_V(c=48, pitch=44)), I)
    row("patchify4", pf(im=None), I)
    row("patchify4", pf(h=30), I)
    row("patchify4", pf(o=v), I)
    row("add", [v, None, v, None], I, null=True)
    row("add", [v, v, _V(c=0), None], I)
    row("add", [v, v4, v, None], I)
    row("sigmoid", [v, _V(c=64, pitch=68), None], I)
    row("sigmoid", [None, v, None], I, null=True)
    row("sigmoid", [v, v4, None], I)
    iam = lambda raw=_P, o=_V(n=1, h=1, w=100, c=64): [raw, _P, 100, 64, o, None]
    row("iam_normalize", iam(o=None), I, null=True)
    row("iam_normalize", iam(o=_V(n=1, h=1, w=100, c=64, pitch=60)), I)
    row("iam_normalize", iam(raw=None), I)
    row("iam_normalize", iam(o=v), I)

    # attention.cu: [B][1][L][heads x 32] token views
    t = _V(n=2, h=1, w=100, c=64)
    af = lambda q=t, k=t, vv=t, o=t: [q, k, vv, None, _F(0.125), o, _P, None]
    row("attention_fwd", af(q=None), I, null=True)
    row("attention_fwd", af(k=_V(n=2, h=2, w=100, c=64)), I)
    row("attention_fwd", af(vv=_V(n=2, h=1, w=100, c=48)), I)
    row("attention_fwd", af(o=_V(n=2, h=1, w=100, c=64, pitch=60)), I)
    row("attention_fwd", af(o=_V(n=2, h=1, w=50, c=64)), I)
    afd = lambda q=t: [q, t, t, None, _F(0.125), t, _P, _F(0.1), 7, None]
    row("attention_fwd_dropout", afd(q=None), I, who="attention_fwd", null=True)
    ab = lambda q=t, dout=t, lse=_P, dq=t, dk=t, dv=t: [q, t, t, t, dout, None, _F(0.125), lse, dq, dk, dv, _P, None]
    row("attention_bwd", ab(dv=None), I, null=True)
    row("attention_bwd", ab(dout=_V(n=2, h=1, w=100, c=64, off=8, pitch=64)), I)
    row("attention_bwd", ab(dq=_V(n=2, h=1, w=100, c=16)), I)
    row("attention_bwd", ab(lse=None), I, null=True)
    row("attention_bwd", ab(dq=_V(n=2, h=1, w=50, c=64)), I)
    row("attention_bwd", ab(dk=_V(n=2, h=1, w=50, c=64)), I)
    abd = lambda q=t: [q, t, t, t, t, None, _F(0.125), _P, t, t, t, _P, _F(0.1), 7, None]
    row("attention_bwd_dropout", abd(q=_V(n=0, h=1, w=100, c=64)), I, who="attention_bwd")
    do = lambda x=t, r=None, o=t, p=0.1: [x, r, o, _F(p), 7, _F(1.0), None]
    row("dropout", do(x=None), I, null=True)
    row("dropout", do(r=_V(n=2, h=1, w=100, c=64, off=4, pitch=72)), I)
    row("dropout", do(o=_V(n=2, h=1, w=100, c=40)), I)
    row("dropout", do(r=_V(n=2, h=1, w=99, c=64)), I)
    big = _V(n=65536, h=1, w=1024, c=128)
    row("dropout", do(x=big, o=big), U)
    row("dropout", do(x=big, o=big, p=1.0), U)
    row("dropout", do(p=1.0), I)

    # strict.cu: split views (plane j `lo` channels after plane 0)
    s = _V(c=64, pitch=192)
    sb = lambda z=_P, zp=64, r=None, o=s, up=None, pl=3: [z, zp, 0, _P, _P, r, 64, o, 64, up, 64, pl, None]
    row("strict_bn_apply_silu", sb(z=None), I, null=True)
    row("strict_bn_apply_silu", sb(o=None), I, null=True)
    row("strict_bn_apply_silu", sb(o=_V(c=64, pitch=192, ptr=None)), I, null=True)
    row("strict_bn_apply_silu", sb(o=_V(n=0, c=64, pitch=192)), I)
    row("strict_bn_apply_silu", sb(pl=4), I)
    row("strict_bn_apply_silu", sb(o=_V(c=64, pitch=160)), I)
    row("strict_bn_apply_silu", sb(zp=32), I)
    row("strict_bn_apply_silu", sb(r=_V(c=64, pitch=128)), I)
    row("strict_bn_apply_silu", sb(r=_V(h=4, w=4, c=64, pitch=192)), I)
    row("strict_bn_apply_silu", sb(up=_V(h=0, c=64, pitch=192)), I)
    row("strict_bn_apply_silu", sb(up=s), I)
    sp = lambda x=s, o5=s, o9=s, o13=s, lo=64, pl=3: [x, o5, o9, o13, lo, pl, None]
    row("strict_spp_pool", sp(o9=None), I, null=True)
    row("strict_spp_pool", sp(lo=0), I)
    row("strict_spp_pool", sp(x=_V(c=64, pitch=100)), I)
    row("strict_spp_pool", sp(o13=_V(c=32, pitch=192)), I)
    row("strict_spp_pool", sp(o5=_V(h=4, w=4, c=64, pitch=192)), I)
    return rows


def _run_capi_rows():
    """runs every row of _capi_rows() and returns [(return code, yb200_last_error()), ...]"""
    from yolov7_d2_b200 import capi

    L = capi.lib()

    def arg(a):
        if isinstance(a, _V):
            return ctypes.byref(capi.Act(*a.f))
        if isinstance(a, _F):
            return ctypes.c_float(a)
        if isinstance(a, _I64):
            return ctypes.c_int64(a)
        return ctypes.c_void_p(a) if a == _P else a

    out = []
    for fn, args, _, _, _ in _capi_rows():
        rc = getattr(L, "yb200_" + fn)(*[arg(a) for a in args])
        out.append((rc, L.yb200_last_error().decode()))
    return out


def test_every_view_taking_entry_point_rejects_bad_arguments():
    """exact return codes, and messages that name the entry point, for every argument check of the view-taking entry points"""
    import json
    import subprocess
    import sys

    env = dict(os.environ, CUDA_VISIBLE_DEVICES="", PYTHONPATH=os.pathsep.join([ROOT] + [p for p in [os.environ.get("PYTHONPATH")] if p]))
    r = subprocess.run([sys.executable, os.path.abspath(__file__)], capture_output=True, text=True, env=env, cwd=ROOT, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    got = json.loads(r.stdout.strip().splitlines()[-1])
    rows = _capi_rows()
    assert len(got) == len(rows) and len(rows) > 200
    bad = []
    for i, ((fn, args, code, who, null), (rc, msg)) in enumerate(zip(rows, got)):
        if rc != code or who not in msg or (null and "null" not in msg):
            bad.append(f"row {i} yb200_{fn}: returned {rc} ({msg!r}), expected {code} naming {who!r}" + (" with 'null'" if null else ""))
    assert not bad, "\n".join(bad)


if __name__ == "__main__":
    import json
    import sys

    sys.path.insert(0, ROOT)
    print(json.dumps(_run_capi_rows()))
