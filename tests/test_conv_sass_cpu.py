"""CPU check of the sm_90a build: the convolution GEMM keeps its epilogue in registers.

When the compiler cannot resolve an index into a per-thread array at compile time it places the array in local memory; in the
convolution GEMM's epilogue that made every BatchNorm-statistics butterfly level a round trip of local loads and stores, and the forward
convolutions ran 2-3x slower.  Spill counters do not show this (it is a stack frame, not a spill), so the SASS is checked directly.
"""
import os
import re
import shutil
import subprocess

import pytest


def _functions():
    from yolov7_d2_b200 import build, capi

    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not available")
    if build.find_nvcc() is None and not os.path.exists(capi.LIB_PATH):
        pytest.skip("no nvcc and no prebuilt libyb200.so")
    build.build()
    sass = subprocess.run(["cuobjdump", "-sass", capi.LIB_PATH], capture_output=True, text=True).stdout
    funcs = {}
    for part in re.split(r"\n\s*Function : ", sass)[1:]:
        name, _, body = part.partition("\n")
        funcs[name.strip()] = body
    return funcs


def test_gemm_kernels_use_no_local_memory():
    funcs = _functions()
    gemm = {n: b for n, b in funcs.items() if "conv_gemm_persistent_kernel" in n or "wgrad_gemm_kernel" in n}
    assert len([n for n in gemm if "conv_gemm_persistent_kernel" in n]) == 24, "expected 12 tile shapes x 2 epilogue sets"
    local = [n for n, b in gemm.items() if re.search(r"\b(LDL|STL)\b", b)]
    assert not local, "local-memory loads / stores in %s" % local[:4]
