"""CPU checks of the SparseInst meta-architecture's entry points and Python surface, no GPU needed:
  - yb200_normalize_pad / yb200_sparseinst_infer_scores / yb200_sparseinst_paste_masks reject null pointers, bad sizes and bad image tables
    with exact return codes, in a subprocess with the GPUs hidden (a call that wrongly passed validation would fail at its first CUDA call with
    -3 instead of launching on fake pointers);
  - `SparseInst` is bound in the meta-architecture registry; the errors that need no device raise Yb200Error."""
import ctypes
import os
import types

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_P = 0x10000  # a fake, aligned device pointer


class _Images(list):  # a HOST array of yb200_paste_image: (h, w, out_h, out_w, first, count, out_off) per image
    pass


def _rows():
    I, U = -1, -2
    rows = []

    def row(fn, args, code, null=False):
        rows.append((fn, args, code, null))

    npad = lambda im=_P, tb=_P, n=2, mean=_P, std=_P, hp=64, wp=96, out=_P: [im, 0, tb, n, mean, std, hp, wp, out, None]
    row("normalize_pad", npad(im=None), I, null=True)
    row("normalize_pad", npad(tb=None), I, null=True)
    row("normalize_pad", npad(std=None), I, null=True)
    row("normalize_pad", npad(out=None), I, null=True)
    row("normalize_pad", npad(n=0), I)
    row("normalize_pad", npad(hp=0), I)
    row("normalize_pad", npad(wp=-32), I)
    row("normalize_pad", npad(out=None, n=0), I, null=True)  # the null pointer is reported before the sizes

    def sc(lg=_P, ob=_P, mk=_P, B=2, N=100, K=80, HW=160 * 216, outs=(_P,) * 9):
        return [lg, ob, mk, B, N, K, HW, 0.01, 0.45] + list(outs) + [None]

    row("sparseinst_infer_scores", sc(lg=None), I, null=True)
    row("sparseinst_infer_scores", sc(mk=None), I, null=True)
    for i in range(9):
        outs = [_P] * 9
        outs[i] = None
        row("sparseinst_infer_scores", sc(outs=outs), I, null=True)
    row("sparseinst_infer_scores", sc(B=0), I)
    row("sparseinst_infer_scores", sc(N=0), I)
    row("sparseinst_infer_scores", sc(K=-1), I)
    row("sparseinst_infer_scores", sc(HW=0), I)
    row("sparseinst_infer_scores", sc(B=65536, N=32768), U)
    row("sparseinst_infer_scores", sc(B=0, lg=None), I, null=True)

    good = [(64, 96, 48, 72, 0, 3, 0), (50, 70, 100, 140, 3, 2, 3 * 48 * 72)]

    def pm(mk=_P, N=100, hm=16, wm=24, kq=_P, ims=good, B=None, hp=64, wp=96, out=_P):
        return [mk, N, hm, wm, kq, None if ims is None else _Images(ims), len(ims or []) if B is None else B, hp, wp, 0.45, out, None]

    row("sparseinst_paste_masks", pm(mk=None), I, null=True)
    row("sparseinst_paste_masks", pm(kq=None), I, null=True)
    row("sparseinst_paste_masks", pm(ims=None, B=2), I, null=True)
    row("sparseinst_paste_masks", pm(out=None), I, null=True)
    row("sparseinst_paste_masks", pm(N=0), I)
    row("sparseinst_paste_masks", pm(hm=0), I)
    row("sparseinst_paste_masks", pm(hp=0), I)
    row("sparseinst_paste_masks", pm(B=0), U)
    row("sparseinst_paste_masks", pm(ims=[good[0]] * 65), U)
    row("sparseinst_paste_masks", pm(ims=[(65, 96, 48, 72, 0, 3, 0)]), I)  # image taller than the padded batch
    row("sparseinst_paste_masks", pm(ims=[(64, 97, 48, 72, 0, 3, 0)]), I)
    row("sparseinst_paste_masks", pm(ims=[(64, 96, 0, 72, 0, 3, 0)]), I)
    row("sparseinst_paste_masks", pm(ims=[(0, 96, 48, 72, 0, 3, 0)]), I)
    row("sparseinst_paste_masks", pm(ims=[good[0], (50, 70, 100, 140, 4, 2, 0)]), I)  # not compact: first != the counts before it
    row("sparseinst_paste_masks", pm(ims=[(64, 96, 48, 72, 1, 3, 0)]), I)
    row("sparseinst_paste_masks", pm(ims=[(64, 96, 48, 72, 0, 101, 0)]), I)  # more masks than queries
    row("sparseinst_paste_masks", pm(ims=[(64, 96, 48, 72, 0, -1, 0)]), I)
    row("sparseinst_paste_masks", pm(ims=[(64, 96, 48, 72, 0, 3, -1)]), I)
    row("sparseinst_paste_masks", pm(N=40000, ims=[(64, 96, 8, 8, 0, 40000, 0), (64, 96, 8, 8, 40000, 40000, 1 << 22)]), U)  # >= 65536 masks
    return rows


def _run_rows():
    from yolov7_d2_b200 import capi
    from yolov7_d2_b200.sparseinst_model import PasteImage

    L = capi.lib()

    def arg(a):
        if isinstance(a, _Images):
            arr = (PasteImage * max(1, len(a)))()
            for i, t in enumerate(a):
                arr[i] = PasteImage(*t)
            return arr
        if isinstance(a, float):
            return ctypes.c_float(a)
        return ctypes.c_void_p(a) if a == _P else a

    out = []
    for fn, args, _, _ in _rows():
        rc = getattr(L, "yb200_" + fn)(*[arg(a) for a in args])
        out.append((rc, L.yb200_last_error().decode()))
    return out


def test_entry_points_reject_bad_arguments():
    import json
    import subprocess
    import sys

    from yolov7_d2_b200 import build, capi

    if build.find_nvcc() is None and not os.path.exists(capi.LIB_PATH):
        pytest.skip("no nvcc and no prebuilt libyb200.so")
    build.build()
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="", PYTHONPATH=os.pathsep.join([ROOT] + [p for p in [os.environ.get("PYTHONPATH")] if p]))
    r = subprocess.run([sys.executable, os.path.abspath(__file__)], capture_output=True, text=True, env=env, cwd=ROOT, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    got = json.loads(r.stdout.strip().splitlines()[-1])
    rows = _rows()
    assert len(got) == len(rows)
    bad = []
    for i, ((fn, _, code, null), (rc, msg)) in enumerate(zip(rows, got)):
        if rc != code or fn not in msg or (null and "null" not in msg):
            bad.append(f"row {i} yb200_{fn}: returned {rc} ({msg!r}), expected {code}" + (" with 'null'" if null else ""))
    assert not bad, "\n".join(bad)


def test_paste_descriptor_matches_the_header():
    from yolov7_d2_b200 import sparseinst_model as sm

    assert ctypes.sizeof(sm.PasteImage) == 32
    hdr = open(os.path.join(ROOT, "include", "yb200.h")).read()
    assert f"#define YB200_PASTE_MAX_IMAGES {sm.PASTE_MAX_IMAGES}" in hdr


def _cfg(device="cuda", decoder="GroupIAMDecoder"):
    ns = types.SimpleNamespace
    return ns(MODEL=ns(DEVICE=device, SPARSE_INST=ns(DECODER=ns(NAME=decoder))))


def test_registered_as_the_meta_architecture():
    from yolov7_d2_b200 import modeling
    from yolov7_d2_b200.sparseinst_model import SparseInst

    assert modeling.META_ARCH_REGISTRY.get("SparseInst") is SparseInst


def test_errors_that_need_no_device():
    from yolov7_d2_b200 import capi, modeling
    from yolov7_d2_b200.sparseinst_model import SparseInst

    with pytest.raises(capi.Yb200Error, match="no CPU path"):
        SparseInst(_cfg(device="cpu"))
    with pytest.raises(capi.Yb200Error, match="decoder 'IAMDecoderX'"):
        SparseInst(_cfg(decoder="IAMDecoderX"))
    m = SparseInst.__new__(SparseInst)
    torch.nn.Module.__init__(m)
    m.device, m.mask_format = torch.device("cpu"), "polygon"
    inst = modeling.Instances((32, 48), gt_classes=torch.zeros(1, dtype=torch.int64), gt_masks=types.SimpleNamespace(polygons=[[[0.0, 0, 5, 0, 5, 5]]]))
    if not modeling.HAVE_D2:
        with pytest.raises(capi.Yb200Error, match="polygon"):
            m.prepare_targets([inst])
    m.mask_format = "bitmask"
    empty = m.prepare_targets([modeling.Instances((32, 48), gt_classes=torch.zeros(0, dtype=torch.int64))])[0]
    assert empty["masks"].tensor.shape == (0, 32, 48) and empty["masks"].tensor.dtype == torch.bool
    orig = torch.onnx.is_in_onnx_export
    torch.onnx.is_in_onnx_export = lambda: True
    try:
        with pytest.raises(capi.Yb200Error, match="ONNX"):
            m([{"image": torch.zeros(3, 32, 32, dtype=torch.uint8)}])
    finally:
        torch.onnx.is_in_onnx_export = orig


if __name__ == "__main__":
    import json
    import sys

    sys.path.insert(0, ROOT)
    print(json.dumps(_run_rows()))
