"""CPU checks of the DETR meta-architecture's entry points and Python surface, no GPU needed:
  - yb200_detr_mask_pos / yb200_detr_infer / yb200_detr_pack_targets reject null pointers, bad sizes and bad level tables with exact return
    codes, in a subprocess with the GPUs hidden (a call that wrongly passed validation would fail at its first CUDA call with -3 instead of
    launching on fake pointers);
  - `Detr` is bound in the meta-architecture registry; the errors that need no device raise Yb200Error."""
import ctypes
import os
import types

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_P = 0x10000  # a fake, aligned device pointer


class _Levels(list):  # a HOST array of yb200_detr_level: (mask, pos, h, w) per level
    pass


def _rows():
    I, U = -1, -2
    rows = []

    def row(fn, args, code, null=False):
        rows.append((fn, args, code, null))

    good = [(_P, _P, 200, 334), (_P, _P, 25, 42)]

    def mp(lv=good, n=None, B=16, valid=_P, dt=_P, npf=128):
        return [None if lv is None else _Levels(lv), len(lv or []) if n is None else n, B, valid, dt, npf, None]

    row("detr_mask_pos", mp(lv=None, n=2), I, null=True)
    row("detr_mask_pos", mp(valid=None), I, null=True)
    row("detr_mask_pos", mp(dt=None), I, null=True)
    row("detr_mask_pos", mp(lv=[(None, _P, 25, 42)]), I, null=True)
    row("detr_mask_pos", mp(lv=[(_P, None, 25, 42)]), I, null=True)
    row("detr_mask_pos", mp(n=0), U)
    row("detr_mask_pos", mp(lv=[good[1]] * 9), U)
    row("detr_mask_pos", mp(B=0), I)
    row("detr_mask_pos", mp(npf=0), I)
    row("detr_mask_pos", mp(npf=127), I)
    row("detr_mask_pos", mp(lv=[(_P, _P, 0, 42)]), I)
    row("detr_mask_pos", mp(lv=[(_P, _P, 25, -1)]), I)
    row("detr_mask_pos", mp(dt=None, B=0), I, null=True)  # the null pointer is reported before the sizes

    def inf(lg=_P, bx=_P, B=16, Q=100, K1=81, sz=_P, outs=(_P,) * 11):
        return [lg, bx, B, Q, K1, sz, 0.7] + list(outs) + [None]

    row("detr_infer", inf(lg=None), I, null=True)
    row("detr_infer", inf(bx=None), I, null=True)
    row("detr_infer", inf(sz=None), I, null=True)
    for i in range(11):
        outs = [_P] * 11
        outs[i] = None
        row("detr_infer", inf(outs=outs), I, null=True)
    row("detr_infer", inf(B=0), I)
    row("detr_infer", inf(Q=0), I)
    row("detr_infer", inf(K1=1), I)
    row("detr_infer", inf(B=65536, Q=32768), U)
    row("detr_infer", inf(B=0, lg=None), I, null=True)

    def pk(bx=_P, tb=_P, B=16, G=40, out=_P):
        return [bx, tb, B, G, out, None]

    row("detr_pack_targets", pk(bx=None), I, null=True)
    row("detr_pack_targets", pk(tb=None), I, null=True)
    row("detr_pack_targets", pk(out=None), I, null=True)
    row("detr_pack_targets", pk(B=0), I)
    row("detr_pack_targets", pk(G=-1), I)
    return rows


def _run_rows():
    from yolov7_d2_b200 import capi
    from yolov7_d2_b200.detr_model import DetrLevel

    L = capi.lib()

    def arg(a):
        if isinstance(a, _Levels):
            arr = (DetrLevel * max(1, len(a)))()
            for i, t in enumerate(a):
                arr[i] = DetrLevel(*t)
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


def test_level_descriptor_matches_the_header():
    from yolov7_d2_b200 import detr_model as dm

    assert ctypes.sizeof(dm.DetrLevel) == 24
    hdr = open(os.path.join(ROOT, "include", "yb200.h")).read()
    assert f"#define YB200_DETR_MAX_LEVELS {dm.MAX_LEVELS}" in hdr


def test_registered_as_the_meta_architecture():
    from yolov7_d2_b200 import modeling
    from yolov7_d2_b200.detr_model import Detr

    assert modeling.META_ARCH_REGISTRY.get("Detr") is Detr


def _cfg(**kw):
    from oracle.gen_golden_detr_model import cfg_of

    cfg = cfg_of(device=kw.pop("device", "cuda"))
    for k, v in kw.items():
        if k == "MASK_ON":
            cfg.MODEL.MASK_ON = v
        else:
            setattr(cfg.MODEL.DETR, k, v)
    return cfg


def test_errors_that_need_no_device():
    from yolov7_d2_b200 import capi
    from yolov7_d2_b200.detr_model import Detr, PositionEmbeddingSine

    with pytest.raises(capi.Yb200Error, match="no CPU path"):
        Detr(_cfg(device="cpu"))
    with pytest.raises(capi.Yb200Error, match="MASK_ON"):
        Detr(_cfg(MASK_ON=True))
    with pytest.raises(capi.Yb200Error, match="PRE_NORM"):
        Detr(_cfg(PRE_NORM=True))
    with pytest.raises(capi.Yb200Error, match="normalize=True"):
        PositionEmbeddingSine(64, normalize=False)
    m = Detr.__new__(Detr)
    torch.nn.Module.__init__(m)
    m.onnx_export = True
    with pytest.raises(capi.Yb200Error, match="ONNX"):
        m([{"image": torch.zeros(3, 32, 32, dtype=torch.uint8)}])
    m.onnx_export = False
    m.L, m.pixel_mean, m.pixel_std = types.SimpleNamespace(), torch.zeros(3, 1, 1), torch.ones(3, 1, 1)  # no library call may happen
    with pytest.raises(capi.Yb200Error, match="empty batch"):
        m([])
    with pytest.raises(capi.Yb200Error, match=r"image 1 is \(1, 32, 32\)"):
        m([{"image": torch.zeros(3, 32, 32, dtype=torch.uint8)}, {"image": torch.zeros(1, 32, 32, dtype=torch.uint8)}])
    with pytest.raises(capi.Yb200Error, match="float64"):
        m([{"image": torch.zeros(3, 32, 32, dtype=torch.float64)}])


if __name__ == "__main__":
    import json
    import sys

    sys.path.insert(0, ROOT)
    print(json.dumps(_run_rows()))
