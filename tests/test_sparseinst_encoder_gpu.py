"""The SparseInst InstanceContextEncoder on the kernels (yolov7_d2_b200.sparseinst_encoder): kernel by kernel, call by call, and whole.

A. Each new kernel against fp64 on exactly the operands it reads, with the bound of tests/test_convnext_plan_gpu.py (|got - ref| <= r_store |ref|
   + c(K) 2^-24 mag): the floor-mode average pool, the PPM input gradient (uncovered rows and columns included), the bilinear resize and its
   adjoint (with and without the ReLU mask) into and out of channel slices, the nearest x2 add and its masked adjoint.  Channels outside an
   output view must keep their bits and nothing may be written past the end of the output buffer.
B. Every C-ABI call of an encoder forward and backward, recorded through the stand-in library handle of tests/test_sparseinst_kernels_gpu.py,
   replayed on fresh operands against fp64.
C. The whole encoder: the unmodified reference (tests/golden/sparseinst_encoder.npz) and, at the shipped widths, the fp64 oracle, the output and
   each gradient's relative L2 error <= 2.5 x that of the bf16-storage-emulating oracle + 2 %; outputs with and without autograd give the same
   bits; two backward passes give the same bits; no input data gradient runs for inputs that do not require grad; frozen parameters get none;
   the Yb200Error cases raise before any kernel runs.
D. Encoder -> GroupIAMDecoder -> SparseInstCriterion -> sum(c * loss).backward() against the oracle encoder + decoder + the fp64 criterion on
   the engine's match.
"""
import ctypes
import math
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from test_convnext_plan_gpu import GUARD, R_BF16, WORST, _act, _g, _geo, _given, _in_view, _lib, _outside_same, _sl, bound, check
from test_sparseinst_bwd_gpu import REPLAY as GEMM_REPLAY
from test_sparseinst_bwd_gpu import _judge
from test_sparseinst_kernels_gpu import QUERIES, _Recorder, _v

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------------------------------------------
# A. the new kernels against fp64
# ------------------------------------------------------------------------------------------------------------------------------------
def _out_guarded(geo, g):
    """output buffer of the view's geometry inside a flat buffer followed by GUARD elements of 7: random outside the view, NaN inside;
    returns (flat buffer, tensor, copy)"""
    n, h, w, c, pitch, off = geo
    numel = n * h * w * pitch
    buf = torch.full((numel + GUARD,), 7.0, dtype=torch.bfloat16, device="cuda")
    t = buf[:numel].view(n, h, w, pitch)
    t.copy_(torch.randn(n, h, w, pitch, generator=g, device="cuda"))
    t[..., off:off + c] = float("nan")
    return buf, t, t.clone()


def _done(buf, t, t0, geo, what):
    _outside_same(t, t0, geo, what)
    assert bool((buf[t.numel():] == 7.0).all()), f"{what}: wrote past the end of its output"


def _nchw(t):
    return t.double().permute(0, 3, 1, 2)


def _nhwc(t):
    return t.permute(0, 2, 3, 1)


def _geo_of(n, h, w, c, pitch=None, off=0):
    return (n, h, w, c, pitch or c, off)


def run_pool(gx, kh, kw, go, seed=90):
    """yb200_avg_pool2d: bf16(window sum / (kh kw)), floor mode"""
    capi, L = _lib()
    g = _g(seed)
    x = _in_view(gx, g)
    buf, o, o0 = _out_guarded(go, g)
    xa, oa = _act(capi, x, gx), _act(capi, o, go)
    capi.check(L.yb200_avg_pool2d(ctypes.byref(xa), kh, kw, ctypes.byref(oa), capi.stream_ptr()), "avg_pool2d")
    xv = _nchw(_sl(x, gx))
    ref = _nhwc(F.avg_pool2d(xv, (kh, kw)))
    mag = _nhwc(F.avg_pool2d(xv.abs(), (kh, kw)))
    check("avg pool (bf16)", _sl(o, go), ref, bound(ref, mag, kh * kw, R_BF16), f"pooled {gx} / {kh}x{kw}")
    _done(buf, o, o0, go, "pooled")


def run_ppm_grad(gcat, stages, gdx, seed=91):
    """yb200_ppm_input_grad: bf16(dcat + sum_s avgpool adjoint(dpooled_s)); stages = [(geo, kh, kw)]"""
    capi, L = _lib()
    g = _g(seed)
    dcat = _in_view(gcat, g)
    dps = [_in_view(geo, g) for geo, _, _ in stages]
    buf, dx, dx0 = _out_guarded(gdx, g)
    ca, da = _act(capi, dcat, gcat), _act(capi, dx, gdx)
    views = (capi.Act * len(stages))(*[_act(capi, t, geo) for t, (geo, _, _) in zip(dps, stages)])
    khw = (ctypes.c_int32 * (2 * len(stages)))(*[v for _, kh, kw in stages for v in (kh, kw)])
    capi.check(L.yb200_ppm_input_grad(ctypes.byref(ca), views, khw, len(stages), ctypes.byref(da), capi.stream_ptr()), "ppm_input_grad")
    n, h, w, c = gdx[:4]
    ref = _sl(dcat, gcat).double()
    mag = ref.abs()
    for t, (geo, kh, kw) in zip(dps, stages):
        adj = []
        for dp in (_nchw(_sl(t, geo)), _nchw(_sl(t, geo)).abs()):
            x = torch.zeros(n, c, h, w, dtype=torch.float64, device="cuda", requires_grad=True)
            F.avg_pool2d(x, (kh, kw)).backward(dp)
            adj.append(_nhwc(x.grad))
        ref, mag = ref + adj[0], mag + adj[1]
    check("PPM input gradient (bf16)", _sl(dx, gdx), ref, bound(ref, mag, len(stages) + 1, R_BF16), "d lat0")
    _done(buf, dx, dx0, gdx, "d lat0")
    # rows / columns beyond the last full window of every stage receive d cat only
    cover_h = max(kh * geo[1] for geo, kh, _ in stages)
    cover_w = max(kw * geo[2] for geo, _, kw in stages)
    for sl in ((slice(None), slice(cover_h, None)), (slice(None), slice(None), slice(cover_w, None))):
        assert torch.equal(_sl(dx, gdx)[sl], _sl(dcat, gcat)[sl]), "uncovered pixels must receive exactly d cat"


def _resize_terms(hi, wi, ho, wo):
    return (math.ceil(ho / hi) + 2) * (math.ceil(wo / wi) + 2)


def run_resize(gx, go, seed=92):
    """yb200_resize_bilinear: F.interpolate(size=, bilinear, align_corners=False)"""
    capi, L = _lib()
    g = _g(seed)
    x = _in_view(gx, g)
    buf, o, o0 = _out_guarded(go, g)
    xa, oa = _act(capi, x, gx), _act(capi, o, go)
    capi.check(L.yb200_resize_bilinear(ctypes.byref(xa), ctypes.byref(oa), capi.stream_ptr()), "resize_bilinear")
    xv = _nchw(_sl(x, gx))
    size = go[1:3]
    ref = _nhwc(F.interpolate(xv, size=size, mode="bilinear", align_corners=False))
    mag = _nhwc(F.interpolate(xv.abs(), size=size, mode="bilinear", align_corners=False))
    check("bilinear resize (bf16)", _sl(o, go), ref, bound(ref, mag, 4, R_BF16), f"resize {gx[1:3]} -> {size}")
    _done(buf, o, o0, go, "resized")


def run_resize_bwd(gdo, gh, gdx, seed=93):
    """yb200_resize_bilinear_bwd: the adjoint of the resize (masked by h > 0 when h is given), gather form"""
    capi, L = _lib()
    g = _g(seed)
    dout = _in_view(gdo, g)
    h = _in_view(gh, g) if gh else None
    if h is not None:
        hv = _sl(h, gh)
        hv[0, 0, 0, :8] = torch.tensor([0.0, -0.0, 1e-30, -1e-30, 0.0, 1.0, -1.0, 0.0], device="cuda").to(torch.bfloat16)
    buf, dx, dx0 = _out_guarded(gdx, g)
    da, xa = _act(capi, dout, gdo), _act(capi, dx, gdx)
    ha = _act(capi, h, gh) if gh else None
    capi.check(L.yb200_resize_bilinear_bwd(ctypes.byref(da), ctypes.byref(ha) if gh else None, ctypes.byref(xa), capi.stream_ptr()),
               "resize_bilinear_bwd")
    n, hi, wi, c = gdx[:4]
    dv = _nchw(_sl(dout, gdo))
    res = []
    for d in (dv, dv.abs()):
        x = torch.zeros(n, c, hi, wi, dtype=torch.float64, device="cuda", requires_grad=True)
        F.interpolate(x, size=gdo[1:3], mode="bilinear", align_corners=False).backward(d)
        res.append(_nhwc(x.grad))
    ref, mag = res
    if h is not None:
        keep = (_sl(h, gh).double() > 0).double()
        ref, mag = ref * keep, mag * keep
    check("bilinear resize adjoint (bf16)", _sl(dx, gdx), ref, bound(ref, mag, _resize_terms(hi, wi, gdo[1], gdo[2]), R_BF16),
          f"resize adjoint {gdo[1:3]} -> {gdx[1:3]}")
    _done(buf, dx, dx0, gdx, "resize adjoint")


def run_nearest_add(glat, gc, go, inplace=False, seed=94):
    """yb200_upsample_nearest2x_add: bf16(lat + nearest x2(coarse)), out = lat when inplace"""
    capi, L = _lib()
    g = _g(seed)
    lat = _in_view(glat, g)
    coarse = _in_view(gc, g)
    ref = _sl(lat, glat).double() + _sl(coarse, gc).double().repeat_interleave(2, 1).repeat_interleave(2, 2)
    mag = _sl(lat, glat).double().abs() + _sl(coarse, gc).double().abs().repeat_interleave(2, 1).repeat_interleave(2, 2)
    la, ca = _act(capi, lat, glat), _act(capi, coarse, gc)
    if inplace:
        assert glat == go
        lat0 = lat.clone()
        capi.check(L.yb200_upsample_nearest2x_add(ctypes.byref(la), ctypes.byref(ca), ctypes.byref(la), capi.stream_ptr()), "nearest2x_add")
        check("nearest x2 add (bf16)", _sl(lat, go), ref, bound(ref, mag, 2, R_BF16), "prev (in place)")
        _outside_same(lat, lat0, go, "prev")
        return
    buf, o, o0 = _out_guarded(go, g)
    oa = _act(capi, o, go)
    capi.check(L.yb200_upsample_nearest2x_add(ctypes.byref(la), ctypes.byref(ca), ctypes.byref(oa), capi.stream_ptr()), "nearest2x_add")
    check("nearest x2 add (bf16)", _sl(o, go), ref, bound(ref, mag, 2, R_BF16), "prev")
    _done(buf, o, o0, go, "prev")


def run_nearest_bwd(gdy, gh, gdx, seed=95):
    """yb200_upsample_nearest2x_bwd: bf16(2x2 sums of dy), masked by h > 0 when h is given"""
    capi, L = _lib()
    g = _g(seed)
    dy = _in_view(gdy, g)
    h = _in_view(gh, g) if gh else None
    buf, dx, dx0 = _out_guarded(gdx, g)
    ya, xa = _act(capi, dy, gdy), _act(capi, dx, gdx)
    ha = _act(capi, h, gh) if gh else None
    capi.check(L.yb200_upsample_nearest2x_bwd(ctypes.byref(ya), ctypes.byref(ha) if gh else None, ctypes.byref(xa), capi.stream_ptr()), "nearest2x_bwd")
    d = _nchw(_sl(dy, gdy))
    ref, mag = _nhwc(F.avg_pool2d(d, 2) * 4), _nhwc(F.avg_pool2d(d.abs(), 2) * 4)
    if h is not None:
        keep = (_sl(h, gh).double() > 0).double()
        ref, mag = ref * keep, mag * keep
        assert bool((_sl(dx, gdx)[keep == 0] == 0).all()), "masked elements must be exactly zero"
    check("nearest x2 adjoint (bf16)", _sl(dx, gdx), ref, bound(ref, mag, 4, R_BF16), "d coarse")
    _done(buf, dx, dx0, gdx, "d coarse")


# (map, PPM size) pairs of the encoder's maps: the window is (ceil(H/s), ceil(W/s)), the pooled map (H // kh, W // kw)
POOL_MAPS = [(20, 20), (20, 27), (5, 7), (4, 6)]
POOL_CASES = [(h, w, s) for h, w in POOL_MAPS for s in (1, 2, 3, 6)]


@pytest.mark.parametrize("hws", POOL_CASES, ids=lambda t: f"{t[0]}x{t[1]}-s{t[2]}")
def test_pool(cuda, hws):
    h, w, s = hws
    kh, kw = math.ceil(h / s), math.ceil(w / s)
    run_pool(_geo_of(2, h, w, 256, 512, 256), kh, kw, _geo_of(2, h // kh, w // kw, 256))


@pytest.mark.parametrize("hw", POOL_MAPS, ids=lambda t: f"{t[0]}x{t[1]}")
def test_ppm_input_grad(cuda, hw):
    """all four stages of a map (20x27: the 2x1 and 2x3 priors leave rows 20.. / columns 26.. uncovered)"""
    h, w = hw
    stages = []
    for s in (1, 2, 3, 6):
        kh, kw = math.ceil(h / s), math.ceil(w / s)
        stages.append((_geo_of(2, h // kh, w // kw, 64), kh, kw))
    run_ppm_grad(_geo_of(2, h, w, 64, 128, 64), stages, _geo_of(2, h, w, 64))


def test_ppm_input_grad_uncovered(cuda):
    """one stage whose windows leave the last row and the last two columns uncovered: those pixels get d cat, bit for bit"""
    run_ppm_grad(_geo_of(2, 7, 8, 32, 64, 32), [(_geo_of(2, 2, 2, 32), 3, 3)], _geo_of(2, 7, 8, 32))


# (input map, output map, channels): the PPM priors into 64-channel slices of cat512, the fusion's x2 / x4 into slices of cat768
RESIZE_CASES = [((2, 1, 1), (20, 20), 64, 512, 0), ((2, 2, 1), (20, 27), 64, 512, 64), ((2, 2, 3), (20, 27), 64, 512, 128),
                ((2, 5, 5), (20, 20), 64, 512, 192), ((2, 40, 40), (80, 80), 256, 768, 256), ((2, 20, 20), (80, 80), 256, 768, 512),
                ((2, 20, 27), (40, 54), 64, 192, 64), ((1, 5, 7), (20, 28), 16, 32, 16)]


@pytest.mark.parametrize("case", RESIZE_CASES, ids=lambda t: f"{t[0][1]}x{t[0][2]}-{t[1][0]}x{t[1][1]}@{t[4]}")
def test_resize(cuda, case):
    (n, hi, wi), (ho, wo), c, pitch, off = case
    run_resize(_geo_of(n, hi, wi, c), _geo_of(n, ho, wo, c, pitch, off))


@pytest.mark.parametrize("masked", [False, True], ids=["plain", "relu-mask"])
@pytest.mark.parametrize("case", RESIZE_CASES, ids=lambda t: f"{t[0][1]}x{t[0][2]}-{t[1][0]}x{t[1][1]}@{t[4]}")
def test_resize_bwd(cuda, case, masked):
    (n, hi, wi), (ho, wo), c, pitch, off = case
    gdx = _geo_of(n, hi, wi, c)
    run_resize_bwd(_geo_of(n, ho, wo, c, pitch, off), gdx if masked else None, gdx)


@pytest.mark.parametrize("case", [((2, 40, 40), 256, False), ((2, 80, 108), 256, True), ((1, 10, 14), 64, True)],
                         ids=["40x40", "80x108-inplace", "10x14-inplace"])
def test_nearest_add(cuda, case):
    (n, h, w), c, inplace = case
    g = _geo_of(n, h, w, c)
    run_nearest_add(g, _geo_of(n, h // 2, w // 2, c), g, inplace)


@pytest.mark.parametrize("masked", [False, True], ids=["plain", "relu-mask"])
@pytest.mark.parametrize("case", [((2, 80, 80), 256), ((2, 40, 54), 256), ((1, 10, 14), 64)], ids=["80x80", "40x54", "10x14"])
def test_nearest_bwd(cuda, case, masked):
    (n, h, w), c = case
    gdx = _geo_of(n, h // 2, w // 2, c)
    run_nearest_bwd(_geo_of(n, h, w, c), gdx if masked else None, gdx)


# ------------------------------------------------------------------------------------------------------------------------------------
# B. every call of an encoder forward and backward, replayed
# ------------------------------------------------------------------------------------------------------------------------------------
REPLAY = dict(GEMM_REPLAY, pool=run_pool, ppm_grad=run_ppm_grad, resize=run_resize, resize_bwd=run_resize_bwd, nearest_add=run_nearest_add,
              nearest_bwd=run_nearest_bwd)
ENTRY_POINTS = {"yb200_pack_conv_weight", "yb200_conv2d_affine_fwd", "yb200_conv2d_relu_fwd", "yb200_avg_pool2d", "yb200_resize_bilinear",
                "yb200_upsample_nearest2x_add", "yb200_conv2d_wgrad_workspace", "yb200_conv2d_wgrad", "yb200_colsum_workspace", "yb200_colsum",
                "yb200_conv2d_dgrad", "yb200_conv2d_dgrad_relu", "yb200_resize_bilinear_bwd", "yb200_upsample_nearest2x_bwd", "yb200_ppm_input_grad"}


def _case(name, a):
    """replay case of one recorded call (None for the workspace queries)"""
    if name == "yb200_pack_conv_weight":
        if _given(a[6]):
            return dict(fn="pack", cout=a[1], cin=a[2], k=a[3], cout_pad=a[4], cin_pad=a[5])
        return dict(fn="pack_dgrad", cout=a[1], cin=a[2], k=a[3], cout_pad=a[4], cin_pad=a[5])
    if name == "yb200_conv2d_affine_fwd":
        return dict(fn="affine", gx=_geo(a[0]), go=_geo(a[5]), gr=_geo(a[4]), k=a[6], s=a[7], with_scale=_given(a[2]), with_shift=_given(a[3]))
    if name == "yb200_conv2d_relu_fwd":
        return dict(fn="relu", gx=_geo(a[0]), go=_geo(a[3]), k=a[4], s=a[5])
    if name == "yb200_conv2d_wgrad":
        return dict(fn="wgrad", gx=_geo(a[0]), gdz=_geo(a[1]), k=a[2], s=a[3], cin_real=a[4], accumulate=a[6])
    if name == "yb200_colsum":
        return dict(fn="colsum", gx=_geo(a[0]), scale=_v(a[1]), accumulate=a[3])
    if name == "yb200_conv2d_dgrad":
        return dict(fn="dgrad", gdz=_geo(a[0]), gdx=_geo(a[2]), ga=_geo(a[3]), k=a[4], s=a[5])
    if name == "yb200_conv2d_dgrad_relu":
        return dict(fn="dgrad_relu", gdz=_geo(a[0]), gdx=_geo(a[3]), gh=_geo(a[2]), ga=_geo(a[4]), k=a[5])
    if name == "yb200_avg_pool2d":
        return dict(fn="pool", gx=_geo(a[0]), kh=a[1], kw=a[2], go=_geo(a[3]))
    if name == "yb200_resize_bilinear":
        return dict(fn="resize", gx=_geo(a[0]), go=_geo(a[1]))
    if name == "yb200_resize_bilinear_bwd":
        return dict(fn="resize_bwd", gdo=_geo(a[0]), gh=_geo(a[1]) if _given(a[1]) else None, gdx=_geo(a[2]))
    if name == "yb200_upsample_nearest2x_add":
        inplace = a[0]._obj.ptr == a[2]._obj.ptr
        return dict(fn="nearest_add", glat=_geo(a[0]), gc=_geo(a[1]), go=_geo(a[2]), inplace=inplace)
    if name == "yb200_upsample_nearest2x_bwd":
        return dict(fn="nearest_bwd", gdy=_geo(a[0]), gh=_geo(a[1]) if _given(a[1]) else None, gdx=_geo(a[2]))
    if name == "yb200_ppm_input_grad":
        views, khw, n = a[1], a[2], a[3]
        stages = [((views[i].n, views[i].h, views[i].w, views[i].c, views[i].c_pitch, views[i].c_off), khw[2 * i], khw[2 * i + 1]) for i in range(n)]
        return dict(fn="ppm_grad", gcat=_geo(a[0]), stages=stages, gdx=_geo(a[4]))
    if name in QUERIES:
        return None
    raise AssertionError(f"{name}: an encoder call this module does not replay")


def _cfg(num_channels=256):
    ns = types.SimpleNamespace
    return ns(MODEL=ns(SPARSE_INST=ns(ENCODER=ns(NAME="InstanceContextEncoder", NUM_CHANNELS=num_channels, IN_FEATURES=["res3", "res4", "res5"]))))


def _shape(in_channels):
    return {k: types.SimpleNamespace(channels=c) for k, c in zip(("res3", "res4", "res5"), in_channels)}


def _encoder(seed, in_channels=(512, 1024, 2048), num_channels=256):
    from yolov7_d2_b200.sparseinst_encoder import InstanceContextEncoder

    from oracle import sparseinst_encoder_oracle as seo

    enc = InstanceContextEncoder(_cfg(num_channels), _shape(in_channels))
    sd = seo.encoder_state_dict(seed, in_channels, num_channels)
    enc.load_state_dict({k: v.cuda() for k, v in sd.items()}, strict=True)
    return enc, sd


def _features(b, h5, w5, seed, in_channels=(512, 1024, 2048), device="cuda", requires_grad=(True, True, True)):
    g = torch.Generator().manual_seed(seed)
    f = {}
    for i, (k, c) in enumerate(zip(("res3", "res4", "res5"), in_channels)):
        s = 2 ** (2 - i)
        f[k] = torch.randn(b, c, h5 * s, w5 * s, generator=g).to(device).requires_grad_(requires_grad[i])
    return f


def _recorded(enc, feats, seed):
    """one forward with autograd and the backward of a seeded upstream gradient through the stand-in handle: the call log"""
    rec = _Recorder(enc.L)
    enc.L = rec
    try:
        for p in enc.parameters():
            p.grad = None
        out = enc(feats)
        out.backward(torch.randn(out.shape, generator=_g(seed), device="cuda"))
        torch.cuda.synchronize()
    finally:
        enc.L = rec._lib
    return rec.log


RECORD_MAPS = [(2, 20, 20), (2, 20, 27)]
RECORDINGS = {}


def _recordings():
    if not RECORDINGS and torch.cuda.is_available():
        enc, _ = _encoder(100)
        for i, (b, h, w) in enumerate(RECORD_MAPS):
            RECORDINGS[(b, h, w)] = _recorded(enc, _features(b, h, w, 101 + i), 103 + i)
        del enc
        torch.cuda.empty_cache()
    return RECORDINGS


def _distinct():
    seen, out = set(), []
    for m, log in _recordings().items():
        for name, a, _ in log:
            case = _case(name, a)
            if case is None:
                continue
            key = tuple(sorted((k, str(v)) for k, v in case.items()))
            if key in seen:
                continue
            seen.add(key)
            out.append((f"{name[len('yb200_'):]} " + " ".join(f"{k}={v}" for k, v in case.items() if k != "fn"), case))
    return out


def pytest_generate_tests(metafunc):
    if "enc_case" in metafunc.fixturenames:
        cases = _distinct()
        metafunc.parametrize("enc_case", [c[1] for c in cases], ids=[c[0] for c in cases])


def test_encoder_call(cuda, enc_case):
    case = dict(enc_case)
    REPLAY[case.pop("fn")](**case)


def test_recording_is_complete(cuda):
    """every entry point an encoder forward and backward calls is replayed, and every call succeeded"""
    for m, log in _recordings().items():
        names = {name for name, _, _ in log}
        assert names == ENTRY_POINTS, f"{m}: entry points called {sorted(names)}, replayed {sorted(ENTRY_POINTS)}"
        assert all(rc == 0 for name, _, rc in log if name not in QUERIES), f"{m}: a call failed"
    cases = [c for _, c in _distinct()]
    assert {(c["gx"][1], c["gx"][2], c["go"][1], c["go"][2]) for c in cases if c["fn"] == "pool"} >= {(20, 27, 2, 1), (20, 27, 2, 3), (20, 20, 2, 2)}
    assert any(c["fn"] == "ppm_grad" and len(c["stages"]) == 4 for c in cases)


# ------------------------------------------------------------------------------------------------------------------------------------
# C. the whole encoder
# ------------------------------------------------------------------------------------------------------------------------------------
def _engine(enc, feats, up):
    for p in enc.parameters():
        p.grad = None
    out = enc(feats)
    out.backward(up.cuda())
    g = {k: p.grad for k, p in enc.named_parameters()}
    g.update({f"d_{k}": v.grad for k, v in feats.items()})
    g["out"] = out.detach()
    return g


def _oracle(feats, sd, up, storage, device):
    from oracle import sparseinst_encoder_oracle as seo

    f = {k: v.detach().double().to(device).requires_grad_(True) for k, v in feats.items()}
    sdd = {k: v.detach().double().to(device).requires_grad_(True) for k, v in sd.items()}
    out = (seo.encoder_forward_storage if storage else seo.encoder_forward)(f, sdd)
    out.backward(up.double().to(device))
    g = {k: v.grad for k, v in sdd.items()}
    g.update({f"d_{k}": v.grad for k, v in f.items()})
    g["out"] = out.detach()
    return g


def _fixture_cases():
    from oracle.gen_golden_sparseinst_encoder import CASES

    return CASES


@pytest.mark.parametrize("case", _fixture_cases(), ids=[c[0] for c in _fixture_cases()])
def test_encoder_matches_the_reference(cuda, case):
    from test_sparseinst_encoder_oracle_golden import gold

    from oracle.gen_golden_sparseinst_encoder import IN_CHANNELS, NUM_CHANNELS, features, state_dict, upstream

    enc, _ = _encoder(0, IN_CHANNELS, NUM_CHANNELS)
    sd = state_dict(case)
    enc.load_state_dict({k: v.cuda() for k, v in sd.items()}, strict=True)
    feats = {k: v.float().cuda().requires_grad_(True) for k, v in features(case).items()}
    up = upstream(case).float()
    got = _engine(enc, feats, up)
    ref_out, ref = gold(case)
    ref["out"] = ref_out
    emu = _oracle(feats, sd, up, True, "cpu")
    assert sorted(got) == sorted(ref)
    _judge(got, ref, emu, case[0])


@pytest.mark.parametrize("hw", [(20, 20), (20, 27)], ids=["640x640", "640x864"])
def test_shipped_widths_against_fp64(cuda, hw):
    """2 x (512, 1024, 2048) at 80/40/20 (and 80x108/40x54/20x27): the output and every gradient against the fp64 oracle on the device"""
    enc, sd = _encoder(110)
    feats = _features(2, *hw, 111)
    up = torch.randn(2, 256, 4 * hw[0], 4 * hw[1], generator=torch.Generator().manual_seed(112))
    got = _engine(enc, feats, up)
    ref = _oracle(feats, sd, up, False, "cuda")
    emu = _oracle(feats, sd, up, True, "cuda")
    assert all(got[k] is not None and torch.isfinite(got[k]).all() for k in ref), "missing or non-finite gradients"
    _judge(got, ref, emu, f"encoder {hw}")


def test_grad_mode_forward_and_backward_are_bit_exact(cuda):
    """grad-mode output = no-grad output, bit for bit; two identical backward passes give the same bits"""
    enc, _ = _encoder(113)
    feats = _features(2, 20, 27, 114)
    with torch.no_grad():
        ref = enc(feats)
    up = torch.randn(ref.shape, generator=_g(115), device="cuda")
    runs = [_engine(enc, feats, up) for _ in range(2)]
    assert torch.equal(runs[0]["out"], ref), "the grad-mode forward differs from the no-grad forward"
    for k, v in runs[0].items():
        assert torch.equal(v, runs[1][k]), f"{k}: two backward passes differ"


@pytest.mark.parametrize("req", [(True, False, False), (False, False, False)], ids=["res3-only", "none"])
def test_no_input_gradient_without_requires_grad(cuda, req):
    """the res5 / res4 data gradients (256 -> 2048 / 1024) do not run for inputs that do not require grad"""
    enc, _ = _encoder(116)
    feats = _features(2, 20, 20, 117, requires_grad=req)
    log = _recorded(enc, feats, 118)
    launched = {_geo(a[2])[1:4:2] for name, a, _ in log if name == "yb200_conv2d_dgrad"}  # (rows, channels) of every dx
    for want, hc in zip(req, ((80, 512), (40, 1024), (20, 2048))):
        assert (hc in launched) == want, f"data gradient to {hc[1]} channels at {hc[0]} rows: launched {hc in launched}, wanted {want}"
    for want, (k, v) in zip(req, feats.items()):
        assert (v.grad is not None) == want, k
    assert all(p.grad is not None for p in enc.parameters())


def test_frozen_parameters_get_no_gradient(cuda):
    enc, _ = _encoder(119)
    frozen = {"fpn_laterals.0.weight", "ppm.stages.2.1.bias", "ppm.bottleneck.weight", "fusion.bias", "fpn_outputs.1.weight"}
    for k, p in enc.named_parameters():
        p.requires_grad_(k not in frozen)
    feats = _features(2, 20, 20, 120)
    _recorded(enc, feats, 121)
    for k, p in enc.named_parameters():
        assert (p.grad is None) == (k in frozen), k
    assert all(v.grad is not None and torch.isfinite(v.grad).all() for v in feats.values())


def test_errors_raise_before_any_kernel(cuda):
    from yolov7_d2_b200 import capi
    from yolov7_d2_b200.sparseinst_encoder import InstanceContextEncoder

    with pytest.raises(capi.Yb200Error, match="multiple of 64"):
        InstanceContextEncoder(_cfg(96), _shape((512, 1024, 2048)))
    with pytest.raises(capi.Yb200Error, match="multiples of 16"):
        InstanceContextEncoder(_cfg(), _shape((520, 1024, 2048)))
    enc, _ = _encoder(122)
    rec = _Recorder(enc.L)
    enc.L = rec
    try:
        good = _features(1, 4, 6, 123, requires_grad=(False, False, False))
        bad = [({k: v.cpu() for k, v in good.items()}, "CUDA tensor"),
               ({k: v for k, v in good.items() if k != "res4"}, "missing"),
               (dict(good, res4=good["res4"][:, :, :7]), "exactly twice"),
               (dict(good, res3=good["res3"][:, :500]), "expected"),
               ]
        for feats, msg in bad:
            with pytest.raises(capi.Yb200Error, match=msg):
                enc(feats)
    finally:
        enc.L = rec._lib
    assert not rec.log, f"kernels ran before the error: {[n for n, _, _ in rec.log]}"


# ------------------------------------------------------------------------------------------------------------------------------------
# D. encoder + decoder + criterion
# ------------------------------------------------------------------------------------------------------------------------------------
def test_encoder_decoder_and_criterion_train_end_to_end(cuda):
    """one training step's gradients: encoder -> GroupIAMDecoder -> SparseInstCriterion -> sum(c * loss).backward(), against the oracle
    encoder + decoder and the fp64 criterion on the engine's match, under the same yardstick; the decoder's d features is the encoder's upstream"""
    from test_sparseinst_criterion_gpu import _cfg as crit_cfg
    from test_sparseinst_criterion_gpu import _ellipses
    from test_sparseinst_kernels_gpu import _decoder
    from yolov7_d2_b200.sparseinst_criterion import _Targets, build_sparse_inst_criterion

    from oracle import sparseinst_criterion_oracle as sco
    from oracle import sparseinst_encoder_oracle as seo
    from oracle import sparseinst_oracle as sio
    from oracle import sparseinst_storage_oracle as sso

    enc, esd = _encoder(130)
    dec, dsd = _decoder("Group", seed=131)
    g = torch.Generator().manual_seed(132)
    B, IN = 2, 320
    feats = _features(B, IN // 32, IN // 32, 133)
    sizes = [3, 5]
    mask_list = [_ellipses(g, n, IN - 16 * b, IN) for b, n in enumerate(sizes)]
    labels = torch.randint(0, 80, (sum(sizes),), generator=g)
    off = np.concatenate([[0], np.cumsum(sizes)])
    targets = [{"labels": labels[off[b]:off[b + 1]].cuda(), "masks": sco.BitMasks(m.cuda())} for b, m in enumerate(mask_list)]
    coef = {"loss_ce": 0.7, "loss_objectness": 1.3, "loss_dice": 0.4, "loss_mask": 1.9}
    weights = (2.0, 5.0, 2.0, 1.0)
    crit = build_sparse_inst_criterion(crit_cfg(80, 0.8, 0.2, weights))
    out = dec(enc(feats))
    losses = crit(out, targets, (IN, IN))
    sum(coef[k] * v for k, v in losses.items()).backward()
    got = {f"enc.{k}": p.grad for k, p in enc.named_parameters()}
    got.update({f"dec.{k}": p.grad for k, p in dec.named_parameters()})
    got.update({f"d_{k}": v.grad for k, v in feats.items()})
    assert all(v is not None and torch.isfinite(v).all() and v.abs().sum() > 0 for v in got.values()), "a parameter or input got no gradient"
    tg_out = {k: out[k].detach() for k in ("pred_logits", "pred_masks", "pred_scores")}
    tg = _Targets(targets, (IN, IN), tg_out["pred_masks"].shape, cuda, "test")
    indices, _ = crit.matcher.match(tg_out["pred_logits"].float().contiguous(), tg_out["pred_masks"].float().contiguous(), tg)
    wd = dict(zip(("loss_ce", "loss_mask", "loss_dice", "loss_objectness"), weights))

    def oracle(storage):
        f = {k: v.detach().double().cuda().requires_grad_(True) for k, v in feats.items()}
        es = {k: v.double().cuda().requires_grad_(True) for k, v in esd.items()}
        ds = {k: v.double().cuda().requires_grad_(True) for k, v in dsd.items()}
        x = (seo.encoder_forward_storage if storage else seo.encoder_forward)(f, es)
        o = (sso if storage else sio).decoder_forward(x, ds, groups=4)
        tm = sco.target_masks([m.cpu() for m in mask_list], (IN, IN), o["pred_masks"].shape[-2:], torch.float64).cuda()
        ref = sco.losses(o["pred_logits"], o["pred_masks"], o["pred_scores"], tm, sizes, labels.cuda(), indices, wd, float(sum(sizes)))
        sum(coef[k] * v for k, v in ref.items()).backward()
        r = {f"enc.{k}": v.grad for k, v in es.items()}
        r.update({f"dec.{k}": v.grad for k, v in ds.items()})
        r.update({f"d_{k}": v.grad for k, v in f.items()})
        return r

    _judge(got, oracle(False), oracle(True), "encoder + GroupIAMDecoder + criterion")


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    saved = dict(WORST)
    WORST.clear()
    yield
    if WORST:
        print("\nworst |err| / bound per case class: " + "; ".join(f"{k}: {v:.3g}" for k, v in sorted(WORST.items())))
    for k, v in saved.items():
        WORST[k] = max(WORST.get(k, 0.0), v)
