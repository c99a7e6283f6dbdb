"""The SparseInst IAM decoders' backward (yolov7_d2_b200.sparseinst, `_DecoderFn`): kernel by kernel, call by call, and whole.

A. Each new kernel against fp64 on exactly the operands it reads, with the bound of tests/test_convnext_plan_gpu.py (|got - ref| <= r_store |ref|
   + c(K) 2^-24 mag): the bilinear x2 adjoint, the normalisation backward (clamp-active rows, the grouped row map), the sigmoid backward (+-30 and
   +-90 logits, exact zeros in the padded maps), the data gradient through a ReLU at the decoders' geometries, and the 272-channel input dgrad.
B. Every C-ABI call of a decoder backward, recorded through the stand-in library handle of tests/test_sparseinst_kernels_gpu.py, replayed on
   fresh operands against fp64.
C. Whole decoders: the gradients of the unmodified reference (tests/golden/sparseinst_bwd.npz) and, at the shipped size, of the fp64 oracle,
   each gradient's relative L2 error <= 2.5 x that of the bf16-storage-emulating oracle + 2 %; forwards with and without autograd give the same
   bits; two backward passes give the same bits; no input gradient is computed when features do not require grad; frozen parameters get none.
D. Decoder -> SparseInstCriterion -> sum(c * loss).backward() against the oracle decoder + the fp64 criterion on the engine's match.
E. SCALE_FACTOR 1.5: the forward is unchanged and the backward raises Yb200Error.
"""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from test_convnext_plan_gpu import (R_BF16, U, WORST, _act, _g, _geo, _given, _guard_ok, _guarded, _in_view, _lib, _out_view, _outside_same, _sl,
                                    _weights, bound, check, dgrad_ref, run_dgrad)
from test_sparseinst_kernels_gpu import CLAMP, RUN, TINY, _Recorder, _decoder, _v

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------------------------------------------
# A. the new kernels against fp64
# ------------------------------------------------------------------------------------------------------------------------------------
def run_upsample_bwd(n, maps, h, w, c, seed=50):
    """yb200_upsample_bilinear2x_bwd_f32: d in = the adjoint of F.interpolate(x2, bilinear, align_corners=False), bf16 NHWC, maps >= `maps` zero"""
    capi, L = _lib()
    g = _g(seed)
    dout = torch.randn(n, maps, 2 * h, 2 * w, generator=g, device="cuda") * 3.0
    buf, dx = _guarded((n, h, w, c), float("nan"), torch.bfloat16)
    da = capi.act(dx)
    capi.check(L.yb200_upsample_bilinear2x_bwd_f32(capi.ptr(dout), maps, ctypes.byref(da), capi.stream_ptr()), "upsample_bilinear2x_bwd_f32")
    x = torch.zeros(n, maps, h, w, dtype=torch.float64, device="cuda", requires_grad=True)
    F.interpolate(x, scale_factor=2, mode="bilinear", align_corners=False).backward(dout.double())
    ref = x.grad.permute(0, 2, 3, 1)
    x.grad = None
    F.interpolate(x, scale_factor=2, mode="bilinear", align_corners=False).backward(dout.double().abs())  # the weights are >= 0
    mag = x.grad.permute(0, 2, 3, 1)
    check("bilinear x2 adjoint (bf16)", dx[..., :maps], ref, bound(ref, mag, 16, R_BF16), f"d masks {n}x{maps}x{h}x{w}")
    assert bool((dx[..., maps:] == 0).all()), "padded maps of d masks are not zero"
    _guard_ok(buf, n * h * w * c, "d masks")


def run_normalize_bwd(b, rows, cols, rows_per_group, g_rows, seed=51):
    """yb200_iam_normalize_bwd: d raw = G / max(norm, 1e-6) (bf16, both layouts), d norm = -sum G raw / max(norm, 1e-6)^2 or 0 where clamped"""
    capi, L = _lib()
    g = _g(seed)
    groups = rows // rows_per_group
    G = (torch.randn(b, 1, g_rows, groups * cols, generator=g, device="cuda")).to(torch.bfloat16)
    raw = torch.randn(b, rows, cols, generator=g, device="cuda") * 4.0
    norm = torch.rand(b, rows, generator=g, device="cuda") * 1e3 + 1e-2
    special = torch.tensor([0.0, 9.4e-14, 6400 * 9.4e-14, 5e-7, 0.999e-6, CLAMP, 1.001e-6, 2e-6, 1e-5], device="cuda")
    norm[:, 1:2 * len(special):2] = special
    draw = torch.full((b, rows, cols), float("nan"), dtype=torch.bfloat16, device="cuda")
    draw_t = torch.full((b, cols, rows), float("nan"), dtype=torch.bfloat16, device="cuda")
    buf, dnorm = _guarded((b, rows), float("nan"))
    ga = capi.act(G)
    capi.check(L.yb200_iam_normalize_bwd(ctypes.byref(ga), capi.ptr(raw), capi.ptr(norm), rows, cols, rows_per_group, capi.ptr(draw), capi.ptr(draw_t),
                                         capi.ptr(dnorm), capi.stream_ptr()), "iam_normalize_bwd")
    r = torch.arange(rows, device="cuda")
    i, k = r % rows_per_group, r // rows_per_group
    Gp = torch.cat([G, torch.zeros(b, 1, max(rows_per_group - g_rows, 0), groups * cols, dtype=G.dtype, device="cuda")], 2)
    Gr = Gp[:, 0][:, i].view(b, rows, groups, cols)[:, r, k].double()  # [b, rows, cols]: row i of the view, columns of group k
    m = norm.double().clamp_min(CLAMP)
    ref = Gr / m[..., None]
    check("normalise backward (bf16)", draw, ref, (R_BF16 + U) * ref.abs(), "d raw")
    assert torch.equal(draw_t, draw.transpose(1, 2)), "the transposed d raw differs from d raw"
    live = norm.double() >= CLAMP
    dr = draw.double() * raw.double()  # summed from the stored d raw (the kernel's documented operands)
    dref = torch.where(live, -dr.sum(-1) / m, torch.zeros_like(m))
    dmag = torch.where(live, dr.abs().sum(-1) / m, torch.zeros_like(m))
    check("normalise backward (fp32)", dnorm, dref, bound(dref, dmag, cols, 2 * U), "d normaliser")
    s = -(Gr * raw.double()).sum(-1) / m ** 2  # and that is -sum G raw / m^2 up to the bf16 rounding of d raw
    assert bool(((dref - torch.where(live, s, torch.zeros_like(s))).abs() <= R_BF16 * (Gr * raw.double()).abs().sum(-1) / m ** 2 + 1e-300).all())
    assert bool((dnorm[~live] == 0).all()) and (~live).any() and live.any()
    _guard_ok(buf, b * rows, "d normaliser")


def sigmoid_grad_bound(ref):
    """dy * e / (1 + e)^2, e = expf(-|x|) (2 ulp) and four correctly rounded operations, then the bf16 rounding; TINY where it underflows"""
    return (R_BF16 + 8 * U) * ref.abs() + TINY


def run_sigmoid_bwd(gdy, gx, gdx, group_in, group_out, seed=52):
    """yb200_sigmoid_bwd on N(0, 8^2) logits with +-30 (the padded maps' bias) and +-90 in every channel; maps >= group_in of a group are 0"""
    capi, L = _lib()
    g = _g(seed)
    dy = _in_view(gdy, g)
    x = _in_view(gx, g, scale=8.0)
    v = _sl(x, gx)
    for j, val in enumerate((-30.0, 30.0, 90.0, -90.0)):
        v[0, 0, j] = val
    dx, dx0 = _out_view(gdx, g)
    dya, xa, dxa = _act(capi, dy, gdy), _act(capi, x, gx), _act(capi, dx, gdx)
    capi.check(L.yb200_sigmoid_bwd(ctypes.byref(dya), ctypes.byref(xa), ctypes.byref(dxa), group_in, group_out, capi.stream_ptr()), "sigmoid_bwd")
    e = torch.exp(-v.double().abs())
    val = _sl(dy, gdy).double() * e / (1 + e) ** 2  # p (1 - p) would lose 1 - p near p = 1 even in fp64
    ng = gdy[3] // group_in
    got = _sl(dx, gdx).view(*gdx[:3], ng, group_out)
    ref = val.view(*gdy[:3], ng, group_in)
    check("sigmoid backward (bf16)", got[..., :group_in], ref, sigmoid_grad_bound(ref), "d iam")
    assert bool((got[..., group_in:] == 0).all()), "maps beyond group_in are not exactly zero"
    _outside_same(dx, dx0, gdx, "d iam")


def run_dgrad_relu(gdz, gdx, gh, ga, k, linear=False, seed=53):
    """yb200_conv2d_dgrad_relu (linear: yb200_linear_dgrad_relu, ksize 1, no addend): bf16((h > 0 ? dz W : 0) + addend)"""
    capi, L = _lib()
    g = _g(seed)
    dz = _in_view(gdz, g)
    cout, cin = gdz[3], gdx[3]
    w, _, wd = _weights(capi, L, cout, cin, k, g)
    h = _in_view(gh, g)
    hv = _sl(h, gh)
    hv[0, 0, 0, :8] = torch.tensor([0.0, -0.0, 1e-30, -1e-30, 0.0, 1.0, -1.0, 0.0], device="cuda").to(torch.bfloat16)  # zeros mask, like negatives
    add = _in_view(ga, g) if ga else None
    dx, dx0 = _out_view(gdx, g)
    dza, ha, dxa = _act(capi, dz, gdz), _act(capi, h, gh), _act(capi, dx, gdx)
    aa = _act(capi, add, ga) if ga else None
    if linear:
        rc = L.yb200_linear_dgrad_relu(ctypes.byref(dza), capi.ptr(wd), ctypes.byref(ha), ctypes.byref(dxa), None, capi.stream_ptr())
    else:
        rc = L.yb200_conv2d_dgrad_relu(ctypes.byref(dza), capi.ptr(wd), ctypes.byref(ha), ctypes.byref(dxa), ctypes.byref(aa) if ga else None, k, 1,
                                       capi.stream_ptr())
    capi.check(rc, "dgrad_relu")
    ref, mag, kk = dgrad_ref(_sl(dz, gdz).double(), w, k, 1, (gdx[0], gdx[1], gdx[2], cin))
    keep = (hv.double() > 0).double()
    ref, mag = ref * keep, mag * keep
    if ga:
        av = _sl(add, ga).double()
        ref, mag = ref + av, mag + av.abs()
    check("dgrad + ReLU backward (bf16)", _sl(dx, gdx), ref, bound(ref, mag, kk, R_BF16), "dx")
    _outside_same(dx, dx0, gdx, "dx")


def run_pack_dgrad(cout, cin, k, cout_pad, cin_pad, seed=54):
    """yb200_pack_conv_weight, data-gradient operand only: [cin_pad][k*k][cout_pad] bf16, zero padded"""
    capi, L = _lib()
    g = _g(seed)
    w = torch.randn(cout, cin, k, k, generator=g, device="cuda") * 0.05
    wd = torch.full((cin_pad, k * k, cout_pad), float("nan"), dtype=torch.bfloat16, device="cuda")
    capi.check(L.yb200_pack_conv_weight(capi.ptr(w), cout, cin, k, cout_pad, cin_pad, None, capi.ptr(wd), capi.stream_ptr()), "pack_conv_weight")
    want = torch.zeros(cin_pad, k * k, cout_pad, dtype=torch.bfloat16, device="cuda")
    want[:cin, :, :cout] = w.permute(1, 2, 3, 0).reshape(cin, k * k, cout).to(torch.bfloat16)
    assert torch.equal(wd.view(torch.int16), want.view(torch.int16)), "data-gradient operand differs from the bf16 rounding"


@pytest.mark.parametrize("nhw", [(2, 80, 80), (2, 13, 17), (1, 1, 65)], ids=lambda s: "x".join(map(str, s)))
def test_upsample_bwd(cuda, nhw):
    n, h, w = nhw
    run_upsample_bwd(n, 100, h, w, 112)


def test_upsample_bwd_edges(cuda):
    """single rows / columns and maps that do not fill a 64-channel pass"""
    for n, maps, h, w, c in [(1, 3, 1, 1, 8), (2, 5, 2, 33, 16), (1, 20, 7, 1, 32)]:
        run_upsample_bwd(n, maps, h, w, c, seed=55 + h)


@pytest.mark.parametrize("case", [(2, 112, 256, 112, 112), (2, 416, 256, 104, 112), (1, 96, 64, 24, 32), (3, 32, 64, 32, 32)],
                         ids=["base", "group", "group-small", "base-small"])
def test_normalize_bwd(cuda, case):
    run_normalize_bwd(*case)


@pytest.mark.parametrize("case", [((2, 40, 40, 112, 112, 0), 112, 112, 1), ((2, 40, 40, 416, 416, 0), 104, 128, 4), ((1, 9, 13, 96, 96, 0), 24, 32, 4)],
                         ids=["base", "group", "group-small"])
def test_sigmoid_bwd(cuda, case):
    gdy, gi, go, ng = case
    run_sigmoid_bwd(gdy, gdy, gdy[:3] + (go * ng, go * ng, 0), gi, go)


DGRAD_RELU = {
    "inst-conv 256": ((2, 80, 80, 256, 256, 0), (2, 80, 80, 256, 256, 0), False),
    "iam 112 + addend": ((2, 80, 80, 112, 112, 0), (2, 80, 80, 256, 256, 0), True),
    "group slice 2": ((2, 64, 64, 128, 512, 256), (2, 64, 64, 64, 256, 128), True),
    "group slice 3": ((2, 40, 40, 128, 512, 384), (2, 40, 40, 64, 256, 192), False),
}


@pytest.mark.parametrize("name", list(DGRAD_RELU))
def test_dgrad_relu(cuda, name):
    gdz, gdx, with_add = DGRAD_RELU[name]
    run_dgrad_relu(gdz, gdx, gdx, gdx if with_add else None, 3)


@pytest.mark.parametrize("with_addend", [False, True])
def test_input_dgrad_272(cuda, with_addend):
    """the input's data gradient: 256 -> 272 channels (2 coordinates + 256 features + 14 zero), plain dgrad, the second with the first as addend"""
    g = (2, 80, 80, 272, 272, 0)
    run_dgrad((2, 80, 80, 256, 256, 0), g, g if with_addend else None, 3, 1)


# ------------------------------------------------------------------------------------------------------------------------------------
# B. every call of a decoder backward, replayed
# ------------------------------------------------------------------------------------------------------------------------------------
BWD_ENTRY_POINTS = {"yb200_upsample_bilinear2x_bwd_f32", "yb200_conv2d_wgrad_workspace", "yb200_conv2d_wgrad", "yb200_pack_conv_weight", "yb200_conv2d_dgrad",
                    "yb200_linear_dgrad_relu", "yb200_colsum_workspace", "yb200_colsum", "yb200_iam_normalize_bwd", "yb200_conv2d_affine_fwd",
                    "yb200_sigmoid_bwd", "yb200_conv2d_dgrad_relu"}
QUERIES = ("yb200_conv2d_wgrad_workspace", "yb200_colsum_workspace")
BWD_MAPS = {"Base": [(2, 80, 80), (2, 64, 64), (1, 13, 17)], "Group": [(2, 64, 64), (2, 40, 40)]}
REPLAY = dict(RUN, upsample_bwd=run_upsample_bwd, normalize_bwd=run_normalize_bwd, sigmoid_bwd=run_sigmoid_bwd, dgrad_relu=run_dgrad_relu,
              pack_dgrad=run_pack_dgrad, dgrad=run_dgrad)


def _bwd_case(name, a):
    if name == "yb200_upsample_bilinear2x_bwd_f32":
        d = _geo(a[2])
        return dict(fn="upsample_bwd", n=d[0], maps=a[1], h=d[1], w=d[2], c=d[3])
    if name == "yb200_conv2d_wgrad":
        return dict(fn="wgrad", gx=_geo(a[0]), gdz=_geo(a[1]), k=a[2], s=a[3], cin_real=a[4], accumulate=a[6])
    if name == "yb200_pack_conv_weight":
        assert not _given(a[6]) and _given(a[7]), "the backward packs data-gradient operands only"
        return dict(fn="pack_dgrad", cout=a[1], cin=a[2], k=a[3], cout_pad=a[4], cin_pad=a[5])
    if name == "yb200_conv2d_dgrad":
        return dict(fn="dgrad", gdz=_geo(a[0]), gdx=_geo(a[2]), ga=_geo(a[3]), k=a[4], s=a[5])
    if name == "yb200_linear_dgrad_relu":
        assert not _given(a[4]), "the decoder backward sums biases with yb200_colsum, not the atomic bias sum"
        return dict(fn="dgrad_relu", gdz=_geo(a[0]), gdx=_geo(a[3]), gh=_geo(a[2]), ga=None, k=1, linear=True)
    if name == "yb200_conv2d_dgrad_relu":
        return dict(fn="dgrad_relu", gdz=_geo(a[0]), gdx=_geo(a[3]), gh=_geo(a[2]), ga=_geo(a[4]), k=a[5])
    if name == "yb200_colsum":
        return dict(fn="colsum", gx=_geo(a[0]), scale=_v(a[1]), accumulate=a[3])
    if name == "yb200_iam_normalize_bwd":
        gg = _geo(a[0])
        return dict(fn="normalize_bwd", b=gg[0], rows=a[3], cols=a[4], rows_per_group=a[5], g_rows=gg[2])
    if name == "yb200_conv2d_affine_fwd":
        return dict(fn="affine", gx=_geo(a[0]), go=_geo(a[5]), gr=_geo(a[4]), k=a[6], s=a[7], with_scale=_given(a[2]), with_shift=_given(a[3]))
    if name == "yb200_sigmoid_bwd":
        return dict(fn="sigmoid_bwd", gdy=_geo(a[0]), gx=_geo(a[1]), gdx=_geo(a[2]), group_in=a[3], group_out=a[4])
    if name in QUERIES:
        return None
    raise AssertionError(f"{name}: a decoder backward call this module does not replay")


def _backward_recorded(dec, feat, seed, refuse=()):
    """one forward with autograd, then the backward of seeded upstream gradients through the stand-in handle: (log, grads, d features)"""
    out = dec(feat)
    g = _g(seed)
    ups = [torch.randn(t.shape, generator=g, device="cuda") * s for t, s in ((out["pred_logits"], 1.0), (out["pred_masks"], 0.1), (out["pred_scores"], 1.0))]
    rec = _Recorder(dec.L, refuse)
    dec.L = rec
    try:
        for p in dec.parameters():
            p.grad = None
        torch.autograd.backward([out["pred_logits"], out["pred_masks"], out["pred_scores"]], ups)
        torch.cuda.synchronize()
    finally:
        dec.L = rec._lib
    return rec.log


BWD_RECORDINGS = {}


def _bwd_recordings():
    if not BWD_RECORDINGS and torch.cuda.is_available():
        for kind, maps in BWD_MAPS.items():
            dec, _ = _decoder(kind, seed=60)
            BWD_RECORDINGS[kind] = []
            for i, (n, h, w) in enumerate(maps):
                feat = torch.randn(n, 256, h, w, generator=_g(61 + i), device="cuda").requires_grad_(True)
                log = _backward_recorded(dec, feat, 62 + i)
                BWD_RECORDINGS[kind].append(((n, h, w), log))
            del dec
        torch.cuda.empty_cache()
    return BWD_RECORDINGS


def _bwd_distinct():
    seen, out = set(), []
    for kind, recs in _bwd_recordings().items():
        for _, log in recs:
            for name, a, _ in log:
                case = _bwd_case(name, a)
                if case is None:
                    continue
                key = tuple(sorted((k, str(v)) for k, v in case.items()))
                if key in seen:
                    continue
                seen.add(key)
                out.append((f"{kind}: {name[len('yb200_'):]} " + " ".join(f"{k}={v}" for k, v in case.items() if k != "fn"), case))
    return out


def pytest_generate_tests(metafunc):
    if "bwd_case" in metafunc.fixturenames:
        cases = _bwd_distinct()
        metafunc.parametrize("bwd_case", [c[1] for c in cases], ids=[c[0] for c in cases])


def test_backward_call(cuda, bwd_case):
    case = dict(bwd_case)
    REPLAY[case.pop("fn")](**case)


def test_backward_recording_is_complete(cuda):
    """every entry point a decoder backward calls is replayed; the group backward's d iam is 128 maps per group ([.., 512]); no atomics"""
    recs = _bwd_recordings()
    for kind in BWD_MAPS:
        names = {name for _, log in recs[kind] for name, _, _ in log}
        assert names == BWD_ENTRY_POINTS, f"{kind}: entry points called {sorted(names)}, replayed {sorted(BWD_ENTRY_POINTS)}"
        assert all(rc == 0 for _, log in recs[kind] for name, _, rc in log if name not in QUERIES), f"{kind}: a backward call failed"
    cases = [c for _, c in _bwd_distinct()]
    grp = [c for c in cases if c["fn"] == "dgrad_relu" and c["gdz"][4] == 512]
    assert {c["gdz"][5] for c in grp} == {0, 128, 256, 384} and all(c["gdz"][3] == 128 and c["gdx"][3] == 64 for c in grp), grp
    assert any(c["fn"] == "wgrad" and c["gdz"][3:5] == (128, 512) for c in cases), "no 128-of-512 weight gradient of the grouped IAM conv"
    assert any(c["fn"] == "sigmoid_bwd" and (c["group_in"], c["group_out"]) == (104, 128) for c in cases)
    assert any(c["fn"] == "dgrad" and c["gdx"][3] == 272 and c["ga"] is not None for c in cases), "no input dgrad with addend"


# ------------------------------------------------------------------------------------------------------------------------------------
# C. whole decoders
# ------------------------------------------------------------------------------------------------------------------------------------
def rel_l2(got, ref):
    got, ref = got.double().cpu(), ref.double().cpu()
    return float((got - ref).norm() / ref.norm().clamp_min(1e-300))


def _judge(grads, ref, emu, what):
    """DETR's rule: every gradient's relative L2 error <= 2.5 x the storage-emulating oracle's + 2 %"""
    bad = []
    for k in ref:
        e, y = rel_l2(grads[k], ref[k]), rel_l2(emu[k], ref[k])
        WORST["whole-decoder rel-L2 / allowance"] = max(WORST.get("whole-decoder rel-L2 / allowance", 0.0), e / (2.5 * y + 0.02))
        if not e <= 2.5 * y + 0.02:
            bad.append(f"{k}: rel L2 {e:.4f} vs emulated {y:.4f}")
    assert not bad, f"{what}: " + "; ".join(bad)


def _oracle(feat, sd, groups, ups, num_convs, emulate, device):
    """fp64 gradients of the oracle decoder (emulate: of its bf16-storage restatement, oracle/sparseinst_storage_oracle.py)"""
    from oracle import sparseinst_oracle as sio
    from oracle import sparseinst_storage_oracle as sso

    feat = feat.detach().double().to(device).requires_grad_(True)
    sdd = {k: v.detach().double().to(device).requires_grad_(True) for k, v in sd.items()}
    out = (sso if emulate else sio).decoder_forward(feat, sdd, num_convs=num_convs, groups=groups)
    torch.autograd.backward([out["pred_logits"], out["pred_masks"], out["pred_scores"]], [u.double().to(device) for u in ups])
    g = {k: v.grad for k, v in sdd.items()}
    g["features"] = feat.grad
    return g


def _engine(dec, feat, ups):
    feat = feat.detach().cuda().requires_grad_(True)
    for p in dec.parameters():
        p.grad = None
    out = dec(feat)
    torch.autograd.backward([out["pred_logits"], out["pred_masks"], out["pred_scores"]], [u.cuda() for u in ups])
    g = {k: p.grad for k, p in dec.named_parameters()}
    g["features"] = feat.grad
    return g, out


def _small_decoder(case):
    from test_sparseinst_gpu import _cfg
    from yolov7_d2_b200.sparseinst import BaseIAMDecoder, GroupIAMDecoder

    from oracle.gen_golden_sparseinst_bwd import state_dict

    _, groups, _, _, _, _, d = case
    cfg = _cfg(d["dim"], d["nm"], d["kd"], d["nc"], d["convs"], d["cin"])
    if groups:
        cfg.MODEL.SPARSE_INST.DECODER.GROUPS = groups
    dec = (GroupIAMDecoder if groups else BaseIAMDecoder)(cfg)
    sd = state_dict(case)
    dec.load_state_dict({k: v.cuda() for k, v in sd.items()}, strict=True)
    return dec, sd


def _fixture_cases():
    from oracle.gen_golden_sparseinst_bwd import CASES

    return CASES


@pytest.mark.parametrize("case", _fixture_cases(), ids=[c[0] for c in _fixture_cases()])
def test_gradients_match_the_reference(cuda, case):
    from test_sparseinst_bwd_oracle_golden import gold_grads

    from oracle.gen_golden_sparseinst_bwd import case_upstream, features

    groups, d = case[1], case[6]
    dec, sd = _small_decoder(case)
    feat = features(case).float()
    ups = [u.float() for u in case_upstream(case)]
    got, _ = _engine(dec, feat, ups)
    ref = gold_grads(case)
    emu = _oracle(feat, sd, groups, ups, d["convs"], True, "cpu")
    assert sorted(got) == sorted(ref)
    _judge(got, ref, emu, case[0])


@pytest.mark.parametrize("kind", ["Base", "Group"])
def test_shipped_size_against_fp64(cuda, kind):
    """2 x 256 x 80 x 80, 100 masks, dim 256, kernel dim 128, 80 classes: every gradient against the fp64 oracle on the device"""
    dec, sd = _decoder(kind, seed=70)
    groups = 4 if kind == "Group" else 0
    g = torch.Generator().manual_seed(71)
    feat = torch.randn(2, 256, 80, 80, generator=g)
    ups = [torch.randn(2, 100, 80, generator=g), torch.randn(2, 100, 160, 160, generator=g) * 0.1, torch.randn(2, 100, 1, generator=g)]
    got, _ = _engine(dec, feat, ups)
    ref = _oracle(feat, sd, groups, ups, 4, False, "cuda")
    emu = _oracle(feat, sd, groups, ups, 4, True, "cuda")
    assert all(got[k] is not None and torch.isfinite(got[k]).all() for k in ref), "missing or non-finite gradients"
    _judge(got, ref, emu, kind)


@pytest.mark.parametrize("kind", ["Base", "Group"])
def test_grad_mode_forward_and_backward_are_bit_exact(cuda, kind):
    """grad-mode outputs = no-grad outputs, bit for bit; two identical backward passes give the same bits (2 x 64 x 64 and the per-image mask GEMM
    path at 2 x 40 x 40)"""
    dec, _ = _decoder(kind, seed=72)
    for i, (n, h, w) in enumerate([(2, 64, 64), (2, 40, 40)]):
        feat = torch.randn(n, 256, h, w, generator=_g(73 + i), device="cuda")
        with torch.no_grad():
            ref = dec(feat)
        g = _g(75 + i)
        ups = [torch.randn(ref[k].shape, generator=g, device="cuda") for k in ("pred_logits", "pred_masks", "pred_scores")]
        runs = [_engine(dec, feat, ups) for _ in range(2)]
        for k in ref:
            assert torch.equal(runs[0][1][k], ref[k]), f"{k}: the grad-mode forward differs from the no-grad forward"
        for k, v in runs[0][0].items():
            assert torch.equal(v, runs[1][0][k]), f"{k}: two backward passes differ"


def test_no_input_gradient_without_requires_grad(cuda):
    dec, _ = _decoder("Base", seed=76)
    feat = torch.randn(2, 256, 40, 40, generator=_g(77), device="cuda")
    log = _backward_recorded(dec, feat, 78)
    first = [a for name, a, _ in log if name == "yb200_conv2d_dgrad" and _geo(a[2])[3] == 272]
    assert not first, "a first-layer data gradient ran for features that do not require grad"
    assert all(p.grad is not None for p in dec.parameters())


def test_frozen_parameters_get_no_gradient(cuda):
    dec, _ = _decoder("Group", seed=79)
    frozen = {"mask_branch.projection.weight", "inst_branch.iam_conv.bias", "inst_branch.fc.weight", "inst_branch.inst_convs.0.weight"}
    for k, p in dec.named_parameters():
        p.requires_grad_(k not in frozen)
    feat = torch.randn(2, 256, 40, 40, generator=_g(80), device="cuda").requires_grad_(True)
    _backward_recorded(dec, feat, 81)
    for k, p in dec.named_parameters():
        assert (p.grad is None) == (k in frozen), k
    assert feat.grad is not None and torch.isfinite(feat.grad).all()


# ------------------------------------------------------------------------------------------------------------------------------------
# D. decoder + criterion
# ------------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["Base", "Group"])
def test_decoder_and_criterion_train_end_to_end(cuda, kind):
    """one training step's gradients: decoder -> SparseInstCriterion -> sum(c * loss).backward(), against the oracle decoder and the fp64
    criterion on the engine's match, under the same yardstick"""
    from test_sparseinst_criterion_gpu import _cfg as crit_cfg
    from test_sparseinst_criterion_gpu import _ellipses
    from yolov7_d2_b200.sparseinst_criterion import _Targets, build_sparse_inst_criterion

    from oracle import sparseinst_criterion_oracle as sco
    from oracle import sparseinst_oracle as sio
    from oracle import sparseinst_storage_oracle as sso

    dec, sd = _decoder(kind, seed=82)
    groups = 4 if kind == "Group" else 0
    g = torch.Generator().manual_seed(83)
    B, IN, H = 2, 320, 40
    feat = torch.randn(B, 256, H, H, generator=g)
    sizes = [3, 5]
    mask_list = [_ellipses(g, n, IN - 16 * b, IN) for b, n in enumerate(sizes)]
    labels = torch.randint(0, 80, (sum(sizes),), generator=g)
    off = np.concatenate([[0], np.cumsum(sizes)])
    targets = [{"labels": labels[off[b]:off[b + 1]].cuda(), "masks": sco.BitMasks(m.cuda())} for b, m in enumerate(mask_list)]
    coef = {"loss_ce": 0.7, "loss_objectness": 1.3, "loss_dice": 0.4, "loss_mask": 1.9}
    weights = (2.0, 5.0, 2.0, 1.0)
    crit = build_sparse_inst_criterion(crit_cfg(80, 0.8, 0.2, weights))
    fcu = feat.cuda().requires_grad_(True)
    out = dec(fcu)
    losses = crit(out, targets, (IN, IN))
    sum(coef[k] * v for k, v in losses.items()).backward()
    got = {k: p.grad for k, p in dec.named_parameters()}
    got["features"] = fcu.grad
    assert all(v is not None and torch.isfinite(v).all() and v.abs().sum() > 0 for v in got.values()), "a decoder parameter got no gradient"
    tg_out = {k: out[k].detach() for k in ("pred_logits", "pred_masks", "pred_scores")}
    tg = _Targets(targets, (IN, IN), tg_out["pred_masks"].shape, cuda, "test")
    indices, _ = crit.matcher.match(tg_out["pred_logits"].float().contiguous(), tg_out["pred_masks"].float().contiguous(), tg)
    wd = dict(zip(("loss_ce", "loss_mask", "loss_dice", "loss_objectness"), weights))

    def oracle(emulate):
        f = feat.double().cuda().requires_grad_(True)
        sdd = {k: v.double().cuda().requires_grad_(True) for k, v in sd.items()}
        o = (sso if emulate else sio).decoder_forward(f, sdd, groups=groups)
        tm = sco.target_masks([m.cpu() for m in mask_list], (IN, IN), o["pred_masks"].shape[-2:], torch.float64).cuda()
        ref = sco.losses(o["pred_logits"], o["pred_masks"], o["pred_scores"], tm, sizes, labels.cuda(), indices, wd, float(sum(sizes)))
        sum(coef[k] * v for k, v in ref.items()).backward()
        r = {k: v.grad for k, v in sdd.items()}
        r["features"] = f.grad
        return r

    _judge(got, oracle(False), oracle(True), f"{kind} + criterion")


# ------------------------------------------------------------------------------------------------------------------------------------
# E. errors
# ------------------------------------------------------------------------------------------------------------------------------------
def test_scale_factor_other_than_two_has_no_backward(cuda):
    from test_sparseinst_gpu import _cfg
    from yolov7_d2_b200 import capi
    from yolov7_d2_b200.sparseinst import BaseIAMDecoder

    from oracle import sparseinst_oracle as sio

    cfg = _cfg(64, 20, 32, 8, 2, 30)
    cfg.MODEL.SPARSE_INST.DECODER.SCALE_FACTOR = 1.5
    dec = BaseIAMDecoder(cfg)
    sd = sio.decoder_state_dict(84, in_channels=30, dim=64, num_masks=20, kernel_dim=32, num_classes=8, num_convs=2)
    dec.load_state_dict({k: v.cuda() for k, v in sd.items()}, strict=True)
    feat = torch.randn(2, 30, 12, 20, generator=_g(85), device="cuda")
    with torch.no_grad():
        ref = dec(feat)
    out = dec(feat.clone().requires_grad_(True))
    for k in ref:
        assert torch.equal(out[k].detach(), ref[k]), k
    with pytest.raises(capi.Yb200Error, match="backward implemented for SCALE_FACTOR 2"):
        out["pred_masks"].sum().backward()


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    saved = dict(WORST)
    WORST.clear()
    yield
    if WORST:
        print("\nworst |err| / bound per case class: " + "; ".join(f"{k}: {v:.3g}" for k, v in sorted(WORST.items())))
    for k, v in saved.items():
        WORST[k] = max(WORST.get(k, 0.0), v)

