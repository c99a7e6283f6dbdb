"""The SparseInst IAM decoders' kernels, call by call, against fp64 at the shipped configuration, and the batched mask GEMM on its own.

tests/test_sparseinst_gpu.py checks the decoders end to end (5e-2 of each output's max after about twelve bf16 kernels); this module checks
every kernel the decoders call, on the geometries they call it with, against the bound of tests/test_convnext_plan_gpu.py:

    |got - ref| <= r_store * |ref| + c(K) * 2^-24 * mag,      c(K) = 16 * sqrt(K) + 16

with the references of that module where one exists (convolutions, the pixel contraction, the prediction GEMM) and the ones below for the
rest (sigmoid, normalise, column sums, the per-image 1x1 GEMM, the bilinear x2).  Every reference runs in float64 on exactly the bf16 /
fp32 operands the kernel reads.  tests/test_sparseinst_kernels_tol_cpu.py shows that the bound rejects the defects these kernels could
plausibly have (a neighbour image's kernels, a dropped k-block or 16-row slice, a pixel tile dropped or counted twice, an unclamped
normaliser, a sigmoid read one channel off).

A. One forward of each decoder (Base at 2x80x80, 2x64x64, 2x40x40, 1x13x17; Group at 2x64x64, 2x40x40) runs through a stand-in for the
   library handle that records every call; each distinct geometry is replayed on fresh buffers (input channels outside a view hold 2^14,
   output channels outside a view must keep their bits, output elements inside a view start as NaN).
B. yb200_conv1x1_nchw_f32_batched, the batch's mask GEMM with one weight matrix per image: which maps it accepts (one image per 128-pixel
   tile as choose_tile picks it), per-image kernels scaled by 2^(12 b) so that reading a neighbour's rows is a gross error, invariance under
   a permutation of the images, and bit equality with the per-image yb200_conv1x1_nchw_f32.
C. The decoders on the batched path against the fp32 oracle, the routing between batched and per-image calls, and bit equality of the
   batched path with the per-image fallback and of two identical forwards.
"""
import ctypes
import math

import pytest
import torch
import torch.nn.functional as F

from test_convnext_plan_gpu import (R_BF16, U, WORST, _act, _g, _geo, _given, _guard_ok, _guarded, _in_view, _lib, _out_view, _outside_same,
                                    _sl, _weights, bound, check, conv_ref, run_affine, run_pred, run_wgrad)

pytestmark = pytest.mark.gpu

CLAMP = float(torch.tensor(1e-6, dtype=torch.float32))  # fmaxf(norm, 1e-6f) of iam_normalize_kernel: the fp32 value of 1e-6
TINY = 2.0 ** -126  # sigmoid: 1 / (1 + e) with e > 2^126 may flush to 0 (__fdividef), and so may a result below the smallest normal


# ------------------------------------------------------------------------------------------------------------------------------------
# fp64 references for the kernels tests/test_convnext_plan_gpu.py has none for; each returns (ref, bound) or (ref, mag, K)
# ------------------------------------------------------------------------------------------------------------------------------------
def sigmoid_bound(x, ref):
    """bf16(__fdividef(1, 1 + __expf(-x))): __expf is within 2 + 1.173 |x| ulp (CUDA programming guide, intrinsic functions), the addition
    rounds once, __fdividef is within 2 ulp; an error d relative to e = exp(-x) moves 1 / (1 + e) by at most d relative.  So the fp32 value
    is within (6 + 1.173 |x|) * 2^-23 of the result, relative, before the bf16 rounding, plus TINY where it underflows."""
    return (R_BF16 + (6.0 + 1.173 * x.abs()) * 2.0 ** -23) * ref.abs() + TINY


def sigmoid_ref(x):
    ref = torch.sigmoid(x)
    return ref, sigmoid_bound(x, ref)


def normalize_ref(raw, norm):
    """inst[r][c] = raw[r][c] / max(norm[r], 1e-6f): one IEEE fp32 division (at most 2^-24 relative), one bf16 rounding"""
    ref = raw / norm.clamp_min(CLAMP)[:, None]
    return ref, (R_BF16 + U) * ref.abs()


def colsum_ref(x, scale=1.0):
    """column sums over every pixel of an NHWC view: K = pixels"""
    x2 = x.reshape(-1, x.shape[-1])
    return scale * x2.sum(0), abs(scale) * x2.abs().sum(0), x2.shape[0]


def bmm_ref(x, wimg):
    """out[n][o][y][x] = sum_c x[n][y][x][c] * w[n][o][c]: torch.bmm(pred_kernel, mask_features) with one weight matrix per image
    (wimg [n or 1][cout][c]); fp32 NCHW"""
    wimg = wimg.expand(x.shape[0], -1, -1)
    ref = torch.einsum("nhwc,noc->nohw", x, wimg)
    mag = torch.einsum("nhwc,noc->nohw", x.abs(), wimg.abs())
    return ref, mag, x.shape[-1]


def upsample_ref(x):
    """F.interpolate(scale_factor=2, bilinear, align_corners=False) in fp64: each output is a convex combination of 4 inputs"""
    ref = F.interpolate(x[None], scale_factor=2, mode="bilinear", align_corners=False)[0]
    mag = F.interpolate(x.abs()[None], scale_factor=2, mode="bilinear", align_corners=False)[0]
    return ref, mag, 4


def choose_tile(n, h, w, npix=128):
    """restatement of choose_tile (csrc/host_common.cu): the (log2 width, log2 height) of the pixel tile with the fewest padded pixels;
    ties keep the widest, then the tallest tile; the rest of the npix pixels span images"""
    lp = npix.bit_length() - 1
    best, pick = None, None
    for lw in range(lp, -1, -1):
        for lh in range(lp - lw, -1, -1):
            tw, th, tn = 1 << lw, 1 << lh, npix >> (lw + lh)
            cost = -(-w // tw) * tw * -(-h // th) * th * -(-n // tn) * tn
            if best is None or cost < best:
                best, pick = cost, (lw, lh)
    return pick


def batched_accepts(n, h, w):
    """yb200_conv1x1_nchw_f32_batched computes a map when each 128-pixel tile holds one image: tile width x height = 128 pixels"""
    lw, lh = choose_tile(n, h, w)
    return lw + lh == 7


BATCHED_ACCEPTED = [(2, 80, 80), (2, 64, 64), (2, 72, 96), (3, 96, 96), (1, 13, 17), (2, 1, 65)]
BATCHED_REFUSED = [(2, 40, 40), (2, 12, 20), (2, 60, 80)]


# ------------------------------------------------------------------------------------------------------------------------------------
# replays of the kernels tests/test_convnext_plan_gpu.py does not replay
# ------------------------------------------------------------------------------------------------------------------------------------
def run_pack(cout, cin, k, cout_pad, cin_pad, seed=20):
    """yb200_pack_conv_weight: OIHW fp32 -> [cout_pad][k*k][cin_pad] bf16, round to nearest even, zero padding"""
    capi, L = _lib()
    g = _g(seed)
    w = torch.randn(cout, cin, k, k, generator=g, device="cuda") * 0.05
    ties = w.view(-1)[:64]  # exact halfway cases: 1 + 2^-8 and 1 + 3 * 2^-8 round to even (down, then up)
    ties.copy_(torch.tensor([1.0 + 2.0 ** -8, -(1.0 + 3 * 2.0 ** -8)] * 32, device="cuda") * 2.0 ** -6)
    n = cout_pad * k * k * cin_pad
    buf, wf = _guarded((cout_pad, k * k, cin_pad), float("nan"), torch.bfloat16)
    capi.check(L.yb200_pack_conv_weight(capi.ptr(w), cout, cin, k, cout_pad, cin_pad, capi.ptr(wf), None, capi.stream_ptr()), "pack_conv_weight")
    want = torch.zeros(cout_pad, k * k, cin_pad, dtype=torch.bfloat16, device="cuda")
    want[:cout, :, :cin] = w.permute(0, 2, 3, 1).reshape(cout, k * k, cin).to(torch.bfloat16)
    assert torch.equal(wf.view(torch.int16), want.view(torch.int16)), \
        f"packed weights differ from the bf16 rounding in {int((wf.view(torch.int16) != want.view(torch.int16)).sum())} of {n} elements"
    _guard_ok(buf, n, "packed weights")


def run_relu(gx, go, k, s, seed=21):
    """yb200_conv2d_relu_fwd: bf16(max(conv + bias, 0)); ReLU is 1-Lipschitz, so the convolution's bound carries over"""
    capi, L = _lib()
    g = _g(seed)
    x = _in_view(gx, g)
    cin, cout = gx[3], go[3]
    w, wf, _ = _weights(capi, L, cout, cin, k, g, dgrad=False)
    b = torch.randn(cout, generator=g, device="cuda") * 0.5
    out, out0 = _out_view(go, g)
    xa, oa = _act(capi, x, gx), _act(capi, out, go)
    capi.check(L.yb200_conv2d_relu_fwd(ctypes.byref(xa), capi.ptr(wf), capi.ptr(b), ctypes.byref(oa), k, s, capi.stream_ptr()), "conv2d_relu_fwd")
    ref, mag, kk = conv_ref(_sl(x, gx).double(), w, k, s)
    ref, mag = (ref + b.double()).clamp_min(0.0), mag + b.double().abs()
    check("conv + bias + ReLU (bf16)", _sl(out, go), ref, bound(ref, mag, kk, R_BF16), "out")
    _outside_same(out, out0, go, "out")


def run_sigmoid(gx, go, seed=22):
    """yb200_sigmoid on N(0, 8^2) logits, with the padded maps' -30 and +-90 (where __expf overflows / underflows) in every channel"""
    capi, L = _lib()
    g = _g(seed)
    x = _in_view(gx, g, scale=8.0)
    v = _sl(x, gx)
    for i, val in enumerate((-30.0, 90.0, -90.0, -88.0, 88.0)):
        v[0, 0, i] = val
    out, out0 = _out_view(go, g)
    xa, oa = _act(capi, x, gx), _act(capi, out, go)
    capi.check(L.yb200_sigmoid(ctypes.byref(xa), ctypes.byref(oa), capi.stream_ptr()), "sigmoid")
    got = _sl(out, go)
    ref, bnd = sigmoid_ref(v.double())
    check("sigmoid (bf16)", got, ref, bnd, "prob")
    assert bool((got[0, 0, 1] == 1).all()) and bool((got[0, 0, 2] == 0).all()), "sigmoid(+-90) must round to 1 / 0"
    _outside_same(out, out0, go, "prob")


def run_colsum(gx, scale, accumulate, seed=23):
    """yb200_colsum over the probabilities (K = pixels): fp32 per-channel sums of block partials"""
    capi, L = _lib()
    g = _g(seed)
    x = _in_view(gx, g)
    v = _sl(x, gx)
    v.copy_(torch.sigmoid(v.float() * 4.0).to(torch.bfloat16))  # probabilities, as the decoder sums them
    c = gx[3]
    o0 = torch.randn(c, generator=g, device="cuda")
    buf, out = _guarded((c,), o0 if accumulate else float("nan"))
    xa = _act(capi, x, gx)
    ws = torch.empty(max(16, L.yb200_colsum_workspace(ctypes.byref(xa))), dtype=torch.uint8, device="cuda")
    capi.check(L.yb200_colsum(ctypes.byref(xa), ctypes.c_float(scale), capi.ptr(out), accumulate, capi.ptr(ws), capi.stream_ptr()), "colsum")
    ref, mag, kk = colsum_ref(v.double(), scale)
    if accumulate:
        ref, mag = ref + o0.double(), mag + o0.double().abs()
    check("column sums (fp32)", out, ref, bound(ref, mag, kk, 0.0), "sums")
    _guard_ok(buf, c, "sums")


def run_normalize(rows, cols, go, seed=24):
    """yb200_iam_normalize with normalisers on both sides of the 1e-6 clamp: summed probabilities of real maps, the padded maps' H*W*9.4e-14
    (always clamped), zero, and values just below, at and just above the clamp"""
    capi, L = _lib()
    g = _g(seed)
    raw = torch.randn(rows, cols, generator=g, device="cuda") * 4.0
    norm = torch.rand(rows, generator=g, device="cuda") * 1e3 + 1e-2
    special = torch.tensor([0.0, 9.4e-14, 6400 * 9.4e-14, 5e-7, 0.999e-6, CLAMP, 1.001e-6, 2e-6, 1e-5], device="cuda")
    norm[1:2 * len(special):2] = special
    norm[-12:] = 6400 * 9.4e-14
    out, out0 = _out_view(go, g)
    oa = _act(capi, out, go)
    capi.check(L.yb200_iam_normalize(capi.ptr(raw), capi.ptr(norm), rows, cols, ctypes.byref(oa), capi.stream_ptr()), "iam_normalize")
    ref, bnd = normalize_ref(raw.double(), norm.double())
    assert (norm < CLAMP).any() and (norm > CLAMP).any()
    check("normalise (bf16)", _sl(out, go)[0, 0], ref, bnd, "inst")
    _outside_same(out, out0, go, "inst")


def _img_weights(nimg, cout, c, g):
    """bf16 kernels [nimg][cout][c]; image b's are scaled by 2^(12 b), so that reading a neighbour's rows is a gross error"""
    w = torch.randn(nimg, cout, c, generator=g, device="cuda") / math.sqrt(c)
    w = w * torch.tensor([2.0 ** (12 * b) for b in range(nimg)], device="cuda")[:, None, None]
    return w.to(torch.bfloat16)


def _nchw_call(capi, L, x, wimg, cout, out, batched, bias=None):
    xa = capi.act(x)
    if batched:
        return L.yb200_conv1x1_nchw_f32_batched(ctypes.byref(xa), capi.ptr(wimg), cout, capi.ptr(out), capi.stream_ptr())
    return L.yb200_conv1x1_nchw_f32(ctypes.byref(xa), capi.ptr(wimg), capi.ptr(bias), cout, capi.ptr(out), capi.stream_ptr())


def _refused(capi, L, x, wimg, cout, g):
    n, h, w, _ = x.shape
    out = torch.randn(n, cout, h, w, generator=g, device="cuda")
    out0 = out.clone()
    rc = _nchw_call(capi, L, x, wimg, cout, out, True)
    torch.cuda.synchronize()
    assert rc == capi.ERR_UNSUPPORTED, (rc, L.yb200_last_error())
    assert torch.equal(out, out0), "a refused call wrote its output"


def run_nchw(gx, cout, batched, bias=False, seed=25):
    """yb200_conv1x1_nchw_f32[_batched]: fp32 NCHW [n][cout][h][w] = the image's kernels x its mask features; a batched call at a map
    where a pixel tile would span images must be refused and leave its output alone"""
    capi, L = _lib()
    g = _g(seed)
    x = _in_view(gx, g)
    n, h, w, c = gx[:4]
    wimg = _img_weights(n if batched else 1, cout, c, g)
    b = torch.randn(cout, generator=g, device="cuda") if bias else None
    if batched and not batched_accepts(n, h, w):
        _refused(capi, L, _sl(x, gx).contiguous(), wimg, cout, g)
        return
    buf, out = _guarded((n, cout, h, w), float("nan"))
    capi.check(_nchw_call(capi, L, _sl(x, gx).contiguous(), wimg, cout, out, batched, b), "conv1x1_nchw_f32" + ("_batched" if batched else ""))
    ref, mag, kk = bmm_ref(_sl(x, gx).double(), wimg.double())
    if bias:
        ref, mag = ref + b.double()[:, None, None], mag + b.double().abs()[:, None, None]
    check("mask GEMM (fp32)", out, ref, bound(ref, mag, kk, 0.0), "masks")
    _guard_ok(buf, n * cout * h * w, "masks")


def run_upsample(planes, h, w, seed=26):
    """yb200_upsample_bilinear2x_f32 at the decoder's plane count"""
    capi, L = _lib()
    g = _g(seed)
    x = torch.randn(planes, h, w, generator=g, device="cuda") * 3.0
    buf, out = _guarded((planes, 2 * h, 2 * w), float("nan"))
    capi.check(L.yb200_upsample_bilinear2x_f32(capi.ptr(x), capi.ptr(out), ctypes.c_int64(planes), h, w, capi.stream_ptr()), "upsample")
    ref, mag, kk = upsample_ref(x.double())
    check("bilinear x2 (fp32)", out, ref, bound(ref, mag, kk, 0.0), "up")
    _guard_ok(buf, planes * 4 * h * w, "up")


RUN = dict(pack=run_pack, relu=run_relu, affine=run_affine, sigmoid=run_sigmoid, wgrad=run_wgrad, colsum=run_colsum, normalize=run_normalize,
           pred=run_pred, nchw=run_nchw, upsample=run_upsample)


# ------------------------------------------------------------------------------------------------------------------------------------
# A. recording the decoders
# ------------------------------------------------------------------------------------------------------------------------------------
BATCHED, PER_IMAGE = "yb200_conv1x1_nchw_f32_batched", "yb200_conv1x1_nchw_f32"
QUERIES = ("yb200_conv2d_wgrad_workspace", "yb200_colsum_workspace")  # workspace sizes: nothing to replay
# every entry point a decoder forward calls (over the maps of MAPS: the per-image mask GEMM runs only where the batched one is refused)
ENTRY_POINTS = {"yb200_pack_conv_weight", "yb200_conv2d_relu_fwd", "yb200_conv2d_affine_fwd", "yb200_sigmoid", "yb200_conv2d_wgrad_workspace",
                "yb200_conv2d_wgrad", "yb200_colsum_workspace", "yb200_colsum", "yb200_iam_normalize", "yb200_conv1x1_bias_f32", BATCHED, PER_IMAGE,
                "yb200_upsample_bilinear2x_f32"}
MAPS = {"Base": [(2, 80, 80), (2, 64, 64), (2, 40, 40), (1, 13, 17)], "Group": [(2, 64, 64), (2, 40, 40)]}
STAGE = {"yb200_sigmoid": "inst_branch iam", "yb200_conv2d_wgrad": "inst_branch iam_prob^T features", "yb200_colsum": "inst_branch iam normaliser",
         "yb200_iam_normalize": "inst_branch inst features", BATCHED: "pred_kernel x mask features", PER_IMAGE: "pred_kernel x mask features",
         "yb200_upsample_bilinear2x_f32": "pred_masks"}


class _Recorder:
    """stands in for a decoder's library handle: records every call (entry point, arguments, return code) and forwards it, except that the
    entry points in `refuse` return ERR_UNSUPPORTED without running"""

    def __init__(self, lib, refuse=()):
        self._lib, self.refuse, self.log = lib, set(refuse), []

    def __getattr__(self, name):
        fn = getattr(self._lib, name)
        if not name.startswith("yb200_") or name == "yb200_last_error":
            return fn

        def rec(*a):
            from yolov7_d2_b200 import capi

            rc = capi.ERR_UNSUPPORTED if name in self.refuse else fn(*a)
            self.log.append((name, a, rc))
            return rc
        return rec


def _v(a):
    return a.value if isinstance(a, (ctypes.c_void_p, ctypes.c_float, ctypes.c_int64)) else a


def _case_of(name, a):
    """replay case of one recorded call (None for the workspace queries)"""
    if name == "yb200_pack_conv_weight":
        return dict(fn="pack", cout=a[1], cin=a[2], k=a[3], cout_pad=a[4], cin_pad=a[5])
    if name == "yb200_conv2d_relu_fwd":
        return dict(fn="relu", gx=_geo(a[0]), go=_geo(a[3]), k=a[4], s=a[5])
    if name == "yb200_conv2d_affine_fwd":
        return dict(fn="affine", gx=_geo(a[0]), go=_geo(a[5]), gr=_geo(a[4]), k=a[6], s=a[7], with_scale=_given(a[2]), with_shift=_given(a[3]))
    if name == "yb200_sigmoid":
        return dict(fn="sigmoid", gx=_geo(a[0]), go=_geo(a[1]))
    if name == "yb200_conv2d_wgrad":
        return dict(fn="wgrad", gx=_geo(a[0]), gdz=_geo(a[1]), k=a[2], s=a[3], cin_real=a[4], accumulate=a[6])
    if name == "yb200_colsum":
        return dict(fn="colsum", gx=_geo(a[0]), scale=_v(a[1]), accumulate=a[3])
    if name == "yb200_iam_normalize":
        return dict(fn="normalize", rows=a[2], cols=a[3], go=_geo(a[4]))
    if name == "yb200_conv1x1_bias_f32":
        return dict(fn="pred", gx=_geo(a[0]), cout=a[3], a_total=a[5], a_off=a[6], c_total=a[7], c_off=a[8])
    if name == BATCHED:
        return dict(fn="nchw", gx=_geo(a[0]), cout=a[2], batched=True)
    if name == PER_IMAGE:
        return dict(fn="nchw", gx=_geo(a[0]), cout=a[3], batched=False, bias=_given(a[2]))
    if name == "yb200_upsample_bilinear2x_f32":
        return dict(fn="upsample", planes=_v(a[2]), h=a[3], w=a[4])
    if name in QUERIES:
        return None
    raise AssertionError(f"{name}: a decoder call this module does not replay")


def _view(g):
    return str(g[3]) if g[4] == g[3] and g[5] == 0 else f"{g[3]}@{g[5]}/{g[4]}"


def _map(g):
    return "x".join(map(str, g[:3]))


def _describe(c):
    fn = c["fn"]
    if fn == "pack":
        return f"{c['cout']}x{c['cin']}x{c['k']}x{c['k']} -> [{c['cout_pad']}][{c['k'] ** 2}][{c['cin_pad']}]"
    if fn in ("relu", "affine"):
        return f"{c['k']}x{c['k']} {_view(c['gx'])}->{_view(c['go'])} {_map(c['gx'])}"
    if fn == "sigmoid":
        return f"{_view(c['gx'])} {_map(c['gx'])}"
    if fn == "wgrad":
        return f"{_view(c['gdz'])}^T {_view(c['gx'])} over {c['gx'][1] * c['gx'][2]} pixels"
    if fn == "colsum":
        return f"{_view(c['gx'])} over {c['gx'][0] * c['gx'][1] * c['gx'][2]} pixels"
    if fn == "normalize":
        return f"[{c['rows']}][{c['cols']}]"
    if fn == "pred":
        return f"{_view(c['gx'])}->{c['cout']} rows {c['a_total']}"
    if fn == "nchw":
        return f"{_view(c['gx'])}->{c['cout']} {_map(c['gx'])}"
    return f"{c['planes']}x{c['h']}x{c['w']}"


def _weight_labels(dec):
    """(first byte, end, name) of every weight parameter"""
    return [(p.data_ptr(), p.data_ptr() + 4 * p.numel(), n[:-len(".weight")], p[0].numel()) for n, p in dec.named_parameters() if n.endswith(".weight")]


def _label(ranges, src, rows):
    for lo, hi, name, row_numel in ranges:
        if lo <= src < hi:
            r0 = (src - lo) // (4 * row_numel)
            return name if src == lo and rows * row_numel * 4 == hi - lo else f"{name} rows {r0}:{r0 + rows}"
    return "?"


def _cases_of(dec, log):
    """[(stage name, entry point, case)] of one recorded forward, in call order"""
    ranges, packed, out = _weight_labels(dec), {}, []
    for name, a, _ in log:
        case = _case_of(name, a)
        if case is None:
            continue
        if name == "yb200_pack_conv_weight":
            stage = _label(ranges, _v(a[0]), a[1])
            packed[_v(a[6])] = stage
        elif name in ("yb200_conv2d_relu_fwd", "yb200_conv2d_affine_fwd", "yb200_conv1x1_bias_f32"):
            stage = packed.get(_v(a[1]), "?")
            if name == "yb200_conv1x1_bias_f32":  # the head's output: the mask kernels are packed from it
                ranges.append((_v(a[4]), _v(a[4]) + 4 * a[0]._obj.n * a[5] * a[7], stage + " output", a[7]))
        else:
            stage = STAGE[name]
        out.append((stage, name, case))
    return out


def _decoder(kind, seed=None):
    from test_sparseinst_gpu import _cfg
    from yolov7_d2_b200.sparseinst import BaseIAMDecoder, GroupIAMDecoder

    from oracle import sparseinst_oracle as sio

    cfg = _cfg(256, 100, 128, 80, 4, 256)
    if kind == "Group":
        cfg.MODEL.SPARSE_INST.DECODER.GROUPS = 4
    dec = (GroupIAMDecoder if kind == "Group" else BaseIAMDecoder)(cfg)
    sd = None
    if seed is not None:
        sd = sio.decoder_state_dict(seed, groups=4 if kind == "Group" else 0)
        dec.load_state_dict({k: v.cuda() for k, v in sd.items()}, strict=True)
    return dec, sd


def _forward(dec, feat, refuse=()):
    rec = _Recorder(dec.L, refuse)
    dec.L = rec
    try:
        out = dec(feat)
        torch.cuda.synchronize()
    finally:
        dec.L = rec._lib
    return out, rec.log


RECORDINGS = {}


def _recordings():
    """{decoder: [(map, log, cases)]}: one forward per map, recorded when the module is collected on a machine with a GPU"""
    if not RECORDINGS and torch.cuda.is_available():
        for kind, maps in MAPS.items():
            dec, _ = _decoder(kind)
            RECORDINGS[kind] = []
            for i, (n, h, w) in enumerate(maps):
                feat = torch.randn(n, 256, h, w, generator=_g(30 + i), device="cuda")
                _, log = _forward(dec, feat)
                RECORDINGS[kind].append(((n, h, w), log, _cases_of(dec, log)))
            del dec
        torch.cuda.empty_cache()
    return RECORDINGS


def _distinct(kind):
    """[(test id, case)]: each distinct geometry of the decoder once, named after the first stage that called it"""
    seen, out = {}, []
    for _, _, cases in _recordings().get(kind, []):
        for stage, name, case in cases:
            key = tuple(sorted(case.items()))
            if key in seen:
                seen[key][1] += 1
                continue
            seen[key] = [len(out), 1]
            out.append([f"{kind}: {stage} {name[len('yb200_'):]} {_describe(case)}", case])
    for i, n in seen.values():
        if n > 1:
            out[i][0] += f" (+{n - 1} more)"
    return [tuple(x) for x in out]


def pytest_generate_tests(metafunc):
    if "dec_case" in metafunc.fixturenames:
        cases = [c for kind in MAPS for c in _distinct(kind)]
        metafunc.parametrize("dec_case", [c[1] for c in cases], ids=[c[0] for c in cases])


def test_decoder_call(cuda, dec_case):
    case = dict(dec_case)
    RUN[case.pop("fn")](**case)


def test_recording_is_complete(cuda):
    """every entry point the decoders call is one this module replays, and the shipped geometries are among the cases"""
    recs = _recordings()
    for kind in MAPS:
        names = {name for _, log, _ in recs[kind] for name, _, _ in log}
        assert names == ENTRY_POINTS, f"{kind}: entry points called {sorted(names)}, replayed {sorted(ENTRY_POINTS)}"
        cases = [c for _, c in _distinct(kind)]
        # the first 3x3 layer at the largest map: 256 features + 2 coordinates padded to 272 channels (BLOCK_K 16, 17 k-blocks per tap)
        assert any(c["fn"] == "relu" and c["k"] == 3 and c["gx"] == MAPS[kind][0] + (272, 272, 0) for c in cases), "no 272-channel 3x3 layer"
        assert any(c["fn"] == "pred" and c["cout"] == 1 for c in cases), "no 1-wide head"
        assert any(c["fn"] == "nchw" and c["batched"] for c in cases) and any(c["fn"] == "nchw" and not c["batched"] for c in cases)
    group = [c for _, c in _distinct("Group")]
    # the grouped IAM convolution: 104-wide output views at 0 / 104 / 208 / 312 of a 416 pitch, 64-wide input views of a 256 pitch
    offs = {c["go"][5] for c in group if c["fn"] == "affine" and c["go"][3:5] == (104, 416)}
    assert offs == {0, 104, 208, 312}, offs
    assert any(c["fn"] == "relu" and c["k"] == 1 and c["gx"][3] == 1024 for c in group), "no 1x1 fc over 1024 channels"
    assert any(c["fn"] == "wgrad" and c["gdz"][3] == 416 for c in group), "no 416-row pixel contraction"


def test_recorded_mask_gemm_routing(cuda):
    """the decoders call the batched mask GEMM first; it runs where each 128-pixel tile holds one image, else every image has its own call"""
    from yolov7_d2_b200 import capi

    for kind, recs in _recordings().items():
        for (n, h, w), log, _ in recs:
            rcs = [rc for name, _, rc in log if name == BATCHED]
            per = sum(name == PER_IMAGE for name, _, _ in log)
            if batched_accepts(n, h, w):
                assert rcs == [0] and per == 0, (kind, (n, h, w), rcs, per)
            else:
                assert rcs == [capi.ERR_UNSUPPORTED] and per == n, (kind, (n, h, w), rcs, per)


# ------------------------------------------------------------------------------------------------------------------------------------
# B. the batched mask GEMM on its own
# ------------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cout", [112, 128])
@pytest.mark.parametrize("nhw", BATCHED_ACCEPTED + BATCHED_REFUSED, ids=lambda s: "x".join(map(str, s)))
def test_batched_mask_gemm(cuda, nhw, cout):
    capi, L = _lib()
    n, h, w = nhw
    c = 128
    g = _g(40)
    x = (torch.randn(n, h, w, c, generator=g, device="cuda")).to(torch.bfloat16)
    wimg = _img_weights(n, cout, c, g)
    if not batched_accepts(n, h, w):
        _refused(capi, L, x, wimg, cout, g)
        return
    buf, out = _guarded((n, cout, h, w), float("nan"))
    capi.check(_nchw_call(capi, L, x, wimg, cout, out, True), "conv1x1_nchw_f32_batched")
    ref, mag, kk = bmm_ref(x.double(), wimg.double())
    check("mask GEMM (fp32)", out, ref, bound(ref, mag, kk, 0.0), f"masks {n}x{h}x{w} cout {cout}")
    _guard_ok(buf, out.numel(), "masks")
    # an image's masks do not depend on where it sits in the batch
    perm = torch.arange(n - 1, -1, -1, device="cuda")
    outp = torch.full_like(out, float("nan"))
    capi.check(_nchw_call(capi, L, x[perm].contiguous(), wimg[perm].contiguous(), cout, outp, True), "conv1x1_nchw_f32_batched")
    assert torch.equal(outp, out[perm]), "reordering the images changes their masks"
    # the same tile, BLOCK_N / BLOCK_K and k order as the per-image call: the same bits
    for i in range(n):
        oi = torch.full((1, cout, h, w), float("nan"), device="cuda")
        capi.check(_nchw_call(capi, L, x[i:i + 1], wimg[i], cout, oi, False), "conv1x1_nchw_f32")
        assert torch.equal(oi[0], out[i]), f"image {i}: the batched masks differ from the per-image call's"


# ------------------------------------------------------------------------------------------------------------------------------------
# C. the decoders on the batched path
# ------------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,nhw", [("Base", (2, 80, 80)), ("Group", (2, 64, 64))], ids=["Base-2x80x80", "Group-2x64x64"])
def test_decoder_batched_path_against_oracle(cuda, kind, nhw):
    from test_sparseinst_gpu import _check

    from oracle import sparseinst_oracle as sio

    n, h, w = nhw
    dec, sd = _decoder(kind, seed=13)
    feat = torch.randn(n, 256, h, w, generator=torch.Generator().manual_seed(14))
    out, log = _forward(dec, feat.to(cuda))
    assert [rc for name, _, rc in log if name == BATCHED] == [0], "the batched mask GEMM did not run"
    assert not any(name == PER_IMAGE for name, _, _ in log), "the per-image mask GEMM ran"
    ref = sio.decoder_forward(feat, sd, groups=4 if kind == "Group" else 0)
    _check(out["pred_logits"], ref["pred_logits"], "class logits")
    _check(out["pred_scores"], ref["pred_scores"], "objectness")
    if "masks_lowres" in ref:
        _check(dec.last["masks_lowres"], ref["masks_lowres"], "masks before up-sampling")
    _check(out["pred_masks"], ref["pred_masks"], "masks")


@pytest.mark.parametrize("kind", ["Base", "Group"])
def test_decoder_fallback_is_bit_identical(cuda, kind):
    """2x64x64: two identical forwards give the same bits, and so does the per-image fallback (the batched call refused by the stand-in)"""
    dec, _ = _decoder(kind, seed=15)
    feat = torch.randn(2, 256, 64, 64, generator=_g(16), device="cuda")
    runs = [_forward(dec, feat)[0] for _ in range(2)]
    fb, log = _forward(dec, feat, refuse={BATCHED})
    assert sum(name == PER_IMAGE for name, _, _ in log) == 2, "the fallback did not run per image"
    for key in runs[0]:
        assert torch.equal(runs[0][key], runs[1][key]), f"{key}: two identical forwards differ"
        assert torch.equal(runs[0][key], fb[key]), f"{key}: the per-image fallback differs from the batched mask GEMM"


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    saved = dict(WORST)
    WORST.clear()
    yield
    if WORST:
        print("\nworst |err| / bound per case class: " + "; ".join(f"{k}: {v:.3g}" for k, v in sorted(WORST.items())))
    for k, v in saved.items():
        WORST[k] = max(WORST.get(k, 0.0), v)
