"""GPU parity of the wgmma implicit-GEMM convolution family (forward, dgrad, wgrad) through the C ABI.

Reference: torch fp32 convolution (TF32 off) on the same bf16-rounded inputs -- the arithmetic the reference's
BaseConv.conv performs (yolov7/modeling/backbone/layers/wrappers.py:67-80) and its autograd.
Tolerances: outputs are stored in bf16 (rel 2^-8); accumulation is fp32 in both paths.
"""
import ctypes

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

# (N, H, W, Cin, Cout, k, stride)  -- every distinct YOLOX-s shape class (SURVEY.md appendix B) at small N,
# plus ragged sizes that exercise partial tiles.
SHAPES = [
    (8, 32, 32, 16, 32, 3, 1),     # stem-like (Focus, cin padded 12->16)
    (8, 32, 32, 32, 64, 3, 2),     # dark2.0
    (8, 16, 16, 64, 32, 1, 1),
    (8, 16, 16, 32, 32, 3, 1),
    (8, 16, 16, 64, 64, 1, 1),
    (4, 40, 40, 64, 128, 3, 2),    # dark3.0
    (8, 20, 20, 128, 64, 1, 1),
    (8, 20, 20, 64, 64, 3, 1),
    (8, 20, 20, 128, 128, 3, 1),   # head convs
    (8, 20, 20, 128, 256, 3, 2),   # dark4.0
    (8, 10, 10, 256, 512, 3, 2),   # dark5.0
    (8, 20, 20, 1024, 512, 1, 1),  # SPP conv2
    (8, 20, 20, 256, 256, 3, 1),
    (8, 20, 20, 512, 128, 1, 1),
    (3, 24, 36, 64, 64, 3, 1),     # ragged: partial tiles in w, h and n
    (5, 12, 20, 128, 128, 3, 2),   # ragged stride 2
    (2, 80, 80, 128, 128, 3, 1),   # 80x80 head level
    (1, 320, 320, 16, 32, 3, 1),   # full-size stem row tiles
    (1, 32, 32, 16, 32, 3, 1),     # single image
    (16, 64, 64, 16, 32, 3, 1),    # 512 CTAs: several CTAs resident per SM, more than one wave
    (16, 64, 64, 64, 64, 1, 1),    # 512 single-k-block CTAs (memory-bound 1x1)
    (8, 80, 80, 128, 128, 3, 1),   # 400 CTAs x 18 k-blocks
    (8, 80, 80, 128, 80, 1, 1),    # prediction convolutions: cls (80 channels) at the stride-8 level ...
    (8, 20, 20, 128, 80, 1, 1),    # ... and the stride-32 level
    (8, 40, 40, 128, 16, 1, 1),    # reg + obj, 5 channels padded to 16: 16-channel block of the data gradient
]


def _mk(shape, dev, seed):
    n, h, w, cin, cout, k, s = shape
    g = torch.Generator(device="cpu").manual_seed(seed)
    x = torch.randn(n, h, w, cin, generator=g).to(dev).to(torch.bfloat16)
    wt = (torch.randn(cout, cin, k, k, generator=g) / (cin * k * k) ** 0.5).to(dev)
    wt = wt.to(torch.bfloat16).float()  # weights as the kernel sees them
    return x, wt


def _pack(capi, wt, cout_pad, cin_pad, dgrad=True):
    cout, cin, k, _ = wt.shape
    wf = torch.empty(cout_pad, k * k, cin_pad, dtype=torch.bfloat16, device=wt.device)
    wd = torch.empty(cin_pad, k * k, cout_pad, dtype=torch.bfloat16, device=wt.device) if dgrad else None
    capi.check(capi.lib().yb200_pack_conv_weight(capi.ptr(wt), cout, cin, k, cout_pad, cin_pad, capi.ptr(wf), capi.ptr(wd),
                                                 capi.stream_ptr()), "pack")
    return wf, wd


def _close(got, ref, rel, what):
    err = (got.float() - ref.float()).abs()
    tol = rel * ref.float().abs() + rel * ref.float().abs().max()
    bad = (err > tol).sum().item()
    assert bad == 0, f"{what}: {bad}/{err.numel()} outside tol; max err {err.max().item():.4g} ref max {ref.abs().max().item():.4g}"


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_conv_fwd_stats(cuda, shape):
    from yolov7_d2_b200 import capi

    n, h, w, cin, cout, k, s = shape
    x, wt = _mk(shape, cuda, 1)
    wf, _ = _pack(capi, wt, cout, cin, dgrad=False)
    z = torch.full((n, h // s, w // s, cout), float("nan"), dtype=torch.float16, device=cuda)  # pre-BN output is fp16
    ssum = torch.zeros(cout, dtype=torch.float64, device=cuda)
    ssq = torch.zeros(cout, dtype=torch.float64, device=cuda)
    xa, za = capi.act(x), capi.act(z)
    capi.check(capi.lib().yb200_conv2d_fwd(ctypes.byref(xa), capi.ptr(wf), ctypes.byref(za), k, s, capi.ptr(ssum), capi.ptr(ssq),
                                           capi.stream_ptr()), "conv2d_fwd")
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), wt, stride=s, padding=(k - 1) // 2).permute(0, 2, 3, 1)
    _close(z, ref, 2.0 ** -10, "z")
    zf = z.double()
    assert torch.allclose(ssum, zf.sum((0, 1, 2)), rtol=1e-5, atol=1e-3), "sum"
    assert torch.allclose(ssq, (zf * zf).sum((0, 1, 2)), rtol=1e-5, atol=1e-3), "sumsq"


def test_conv_fwd_channel_slices(cuda):
    """input and output are channel slices of wider (concat) buffers"""
    from yolov7_d2_b200 import capi

    n, h, w, cin, cout = 4, 20, 20, 64, 64
    g = torch.Generator().manual_seed(3)
    xb = torch.randn(n, h, w, 192, generator=g).to(cuda).to(torch.bfloat16)
    wt = (torch.randn(cout, cin, 3, 3, generator=g) / 24).to(cuda).to(torch.bfloat16).float()
    wf, _ = _pack(capi, wt, cout, cin, dgrad=False)
    zb = torch.zeros(n, h, w, 128, dtype=torch.float16, device=cuda)
    xa, za = capi.act(xb, 64, 64), capi.act(zb, 64, 64)
    capi.check(capi.lib().yb200_conv2d_fwd(ctypes.byref(xa), capi.ptr(wf), ctypes.byref(za), 3, 1, None, None, capi.stream_ptr()), "fwd")
    ref = F.conv2d(xb[..., 64:128].float().permute(0, 3, 1, 2), wt, padding=1).permute(0, 2, 3, 1)
    _close(zb[..., 64:], ref, 2.0 ** -10, "slice out")
    assert (zb[..., :64] == 0).all(), "neighbouring channels were overwritten"


@pytest.mark.parametrize("cout", [80, 5])
def test_conv1x1_bias_f32(cuda, cout):
    from yolov7_d2_b200 import capi

    n, h, w, cin = 4, 20, 20, 128
    g = torch.Generator().manual_seed(4)
    x = torch.randn(n, h, w, cin, generator=g).to(cuda).to(torch.bfloat16)
    wt = (torch.randn(cout, cin, 1, 1, generator=g) / 11).to(cuda).to(torch.bfloat16).float()
    bias = torch.randn(cout, generator=g).to(cuda)
    wf, _ = _pack(capi, wt, cout, cin, dgrad=False)
    a_total, a_off, c_total, c_off = 500, 100, 85, (5 if cout == 80 else 0)
    out = torch.zeros(n, a_total, c_total, device=cuda)
    xa = capi.act(x)
    capi.check(capi.lib().yb200_conv1x1_bias_f32(ctypes.byref(xa), capi.ptr(wf), capi.ptr(bias), cout, capi.ptr(out), a_total, a_off,
                                                 c_total, c_off, capi.stream_ptr()), "conv1x1_bias_f32")
    ref = (F.conv2d(x.float().permute(0, 3, 1, 2), wt) + bias.view(1, -1, 1, 1)).permute(0, 2, 3, 1).reshape(n, h * w, cout)
    got = out[:, a_off:a_off + h * w, c_off:c_off + cout]
    assert torch.allclose(got, ref, rtol=1e-4, atol=1e-4), (got - ref).abs().max().item()
    out[:, a_off:a_off + h * w, c_off:c_off + cout] = 0
    assert (out == 0).all(), "wrote outside the slice"


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("with_addend", [False, True])
def test_conv_dgrad(cuda, shape, with_addend):
    from yolov7_d2_b200 import capi

    n, h, w, cin, cout, k, s = shape
    _, wt = _mk(shape, cuda, 5)
    _, wd = _pack(capi, wt, cout, cin)
    g = torch.Generator().manual_seed(6)
    dz = torch.randn(n, h // s, w // s, cout, generator=g).to(cuda).to(torch.bfloat16)
    add = torch.randn(n, h, w, cin, generator=g).to(cuda).to(torch.bfloat16) if with_addend else None
    dx = torch.full((n, h, w, cin), float("nan"), dtype=torch.bfloat16, device=cuda)
    dza, dxa = capi.act(dz), capi.act(dx)
    adda = capi.act(add) if with_addend else None
    capi.check(capi.lib().yb200_conv2d_dgrad(ctypes.byref(dza), capi.ptr(wd), ctypes.byref(dxa),
                                             ctypes.byref(adda) if with_addend else None, k, s, capi.stream_ptr()), "dgrad")
    ref = torch.nn.grad.conv2d_input((n, cin, h, w), wt, dz.float().permute(0, 3, 1, 2), stride=s, padding=(k - 1) // 2)
    ref = ref.permute(0, 2, 3, 1)
    if with_addend:
        ref = ref + add.float()
    _close(dx, ref, 2.0 ** -7, "dx")


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_conv_wgrad(cuda, shape):
    from yolov7_d2_b200 import capi

    n, h, w, cin, cout, k, s = shape
    x, wt = _mk(shape, cuda, 7)
    g = torch.Generator().manual_seed(8)
    dz = torch.randn(n, h // s, w // s, cout, generator=g).to(cuda).to(torch.bfloat16)
    cin_real = 12 if cin == 16 else cin
    xa, dza = capi.act(x), capi.act(dz)
    ws_bytes = capi.lib().yb200_conv2d_wgrad_workspace(ctypes.byref(xa), ctypes.byref(dza), k, s)
    assert ws_bytes > 0, capi.lib().yb200_last_error()
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=cuda)
    grad = torch.full((cout, cin_real, k, k), float("nan"), device=cuda)
    capi.check(capi.lib().yb200_conv2d_wgrad(ctypes.byref(xa), ctypes.byref(dza), k, s, cin_real, capi.ptr(grad), 0, capi.ptr(ws),
                                             ctypes.c_int64(ws_bytes), capi.stream_ptr()), "wgrad")
    ref = torch.nn.grad.conv2d_weight(x.float().permute(0, 3, 1, 2), (cout, cin, k, k), dz.float().permute(0, 3, 1, 2), stride=s,
                                      padding=(k - 1) // 2)[:, :cin_real]
    err = (grad - ref).abs().max().item()
    assert err <= 2e-4 * ref.abs().max().item() + 1e-5, f"wgrad max err {err} vs ref max {ref.abs().max().item()}"
    # accumulate mode adds on top
    capi.check(capi.lib().yb200_conv2d_wgrad(ctypes.byref(xa), ctypes.byref(dza), k, s, cin_real, capi.ptr(grad), 1, capi.ptr(ws),
                                             ctypes.c_int64(ws_bytes), capi.stream_ptr()), "wgrad acc")
    err2 = (grad - 2 * ref).abs().max().item()
    assert err2 <= 4e-4 * ref.abs().max().item() + 2e-5, f"wgrad accumulate max err {err2}"


@pytest.mark.parametrize("shape", [(4, 20, 20, 64, 64, 3, 1), (4, 20, 20, 128, 256, 3, 2), (3, 24, 36, 64, 64, 1, 1), (8, 20, 20, 256, 512, 1, 1)],
                         ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("with_res", [False, True])
def test_conv_bn_silu_eval_fused(cuda, shape, with_res):
    """eval-mode BaseConv in one kernel: conv + folded BatchNorm + SiLU (+ Bottleneck shortcut) -- wrappers.py:60-83, 119-123"""
    from yolov7_d2_b200 import capi

    n, h, w, cin, cout, k, s = shape
    x, wt = _mk(shape, cuda, 21)
    wf, _ = _pack(capi, wt, cout, cin, dgrad=False)
    g = torch.Generator().manual_seed(22)
    scale = (torch.rand(cout, generator=g) + 0.5).to(cuda)
    shift = (torch.randn(cout, generator=g) * 0.3).to(cuda)
    res = torch.randn(n, h // s, w // s, cout, generator=g).to(cuda).to(torch.bfloat16) if with_res else None
    out = torch.full((n, h // s, w // s, cout), float("nan"), dtype=torch.bfloat16, device=cuda)
    xa, oa = capi.act(x), capi.act(out)
    ra = capi.act(res) if with_res else None
    capi.check(capi.lib().yb200_conv2d_bn_silu_fwd(ctypes.byref(xa), capi.ptr(wf), capi.ptr(scale), capi.ptr(shift),
                                                   ctypes.byref(ra) if with_res else None, ctypes.byref(oa), k, s, capi.stream_ptr()), "fused")
    z = F.conv2d(x.float().permute(0, 3, 1, 2), wt, stride=s, padding=(k - 1) // 2)
    u = z * scale.view(1, -1, 1, 1) + shift.view(1, -1, 1, 1)
    ref = (u * torch.sigmoid(u)).permute(0, 2, 3, 1)
    if with_res:
        ref = ref.to(torch.bfloat16).float() + res.float()
    _close(out, ref, 2.0 ** -7, "fused out")
