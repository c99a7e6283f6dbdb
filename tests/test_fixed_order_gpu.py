"""Kernel parity, against fp64, of the two fixed-order sums of the training step: the SPP backward and the pixel-grouped stem (forward with
folded BatchNorm statistics, weight gradient folded onto the [32, 12, 3, 3] parameter).

The reference is fp64 torch on the same 16-bit operands, so it is exact up to 2^-53.  Every tolerance is derived from the kernel's arithmetic:
one rounding to the stored type (unit roundoff u = 2^-8 for bf16, 2^-11 for fp16, none for fp32 or fp64 results), plus k * 2^-24 * sum|terms|
for an fp32 accumulation whose additions each round by at most one ulp of a partial sum, where k counts those additions on the longest path and
the fp64 reference computes sum|terms|.  Tensor-core (wgmma) accumulation may truncate rather than round to nearest: a full ulp, 2^-23, so its
k counts every addition twice.
"""
import ctypes

import pytest
import torch
import torch.nn.functional as F

from oracle import yolox_oracle as orc

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24   # fp32 unit roundoff
U_BF16 = 2.0 ** -8
U_F16 = 2.0 ** -11


def nhwc(t):
    return t.permute(0, 2, 3, 1).contiguous()


def nchw(t):
    return t.permute(0, 3, 1, 2).contiguous()


# ------------------------------------------------------------------------------------------------------------------------ SPP backward

def _spp_input(n, c, h, w, ties, g):
    x = torch.randn(n, c, h, w, generator=g)
    if ties:  # values on a 1/2 grid: every window holds several equal maxima (first maximum in row-major order wins, as in ATen)
        x = torch.round(x * 2) / 2
        x[0, : min(c, 8)] = 0.0
        x[0, : min(c, 4), ::2] = -0.0
    return x.to(torch.bfloat16)


SPP_SHAPES = [
    (4, 256, 20, 20),   # YOLOX-s at 640x640 (dark5)
    (2, 32, 25, 25),    # the largest multi-scale input, 800x800
    (2, 32, 15, 25),    # non-square
    (2, 16, 1, 1),      # maps smaller than every window: windows clipped on all sides
    (2, 16, 3, 5),
    (3, 16, 7, 7),
    (2, 8, 20, 20),     # c % 16 != 0: scatter fallback
    (2, 24, 13, 13),    # c % 16 != 0: scatter fallback
    (2, 16, 44, 44),    # 44*44*16*7 B > 200 KiB of shared memory: scatter fallback
]


@pytest.mark.parametrize("ties", [False, True], ids=["random", "many_ties"])
@pytest.mark.parametrize("shape", SPP_SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_spp_pool_bwd_against_fp64(cuda, shape, ties):
    check_spp_pool(cuda, shape, ties)


def check_spp_pool(cuda, shape, ties):
    """yb200_spp_pool (maxima and argmax bytes) and yb200_spp_pool_bwd on an [n, c, h, w] map, against fp64 max pooling and its autograd"""
    from yolov7_d2_b200 import capi

    L = capi.lib()
    n, c, h, w = shape
    g = torch.Generator().manual_seed(n * c + 100 * h + w + ties)
    x = _spp_input(n, c, h, w, ties, g)
    cat = torch.zeros(n, h, w, 4 * c, dtype=torch.bfloat16, device=cuda)
    cat[..., :c] = nhwc(x).to(cuda)
    arg = torch.empty(3, n, h, w, c, dtype=torch.uint8, device=cuda)
    v = [capi.act(cat, i * c, c) for i in range(4)]
    capi.check(L.yb200_spp_pool(ctypes.byref(v[0]), ctypes.byref(v[1]), ctypes.byref(v[2]), ctypes.byref(v[3]), capi.ptr(arg), capi.stream_ptr()),
               "spp_pool")
    xd = x.double().requires_grad_(True)
    ref = torch.cat([xd] + [F.max_pool2d(xd, k, 1, k // 2) for k in (5, 9, 13)], 1)
    assert torch.equal(cat.cpu().double(), nhwc(ref.detach())), "pooled maxima"
    dcat = torch.randn(n, 4 * c, h, w, generator=g).to(torch.bfloat16)
    dcd = nhwc(dcat).to(cuda)
    dv = [capi.act(dcd, i * c, c) for i in range(4)]
    dx = torch.empty(n, h, w, c, dtype=torch.bfloat16, device=cuda)
    scratch = torch.empty(n * h * w * c, dtype=torch.float32, device=cuda)
    capi.check(L.yb200_spp_pool_bwd(ctypes.byref(dv[0]), ctypes.byref(dv[1]), ctypes.byref(dv[2]), ctypes.byref(dv[3]), capi.ptr(arg), capi.ptr(scratch),
                                    ctypes.byref(capi.act(dx)), capi.stream_ptr()), "spp_pool_bwd")
    # fp64 routing of the same bf16 gradients: the sum, the sum of magnitudes and the number of terms that land on each input
    sums = []
    for d in (dcat.double(), dcat.double().abs(), torch.ones_like(dcat, dtype=torch.float64)):
        (gx,) = torch.autograd.grad(ref, xd, d, retain_graph=True)
        sums.append(nhwc(gx))
    r, sabs, cnt = sums
    # fp32 sum of cnt terms (cnt - 1 additions, shared-memory adds or atomics), then one bf16 rounding:
    # |dx - r| <= u_bf16 |r| + (1 + u_bf16) (cnt - 1) 2^-24 sum|terms|
    tol = U_BF16 * r.abs() + (1 + U_BF16) * (cnt - 1) * U32 * sabs
    err = (dx.cpu().double() - r).abs()
    bad = err > tol
    assert not bad.any(), f"{int(bad.sum())} of {bad.numel()} gradients off, worst {float((err - tol).max()):.3g} beyond the bound"


# ------------------------------------------------------------------------------------------------------------------ pixel-grouped stem

@pytest.fixture(scope="module")
def stem(cuda):
    """a small plan with the engine's real stem expansion (w_exp from the parameter, packed to bf16 w_fwd)"""
    from yolov7_d2_b200.engine import YoloxEngine

    eng = YoloxEngine(2, 128, 128, device=cuda)
    assert eng.group4, "the pixel-grouped stem is off"
    eng.load_state_dict(orc.yolox_state_dict(12))
    eng.pack_weights()
    torch.cuda.synchronize()
    op = eng.ops[0]
    assert op.first and tuple(op.w_src.shape) == (32, 12, 3, 3)
    return eng, op


def _choose_tile(n, h, w, npix=128):
    """number of npix-pixel tiles the convolution kernels cover an [n, h, w] grid with (csrc/host_common.cu choose_tile)"""
    lp, best = npix.bit_length() - 1, None
    for lw in range(lp, -1, -1):
        for lh in range(lp - lw, -1, -1):
            tw, th, tn = 1 << lw, 1 << lh, npix >> (lw + lh)
            tiles = -(-w // tw) * -(-h // th) * -(-n // tn)
            if best is None or tiles * npix < best[0]:
                best = (tiles * npix, tiles)
    return best[1]


def _stem_input(n, h, w, g, cuda):
    """Focus output: 12 real channels, 4 zero padding channels (what yb200_preprocess_focus writes)"""
    x = torch.zeros(n, h, w, 16, dtype=torch.bfloat16)
    x[..., :12] = torch.randn(n, h, w, 12, generator=g).to(torch.bfloat16)
    return x.to(cuda)


@pytest.mark.parametrize("n,h,w", [(2, 128, 128), (1, 320, 320), (3, 77, 96)], ids=["128x128", "320x320", "ragged_77x96"])
def test_stem_fwd_fold_against_fp64(stem, cuda, n, h, w):
    """z = conv3x3(x, W) stored in fp16, and the per-channel sum / sum of squares of the stored z, folded from the 4 x 32 grouped columns onto
    the 32 channels.  Every row's first and last pixel (image borders) and every group's first and last pixel (where the kernel skips the
    side taps the expansion makes zero) are compared like all the others."""
    from yolov7_d2_b200 import capi

    eng, op = stem
    g = torch.Generator().manual_seed(n * 1000 + h + w)
    x = _stem_input(n, h, w, g, cuda)
    z = torch.empty(n, h, w, 32, dtype=torch.float16, device=cuda)
    ssum = torch.zeros(32, dtype=torch.float64, device=cuda)
    ssq = torch.zeros(32, dtype=torch.float64, device=cuda)
    xg, zg = capi.act(x.view(n, h, w // 4, 64)), capi.act(z.view(n, h, w // 4, 128))
    capi.check(eng.L.yb200_conv2d_fwd_fold(ctypes.byref(xg), capi.ptr(op.w_fwd), ctypes.byref(zg), 3, 1, capi.ptr(ssum), capi.ptr(ssq), 32,
                                           capi.stream_ptr()), "conv2d_fwd_fold")
    torch.cuda.synchronize()
    wq = op.w_src.detach().cpu().to(torch.bfloat16).double()   # w_fwd holds the parameter rounded to bf16 (round to nearest)
    xq = nchw(x[..., :12].cpu().double())
    ref = nhwc(F.conv2d(xq, wq, padding=1))
    sabs = nhwc(F.conv2d(xq.abs(), wq.abs(), padding=1))
    # 12 channels x 9 taps = 108 products (exact in fp32) per output, tensor-core accumulation (2 x 108 additions), one fp16 rounding;
    # fp16 results below 2^-14 are subnormal: add half their spacing, 2^-25
    tol = U_F16 * ref.abs() + (1 + U_F16) * 2 * 108 * U32 * sabs + 2.0 ** -25
    zc = z.cpu().double()
    err = (zc - ref).abs()
    bad = err > tol
    if bad.any():
        i = bad.nonzero()[0].tolist()
        pytest.fail(f"{int(bad.sum())} outputs beyond the bound, first at (n, y, x, c) = {i} (x % 4 = {i[2] % 4}), error {float(err[tuple(i)]):.3g} "
                    f"vs {float(tol[tuple(i)]):.3g}")
    # statistics of the stored z: fp32 per warp (32 pixels, 5 butterfly levels), one addition per 128-pixel tile the CTA walks, two levels for
    # the four 32-pixel quadrants; then fp64 atomics across CTAs and the four column groups (2^-53 per addition: negligible here).  Squares
    # round once more.
    k = 5 + _choose_tile(n, h, w // 4) + 2
    rs, rq = zc.sum((0, 1, 2)), (zc * zc).sum((0, 1, 2))
    ss_abs = zc.abs().sum((0, 1, 2))
    es, eq = (ssum.cpu() - rs).abs(), (ssq.cpu() - rq).abs()
    assert (es <= k * U32 * ss_abs).all(), (es / (k * U32 * ss_abs)).max()
    assert (eq <= (k + 1) * U32 * rq).all(), (eq / ((k + 1) * U32 * rq)).max()


@pytest.mark.parametrize("overlap", [False, True], ids=["main_stream", "side_stream"])
def test_stem_wgrad_grouped_fold_against_fp64(stem, cuda, overlap):
    """yb200_conv2d_wgrad_grouped + the engine's fixed-order fold onto the [32, 12, 3, 3] parameter equals dL/dW of the plain 12 -> 32
    convolution; accumulate=1 adds a second copy.  Dropping any one of the four positions of the fold breaks the bound."""
    eng, op = stem
    xb = op.x.buf
    n, h, w = xb.n, xb.h, xb.w
    g = torch.Generator().manual_seed(31 + overlap)
    xb.t.copy_(_stem_input(n, h, w, g, cuda))
    dz = eng._dz_buf(op)
    dz.t.copy_(torch.randn(n, h, w, 32, generator=g).to(torch.bfloat16))
    eng.overlap_wgrad = overlap
    try:
        eng._wgrad_stem_grouped(op, dz.t, 0)
        torch.cuda.synchronize()
        g1 = op.g_dst.detach().clone()
        g_exp = op.g_exp.detach().clone()
        eng._wgrad_stem_grouped(op, dz.t, 1)
        torch.cuda.synchronize()
        g2 = op.g_dst.detach().clone()
    finally:
        eng.overlap_wgrad = True
    xq = nchw(xb.t[..., :12].cpu().double())
    dq = nchw(dz.t.cpu().double())
    ref = torch.nn.grad.conv2d_weight(xq, (32, 12, 3, 3), dq, padding=1)
    sabs = torch.nn.grad.conv2d_weight(xq.abs(), (32, 12, 3, 3), dq.abs(), padding=1)
    # n*h*w products per weight (exact in fp32) split over its four grouped positions, tensor-core and split-K accumulation
    # (2 x n*h*w additions), then the fold's 3 fp32 additions; fp32 result, no further rounding
    tol = 2 * (n * h * w + 3) * U32 * sabs

    def beyond(gq):
        return int(((gq.cpu().double() - ref).abs() > tol).sum())

    assert beyond(g1) == 0, f"{beyond(g1)} of {ref.numel()} weight gradients beyond the bound"
    # the fold adds each weight's four positions in ascending position order
    parts = g_exp.reshape(-1)[op.fold_pos].view(-1, 4)
    assert torch.equal(g1.reshape(-1), ((parts[:, 0] + parts[:, 1]) + parts[:, 2]) + parts[:, 3])
    # accumulate: g1 + (a second g1) -- the bound doubles, plus one fp32 rounding of the sum
    err2 = (g2.cpu().double() - 2 * ref).abs()
    assert (err2 <= 2 * tol + U32 * 2 * ref.abs()).all(), float((err2 - 2 * tol).max())
    # negative check: a fold that loses one of the four positions of every weight must fail the same bound
    for k in range(4):
        kept = parts.clone()
        kept[:, k] = 0
        assert beyond(kept.sum(1).view_as(g1)) > 0, f"the bound cannot tell a fold without position {k}"
