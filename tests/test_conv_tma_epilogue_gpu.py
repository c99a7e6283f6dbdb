"""The convolution GEMM's TMA-store epilogue: every 16-bit output mode of the YOLOX kernels (EPI_F16, EPI_F16_STATS, EPI_BF16 with and without
addend, EPI_BF16_BN_SILU with residual) at every column tile (16 / 32 / 64 / 128) and k-block (16 / 32 / 64), against fp64 torch on the same
16-bit operands, and the layouts its tensor maps must express: channel slices of concat buffers, an addend from another slice, the four
output-parity phases of a stride-2 data gradient, the pixel-grouped stem with stat_fold, and tiles that overhang the pixel grid.

Every output buffer sits inside a larger one filled with a sentinel: each element outside the view's channels and pixels must keep it.
Tolerances follow tests/test_fixed_order_gpu.py: one rounding to the stored type, plus 2 k 2^-24 sum|terms| for a tensor-core fp32 sum of k
products.  The BatchNorm statistics are checked against fp64 sums of the stored fp16 values, within an fp32 bound on the additions of
their reduction (a 5-level butterfly over the 32 rows of a quadrant, one addition per tile of the CTA, two levels over the four quadrants).

The SASS check runs without a GPU: the YOLOX GEMM kernels store with UTMASTG from an STSM-written tile and use no local memory.
"""
import ctypes
import os
import re
import shutil
import subprocess

import pytest
import torch
import torch.nn.functional as F

U32 = 2.0 ** -24
U_BF16 = 2.0 ** -8
U_F16 = 2.0 ** -11
SENTINEL = -12345.0  # exactly representable in fp16 and bf16


def nchw(t):
    return t.permute(0, 3, 1, 2)


def nhwc(t):
    return t.permute(0, 2, 3, 1)


class Guarded:
    """an [n, h, w, pitch] 16-bit buffer in the middle of a sentinel-filled allocation (guard zones before and after it)"""

    def __init__(self, shape, dtype, dev, guard=4096):
        numel = shape[0] * shape[1] * shape[2] * shape[3]
        self.store = torch.full((guard + numel + guard,), SENTINEL, dtype=dtype, device=dev)
        self.guard, self.numel = guard, numel
        self.t = self.store[guard:guard + numel].view(*shape)

    def check(self, c_off, c):
        """everything outside channels [c_off, c_off + c) of the buffer, and both guard zones, still holds the sentinel"""
        s = self.store.cpu()
        assert (s[:self.guard] == SENTINEL).all() and (s[self.guard + self.numel:] == SENTINEL).all(), "wrote outside the buffer"
        t = self.t.cpu()
        outside = torch.cat([t[..., :c_off].reshape(-1), t[..., c_off + c:].reshape(-1)])
        assert (outside == SENTINEL).all(), f"{int((outside != SENTINEL).sum())} elements outside the view were written"
        return self.t[..., c_off:c_off + c]


def _rand16(shape, g, dev, scale=1.0):
    return (torch.randn(*shape, generator=g) * scale).to(torch.bfloat16).to(dev)


def _weights(cout, cin, k, g, dev):
    return (torch.randn(cout, cin, k, k, generator=g) / (cin * k * k) ** 0.5).to(torch.bfloat16).float().to(dev)


def _pack(capi, wt):
    cout, cin, k, _ = wt.shape
    wf = torch.empty(cout, k * k, cin, dtype=torch.bfloat16, device=wt.device)
    wd = torch.empty(cin, k * k, cout, dtype=torch.bfloat16, device=wt.device)
    capi.check(capi.lib().yb200_pack_conv_weight(capi.ptr(wt), cout, cin, k, cout, cin, capi.ptr(wf), capi.ptr(wd), capi.stream_ptr()), "pack")
    return wf, wd


def _fwd_ref(x, wt, k, s):
    """fp64 convolution of the 16-bit operands, and the same over |operands| (the scale of the accumulation error)"""
    xd, wd = nchw(x.double().cpu()), wt.double().cpu()
    ref = nhwc(F.conv2d(xd, wd, stride=s, padding=(k - 1) // 2))
    sabs = nhwc(F.conv2d(xd.abs(), wd.abs(), stride=s, padding=(k - 1) // 2))
    return ref, sabs


def _dgrad_ref(dz, wt, k, s, out_hw):
    dzd, wd = nchw(dz.double().cpu()), wt.double().cpu()
    pad = (k - 1) // 2
    opad = [o - ((i - 1) * s - 2 * pad + k) for o, i in zip(out_hw, dz.shape[1:3])]
    ref = nhwc(F.conv_transpose2d(dzd, wd, stride=s, padding=pad, output_padding=opad))
    sabs = nhwc(F.conv_transpose2d(dzd.abs(), wd.abs(), stride=s, padding=pad, output_padding=opad))
    return ref, sabs


def _assert_within(got, ref, tol, what):
    err = (got.double().cpu() - ref).abs()
    bad = err > tol
    if bad.any():
        i = bad.nonzero()[0].tolist()
        pytest.fail(f"{what}: {int(bad.sum())}/{bad.numel()} beyond the bound, first at {i}: error {float(err[tuple(i)]):.3g} vs "
                    f"{float(tol[tuple(i)]):.3g}")


def _tiles(n, h, w):
    """128-pixel tiles covering an (n, h, w) grid (csrc/host_common.cu choose_tile)"""
    best = None
    for lw in range(7, -1, -1):
        for lh in range(7 - lw, -1, -1):
            tw, th, tn = 1 << lw, 1 << lh, 128 >> (lw + lh)
            t = -(-w // tw) * -(-h // th) * -(-n // tn)
            if best is None or t < best:
                best = t
    return best


def _check_stats(z, ssum, ssq, tiles, fold=None):
    """Σ and Σ² of the stored fp16 values: 5 butterfly levels per 32-row quadrant, one addition per tile over at most all tiles, 2 levels over
    the quadrants (and a column fold in fp64); the squares round once more.  The bound below is a generous multiple of that."""
    zc = z.double().cpu().reshape(-1, z.shape[-1])
    if fold:
        zc = zc.reshape(-1, fold)  # column c lands in column c % fold
    k = 2 * tiles + 6 + 4
    rs, rq = zc.sum(0), (zc * zc).sum(0)
    es, eq = (ssum.cpu() - rs).abs(), (ssq.cpu() - rq).abs()
    assert (es <= k * U32 * zc.abs().sum(0) + 1e-30).all(), f"sum off by {float((es / (k * U32 * zc.abs().sum(0))).max()):.3g} bounds"
    assert (eq <= (k + 1) * U32 * rq + 1e-30).all(), f"sum of squares off by {float((eq / ((k + 1) * U32 * rq)).max()):.3g} bounds"


# ---------------------------------------------------------------------------------------------------------------- forward: z, statistics

def run_fwd(capi, x_act, wf, z_act, k, s, stats, cout, dev, fold=0):
    ssum = torch.zeros(fold or cout, dtype=torch.float64, device=dev) if stats else None
    ssq = torch.zeros(fold or cout, dtype=torch.float64, device=dev) if stats else None
    if fold:
        rc = capi.lib().yb200_conv2d_fwd_fold(ctypes.byref(x_act), capi.ptr(wf), ctypes.byref(z_act), k, s, capi.ptr(ssum), capi.ptr(ssq), fold,
                                              capi.stream_ptr())
    else:
        rc = capi.lib().yb200_conv2d_fwd(ctypes.byref(x_act), capi.ptr(wf), ctypes.byref(z_act), k, s, capi.ptr(ssum), capi.ptr(ssq),
                                         capi.stream_ptr())
    capi.check(rc, "conv2d_fwd")
    torch.cuda.synchronize()
    return ssum, ssq


@pytest.mark.gpu
@pytest.mark.parametrize("stats", [False, True], ids=["f16", "f16_stats"])
@pytest.mark.parametrize("cin", [16, 32, 64], ids=lambda c: f"bk{c}")
@pytest.mark.parametrize("cout", [16, 32, 64, 128], ids=lambda c: f"bn{c}")
def test_fwd_modes(cuda, cout, cin, stats):
    from yolov7_d2_b200 import capi

    n, h, w, k, s = 3, 20, 20, 3, 1  # three 20 x 20 images: tiles overhang the image count
    g = torch.Generator().manual_seed(cout * 7 + cin)
    x = _rand16((n, h, w, cin), g, cuda)
    wt = _weights(cout, cin, k, g, cuda)
    wf, _ = _pack(capi, wt)
    zb = Guarded((n, h, w, cout), torch.float16, cuda)
    ssum, ssq = run_fwd(capi, capi.act(x), wf, capi.act(zb.t), k, s, stats, cout, cuda)
    z = zb.check(0, cout)
    ref, sabs = _fwd_ref(x, wt, k, s)
    _assert_within(z, ref, U_F16 * ref.abs() + (1 + U_F16) * 2 * cin * k * k * U32 * sabs + 2.0 ** -25, "z")
    if stats:
        _check_stats(z, ssum, ssq, _tiles(n, h, w))


@pytest.mark.gpu
@pytest.mark.parametrize("half", [0, 1])
@pytest.mark.parametrize("shape", [(2, 13, 21, 32, 48, 3, 1), (2, 26, 42, 64, 128, 3, 2), (1, 7, 9, 16, 16, 1, 1), (4, 40, 40, 64, 64, 1, 1)],
                         ids=lambda s: "x".join(map(str, s)))
def test_fwd_stats_concat_slice(cuda, shape, half):
    """z is one half of a concat buffer (channel pitch 2 cout) on a grid the tiles overhang in w and h"""
    from yolov7_d2_b200 import capi

    n, h, w, cin, cout, k, s = shape
    g = torch.Generator().manual_seed(sum(shape) + half)
    x = _rand16((n, h, w, cin), g, cuda)
    wt = _weights(cout, cin, k, g, cuda)
    wf, _ = _pack(capi, wt)
    oh, ow = h // s, w // s
    zb = Guarded((n, oh, ow, 2 * cout), torch.float16, cuda)
    ssum, ssq = run_fwd(capi, capi.act(x), wf, capi.act(zb.t, half * cout, cout), k, s, True, cout, cuda)
    z = zb.check(half * cout, cout)
    ref, sabs = _fwd_ref(x, wt, k, s)
    _assert_within(z, ref, U_F16 * ref.abs() + (1 + U_F16) * 2 * cin * k * k * U32 * sabs + 2.0 ** -25, "z")
    _check_stats(z, ssum, ssq, _tiles(n, oh, ow))


@pytest.mark.gpu
def test_fwd_stat_fold(cuda):
    """stat_fold: column c of a 1x1 convolution adds to statistic c % 32"""
    from yolov7_d2_b200 import capi

    n, h, w, cin, cout, fold = 2, 12, 20, 64, 128, 32
    g = torch.Generator().manual_seed(17)
    x = _rand16((n, h, w, cin), g, cuda)
    wt = _weights(cout, cin, 1, g, cuda)
    wf, _ = _pack(capi, wt)
    zb = Guarded((n, h, w, cout), torch.float16, cuda)
    ssum, ssq = run_fwd(capi, capi.act(x), wf, capi.act(zb.t), 1, 1, True, cout, cuda, fold=fold)
    z = zb.check(0, cout)
    ref, sabs = _fwd_ref(x, wt, 1, 1)
    _assert_within(z, ref, U_F16 * ref.abs() + (1 + U_F16) * 2 * cin * U32 * sabs + 2.0 ** -25, "z")
    _check_stats(z, ssum, ssq, 4 * _tiles(n, h, w), fold=fold)


@pytest.mark.gpu
@pytest.mark.parametrize("n,h,w", [(2, 128, 128), (3, 77, 96)], ids=["128x128", "ragged_77x96"])
def test_grouped_stem_fold(cuda, n, h, w):
    """the engine's pixel-grouped stem: 4 pixels x 32 channels per row of the grouped view, statistics folded onto 32 channels"""
    from oracle import yolox_oracle as orc
    from yolov7_d2_b200 import capi
    from yolov7_d2_b200.engine import YoloxEngine

    eng = YoloxEngine(2, 128, 128, device=cuda)
    assert eng.group4, "the pixel-grouped stem is off"
    eng.load_state_dict(orc.yolox_state_dict(12))
    eng.pack_weights()
    torch.cuda.synchronize()
    op = eng.ops[0]
    g = torch.Generator().manual_seed(n * 1000 + h + w)
    x = torch.zeros(n, h, w, 16, dtype=torch.bfloat16)
    x[..., :12] = torch.randn(n, h, w, 12, generator=g).to(torch.bfloat16)
    x = x.to(cuda)
    zb = Guarded((n, h, w // 4, 128), torch.float16, cuda)
    ssum, ssq = run_fwd(capi, capi.act(x.view(n, h, w // 4, 64)), op.w_fwd, capi.act(zb.t), 3, 1, True, 128, cuda, fold=32)
    z = zb.check(0, 128).reshape(n, h, w, 32)
    wq = op.w_src.detach().cpu().to(torch.bfloat16).double()
    xq = nchw(x[..., :12].cpu().double())
    ref = nhwc(F.conv2d(xq, wq, padding=1))
    sabs = nhwc(F.conv2d(xq.abs(), wq.abs(), padding=1))
    _assert_within(z, ref, U_F16 * ref.abs() + (1 + U_F16) * 2 * 108 * U32 * sabs + 2.0 ** -25, "z")
    _check_stats(z, ssum, ssq, 4 * _tiles(n, h, w // 4))


# ---------------------------------------------------------------------------------------------------------------- data gradient (EPI_BF16)

def run_dgrad(capi, dz, wd, dx_act, add_act, k, s):
    capi.check(capi.lib().yb200_conv2d_dgrad(ctypes.byref(capi.act(dz)), capi.ptr(wd), ctypes.byref(dx_act),
                                             ctypes.byref(add_act) if add_act is not None else None, k, s, capi.stream_ptr()), "conv2d_dgrad")
    torch.cuda.synchronize()


@pytest.mark.gpu
@pytest.mark.parametrize("with_addend", [False, True], ids=["plain", "addend"])
@pytest.mark.parametrize("cout", [16, 32, 64], ids=lambda c: f"bk{c}")
@pytest.mark.parametrize("cin", [16, 32, 64, 128], ids=lambda c: f"bn{c}")
def test_dgrad_modes(cuda, cin, cout, with_addend):
    from yolov7_d2_b200 import capi

    n, h, w, k, s = 3, 20, 20, 3, 1
    g = torch.Generator().manual_seed(cin * 5 + cout + with_addend)
    dz = _rand16((n, h, w, cout), g, cuda)
    wt = _weights(cout, cin, k, g, cuda)
    _, wd = _pack(capi, wt)
    add = _rand16((n, h, w, cin), g, cuda) if with_addend else None
    dxb = Guarded((n, h, w, cin), torch.bfloat16, cuda)
    run_dgrad(capi, dz, wd, capi.act(dxb.t), capi.act(add) if with_addend else None, k, s)
    dx = dxb.check(0, cin)
    ref, sabs = _dgrad_ref(dz, wt, k, s, (h, w))
    if with_addend:
        ref, sabs = ref + add.double().cpu(), sabs + add.double().abs().cpu()
    _assert_within(dx, ref, U_BF16 * ref.abs() + (1 + U_BF16) * (2 * cout * k * k + 1) * U32 * sabs, "dx")


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(2, 40, 40, 64, 128, 3, 2), (3, 26, 42, 32, 64, 3, 2), (2, 40, 40, 16, 32, 2, 2), (64, 40, 40, 128, 16, 3, 2),
                                   (2, 24, 40, 128, 64, 3, 1)], ids=lambda s: "x".join(map(str, s)))
def test_dgrad_slices_and_phases(cuda, shape):
    """dx is the second slice of a concat buffer and the addend a slice at another offset of another buffer; stride 2 runs the four
    output-parity phases in one launch (one tensor map per phase); the 20 x 20, 13 x 21 grids overhang the tiles"""
    from yolov7_d2_b200 import capi

    n, h, w, cin, cout, k, s = shape  # dx [n, h, w, cin], dz [n, h / s, w / s, cout]
    g = torch.Generator().manual_seed(sum(shape))
    dz = _rand16((n, h // s, w // s, cout), g, cuda)
    wt = _weights(cout, cin, k, g, cuda)
    _, wd = _pack(capi, wt)
    addb = _rand16((n, h, w, 3 * cin), g, cuda)
    dxb = Guarded((n, h, w, 2 * cin), torch.bfloat16, cuda)
    run_dgrad(capi, dz, wd, capi.act(dxb.t, cin, cin), capi.act(addb, 2 * cin, cin), k, s)
    dx = dxb.check(cin, cin)
    ref, sabs = _dgrad_ref(dz, wt, k, s, (h, w))
    add = addb[..., 2 * cin:].double().cpu()
    ref, sabs = ref + add, sabs + add.abs()
    _assert_within(dx, ref, U_BF16 * ref.abs() + (1 + U_BF16) * (2 * cout * k * k + 1) * U32 * sabs, "dx")


# ---------------------------------------------------------------------------------------------------------------- eval: EPI_BF16_BN_SILU

@pytest.mark.gpu
@pytest.mark.parametrize("residual", [False, True], ids=["plain", "residual"])
@pytest.mark.parametrize("cin", [16, 32, 64], ids=lambda c: f"bk{c}")
@pytest.mark.parametrize("cout", [16, 32, 64, 128], ids=lambda c: f"bn{c}")
def test_bn_silu_modes(cuda, cout, cin, residual):
    from yolov7_d2_b200 import capi

    n, h, w, k, s = 2, 26, 42, 3, 2
    g = torch.Generator().manual_seed(cout * 3 + cin + residual)
    x = _rand16((n, h, w, cin), g, cuda)
    wt = _weights(cout, cin, k, g, cuda)
    wf, _ = _pack(capi, wt)
    scale = (0.5 + torch.rand(cout, generator=g)).to(cuda)
    shift = torch.randn(cout, generator=g).to(cuda)
    oh, ow = h // s, w // s
    resb = _rand16((n, oh, ow, 2 * cout), g, cuda) if residual else None
    ob = Guarded((n, oh, ow, 2 * cout), torch.bfloat16, cuda)
    ra = capi.act(resb, 0, cout) if residual else None
    capi.check(capi.lib().yb200_conv2d_bn_silu_fwd(ctypes.byref(capi.act(x)), capi.ptr(wf), capi.ptr(scale), capi.ptr(shift),
                                                   ctypes.byref(ra) if residual else None, ctypes.byref(capi.act(ob.t, cout, cout)), k, s,
                                                   capi.stream_ptr()), "conv2d_bn_silu_fwd")
    torch.cuda.synchronize()
    out = ob.check(cout, cout)
    acc, sabs = _fwd_ref(x, wt, k, s)
    sc, sh = scale.double().cpu(), shift.double().cpu()
    u = acc * sc + sh
    act = u * torch.sigmoid(u)
    # SiLU' is at most 1.1 in magnitude; __expf / __fdividef add a few fp32 ulps; the activation rounds to bf16 before the residual add
    tol = U_BF16 * act.abs() + 1.1 * sc * 2 * cin * k * k * U32 * sabs + 16 * U32 * (act.abs() + u.abs())
    ref = act
    if residual:
        ref = act + resb[..., :cout].double().cpu()
    tol = tol + U_BF16 * ref.abs() + 2.0 ** -126
    _assert_within(out, ref, tol, "out")


# ---------------------------------------------------------------------------------------------------------------- SASS (no GPU needed)

def test_yolox_gemm_kernels_store_through_tma():
    from yolov7_d2_b200 import build, capi

    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not available")
    if build.find_nvcc() is None and not os.path.exists(capi.LIB_PATH):
        pytest.skip("no nvcc and no prebuilt libyb200.so")
    build.build()
    sass = subprocess.run(["cuobjdump", "-sass", capi.LIB_PATH], capture_output=True, text=True).stdout
    kernels = {}
    for part in re.split(r"\n\s*Function : ", sass)[1:]:
        name, _, body = part.partition("\n")
        if "conv_gemm_persistent_kernel" in name and re.search(r"Lb0E", name):  # EXT = false: the YOLOX instantiations
            kernels[name.strip()] = body
    assert len(kernels) == 12, "expected 12 tile shapes of the YOLOX instantiation"
    for name, body in kernels.items():
        assert re.search(r"\bUTMASTG\b", body), f"{name}: no TMA store"
        assert re.search(r"\bSTSM\b", body), f"{name}: no stmatrix"
        assert not re.search(r"\b(LDL|STL)\b", body), f"{name}: local-memory loads / stores"
