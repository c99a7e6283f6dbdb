"""The convolution GEMMs and ConvNeXt kernels at the geometries of both benchmarked plans (YOLOX-s and YOLOX on ConvNeXt-T), against fp64.

Every reference runs in float64 (on the device: tap-by-tap DGEMMs, elementwise fp64 for the depthwise and LayerNorm ops) on exactly the
bf16 operands the kernel reads.  Each element is judged against its own bound, built from the reference's magnitudes:

    |got - ref| <= r_store * |ref| + c(K) * 2^-24 * mag        (+ r_inner * |inner| where a value is rounded inside the epilogue)

  mag      the same operation on absolute values, e.g. conv(|x|, |w|) = sum of |products| of the element (plus |bias|, |residual|, ...).
  r_store  rounding of the stored result: 2^-11 for the fp16 pre-BatchNorm z, 2^-8 for bf16 outputs, 0 for fp32 gradients.
  c(K)     fp32 accumulation of K terms.  bf16 x bf16 products are exact in fp32, so the error is that of summing K terms.  In any order,
           sum_k delta_k * S_k with |delta_k| <= u per addition and |S_k| <= mag; the worst case is K * u * mag, far from what happens:
           under the probabilistic model of Higham and Mary (SIAM J. Sci. Comput. 41(5), 2019) the error is <= lambda * sqrt(K) * u * mag
           with probability >= 1 - 2 exp(-lambda^2 / 2) per addition chain.  We take lambda = 8 (failure probability ~1e-14) and
           u = 2^-23 rather than 2^-24 because the tensor cores may truncate instead of rounding when they align products.  The constant
           16 covers the O(1) fp32 operations of the epilogues (scale / shift FMA, residual add, __expf / __fdividef of SiLU, the
           Abramowitz-Stegun erf of GELU with |error| < 1.5e-7 ~ 2.5 * 2^-24 relative to |u|), each a few units of 2^-24 of a term that
           `mag` bounds.  So c(K) = 2 * lambda * sqrt(K) + 16.

BatchNorm statistics are checked against fp64 sums of the stored z, with K = number of pixels.  tests/test_convnext_plan_tol_cpu.py
applies the same bound to small instances after a known defect (a dropped k-block, tap or column tile, a split counted twice, a border
pixel read one pixel off) and shows that each is rejected while the fp32-computed, storage-rounded result is accepted.

The views are replayed on fresh buffers: input channels outside a view hold a large finite sentinel (2^14), so any read past the view is a
gross error; output channels outside the view hold random data and must be bit-identical afterwards; every output element inside the view
starts as NaN and must be finite afterwards.
"""
import ctypes
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
LAMBDA = 8.0
R_F16, R_BF16 = 2.0 ** -11, 2.0 ** -8
SENTINEL = 2.0 ** 14
GUARD = 64  # fp64 / fp32 elements behind every per-channel output; they must keep their value
WORST = {}  # case class -> worst err / bound seen in this module (printed at the end with -s)


# ------------------------------------------------------------------------------------------------------------------------------------
# bound
# ------------------------------------------------------------------------------------------------------------------------------------
def acc_c(k):
    return 2.0 * LAMBDA * math.sqrt(k) + 16.0


def bound(ref, mag, k, r_store, inner=None, r_inner=0.0):
    b = r_store * ref.abs() + acc_c(k) * U * mag
    if inner is not None:
        b = b + r_inner * inner.abs()
    return b


SLAB = 1 << 25  # elements compared per step: the fp64 temporaries of a check stay ~1 GB at the 64 x 640 x 640 plan's sizes


def excess(got, ref, bnd):
    """worst |got - ref| / bound over the elements (inf if any value is not finite)"""
    got, ref, bnd = got.reshape(-1), ref.reshape(-1), bnd.reshape(-1)
    worst = 0.0
    for i in range(0, got.numel(), SLAB):
        sl = slice(i, i + SLAB)
        gs = got[sl].double()
        if not torch.isfinite(gs).all():
            return math.inf
        worst = max(worst, float(((gs - ref[sl]).abs() / bnd[sl].clamp_min(1e-300)).max()))
    return worst


def check(cls, got, ref, bnd, what):
    r = excess(got, ref, bnd)
    WORST[cls] = max(WORST.get(cls, 0.0), r)
    if r <= 1.0:
        return
    got = got.double()
    if not torch.isfinite(got).all():
        bad = (~torch.isfinite(got)).nonzero()
        raise AssertionError(f"{what}: {bad.shape[0]} non-finite values, first at {bad[0].tolist()}")
    q = (got - ref).abs() / bnd.clamp_min(1e-300)
    bad = (q > 1).nonzero()
    i = tuple(bad[0].tolist())
    raise AssertionError(f"{what}: {bad.shape[0]}/{q.numel()} elements outside the bound, worst ratio {r:.3g}; first at {list(i)}: "
                         f"got {got[i].item():.6g} ref {ref[i].item():.6g} bound {bnd[i].item():.3g}")


# ------------------------------------------------------------------------------------------------------------------------------------
# fp64 references (NHWC activations, OIHW weights); each returns (ref, mag, K)
# ------------------------------------------------------------------------------------------------------------------------------------
def _tap_slices(xp, k, s, oh, ow):
    for kh in range(k):
        for kw in range(k):
            yield kh, kw, (slice(None), slice(kh, kh + s * (oh - 1) + 1, s), slice(kw, kw + s * (ow - 1) + 1, s))


def _pad(x, p):
    return F.pad(x, (0, 0, p, p, p, p)) if p else x


def _chunks(n, chunk):
    """batch slices of `chunk` images (all of them at once when chunk is None): the fp64 temporaries of a reference scale with the chunk"""
    step = chunk or n
    return [slice(i, min(n, i + step)) for i in range(0, n, step)]


def conv_ref(x, w, k, s, chunk=None):
    """z = conv2d(x, w), padding (k - 1) // 2, as one DGEMM per tap (per batch chunk)"""
    n, h, wd, cin = x.shape
    cout, p = w.shape[0], (k - 1) // 2
    oh, ow = h // s, wd // s
    ref = x.new_zeros(n, oh, ow, cout)
    mag = x.new_zeros(n, oh, ow, cout)
    for b in _chunks(n, chunk):
        xp, xa = _pad(x[b], p), _pad(x[b].abs(), p)
        r, m = ref[b].view(-1, cout), mag[b].view(-1, cout)
        for kh, kw, sl in _tap_slices(xp, k, s, oh, ow):
            wt = w[:, :, kh, kw]
            r += xp[sl].reshape(-1, cin) @ wt.t()
            m += xa[sl].reshape(-1, cin) @ wt.abs().t()
    return ref, mag, k * k * cin


def dgrad_ref(dz, w, k, s, xshape, chunk=None):
    """dx = conv2d_input(dz, w): every tap's product scattered back to the input pixels it came from (per batch chunk)"""
    n, h, wd, cin = xshape
    _, oh, ow, cout = dz.shape
    p = (k - 1) // 2
    out = dz.new_empty(n, h, wd, cin)
    out_mag = torch.empty_like(out)
    crop = (slice(None), slice(p, p + h), slice(p, p + wd))
    for b in _chunks(n, chunk):
        nb = b.stop - b.start
        ref = dz.new_zeros(nb, h + 2 * p, wd + 2 * p, cin)
        mag = torch.zeros_like(ref)
        d2, a2 = dz[b].reshape(-1, cout), dz[b].abs().reshape(-1, cout)
        for kh, kw, sl in _tap_slices(ref, k, s, oh, ow):
            wt = w[:, :, kh, kw]
            ref[sl] += (d2 @ wt).view(nb, oh, ow, cin)
            mag[sl] += (a2 @ wt.abs()).view(nb, oh, ow, cin)
        out[b], out_mag[b] = ref[crop], mag[crop]
    return out, out_mag, k * k * cout


def wgrad_ref(x, dz, k, s, chunk=None):
    """grad[co, ci, kh, kw] = sum over output pixels of dz * x(tap); per batch chunk, the chunks' sums added"""
    cin, (n, oh, ow, cout) = x.shape[-1], dz.shape
    p = (k - 1) // 2
    ref = x.new_zeros(cout, cin, k, k)
    mag = torch.zeros_like(ref)
    for b in _chunks(n, chunk):
        xp, xa = _pad(x[b], p), _pad(x[b].abs(), p)
        d2, a2 = dz[b].reshape(-1, cout), dz[b].abs().reshape(-1, cout)
        for kh, kw, sl in _tap_slices(xp, k, s, oh, ow):
            ref[:, :, kh, kw] += d2.t() @ xp[sl].reshape(-1, cin)
            mag[:, :, kh, kw] += a2.t() @ xa[sl].reshape(-1, cin)
    return ref, mag, n * oh * ow


def dw7_ref(x, w49, flip):
    """depthwise 7x7, zero padding 3: out[p] = sum x[p + (ky-3, kx-3)] w[ky][kx] (flip: with the kernel rotated by 180 degrees)"""
    n, h, wd, c = x.shape
    xp, xa = _pad(x, 3), _pad(x.abs(), 3)
    ref, mag = torch.zeros_like(x), torch.zeros_like(x)
    for ky in range(7):
        for kx in range(7):
            wk = w49[:, 6 - ky, 6 - kx] if flip else w49[:, ky, kx]
            ref += xp[:, ky:ky + h, kx:kx + wd] * wk
            mag += xa[:, ky:ky + h, kx:kx + wd] * wk.abs()
    return ref, mag, 49


def dw7_wgrad_ref(x, dy):
    n, h, wd, c = x.shape
    xp = _pad(x, 3)
    ref, mag = x.new_zeros(c, 7, 7), x.new_zeros(c, 7, 7)
    d2, a2 = dy.reshape(-1, c), dy.abs().reshape(-1, c)
    for ky in range(7):
        for kx in range(7):
            xs = xp[:, ky:ky + h, kx:kx + wd].reshape(-1, c)
            ref[:, ky, kx] = (d2 * xs).sum(0)
            mag[:, ky, kx] = (a2 * xs.abs()).sum(0)
    return ref, mag, n * h * wd


def gelu64(u):
    return u * 0.5 * (1.0 + torch.erf(u / math.sqrt(2.0)))


def gelu_grad64(u):
    return 0.5 * (1.0 + torch.erf(u / math.sqrt(2.0))) + u * torch.exp(-0.5 * u * u) / math.sqrt(2.0 * math.pi)


# ------------------------------------------------------------------------------------------------------------------------------------
# buffers and calls
# ------------------------------------------------------------------------------------------------------------------------------------
def _lib():
    from yolov7_d2_b200 import capi

    return capi, capi.lib()


def _g(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _sl(t, geo):
    return t[..., geo[5]:geo[5] + geo[3]]


def _in_view(geo, g, scale=1.0, shift=0.0):
    """bf16 buffer of the view's pitch: the view holds N(shift, scale^2) values, every other channel the sentinel"""
    n, h, w, c, pitch, off = geo
    t = torch.full((n, h, w, pitch), SENTINEL, dtype=torch.bfloat16, device="cuda")
    t[..., off:off + c] = (torch.randn(n, h, w, c, generator=g, device="cuda") * scale + shift).to(torch.bfloat16)
    return t


def _out_view(geo, g, dtype=torch.bfloat16):
    """buffer of the view's pitch: random outside the view, NaN inside; returns (buffer, copy)"""
    n, h, w, c, pitch, off = geo
    t = torch.randn(n, h, w, pitch, generator=g, device="cuda").to(dtype)
    t[..., off:off + c] = float("nan")
    return t, t.clone()


def _act(capi, t, geo):
    return capi.act(t, geo[5], geo[3])


def _outside_same(after, before, geo, what):
    off, c = geo[5], geo[3]
    assert torch.equal(after[..., :off], before[..., :off]) and torch.equal(after[..., off + c:], before[..., off + c:]), \
        f"{what}: channels outside the output view [{off}, {off + c}) of pitch {geo[4]} changed"


def _guarded(shape, fill, dtype=torch.float32):
    """tensor of `shape` followed by GUARD elements of 7; returns (flat buffer, view)"""
    n = math.prod(shape)
    buf = torch.full((n + GUARD,), 7.0, dtype=dtype, device="cuda")
    buf[:n] = fill.reshape(-1) if torch.is_tensor(fill) else fill
    return buf, buf[:n].view(shape)


def _guard_ok(buf, n, what):
    assert (buf[n:] == 7.0).all(), f"{what}: wrote past the end of its output"


def _weights(capi, L, cout, cin, k, g, mask=None, dgrad=True):
    """random bf16-valued weights (fp64 copy) and their packed forward / data-gradient forms"""
    w = (torch.randn(cout, cin, k, k, generator=g, device="cuda") / math.sqrt(cin * k * k)).to(torch.bfloat16).float()
    if mask is not None:
        w = w * mask
    wf = torch.empty(cout, k * k, cin, dtype=torch.bfloat16, device="cuda")
    wd = torch.empty(cin, k * k, cout, dtype=torch.bfloat16, device="cuda") if dgrad else None
    capi.check(L.yb200_pack_conv_weight(capi.ptr(w), cout, cin, k, cout, cin, capi.ptr(wf), capi.ptr(wd), capi.stream_ptr()), "pack")
    return w.double(), wf, wd


def _fold_mask(cout, cin, group):
    """the zeros of a pixel-grouped 3x3 weight matrix (yb200_conv2d_fwd_fold): the left / right neighbour group reaches this group's
    outputs only through its last / first pixel"""
    cpp = cin // group
    m = torch.ones(cout, cin, 3, 3, device="cuda")
    m[:, :(group - 1) * cpp, :, 0] = 0
    m[:, cpp:, :, 2] = 0
    return m


def run_fwd(gx, gz, k, s, stats=True, fold=0, seed=1, chunk=None):
    """yb200_conv2d_fwd (fold > 0: yb200_conv2d_fwd_fold with stat_fold = fold): fp16 z and its BatchNorm statistics"""
    capi, L = _lib()
    g = _g(seed)
    x = _in_view(gx, g)
    cin, cout = gx[3], gz[3]
    w, wf, _ = _weights(capi, L, cout, cin, k, g, _fold_mask(cout, cin, cout // fold) if fold and k == 3 else None, dgrad=False)
    z, z0 = _out_view(gz, g, torch.float16)
    nst = fold or cout
    sb, ssum = _guarded((nst,), 0.0, torch.float64)
    qb, ssq = _guarded((nst,), 0.0, torch.float64)
    xa, za = _act(capi, x, gx), _act(capi, z, gz)
    ps, pq = (capi.ptr(ssum), capi.ptr(ssq)) if stats else (None, None)
    if fold:
        rc = L.yb200_conv2d_fwd_fold(ctypes.byref(xa), capi.ptr(wf), ctypes.byref(za), k, s, ps, pq, fold, capi.stream_ptr())
    else:
        rc = L.yb200_conv2d_fwd(ctypes.byref(xa), capi.ptr(wf), ctypes.byref(za), k, s, ps, pq, capi.stream_ptr())
    capi.check(rc, "conv2d_fwd")
    ref, mag, kk = conv_ref(_sl(x, gx).double(), w, k, s, chunk)
    zs = _sl(z, gz)
    check("fwd z (fp16)", zs, ref, bound(ref, mag, kk, R_F16), "z")
    _outside_same(z, z0, gz, "z")
    if stats:
        zd = zs.double().reshape(-1, nst)
        npix = zd.shape[0]
        check("BatchNorm statistics", ssum, zd.sum(0), bound(zd.sum(0), zd.abs().sum(0), npix, 0.0), "sum of z")
        check("BatchNorm statistics", ssq, (zd * zd).sum(0), bound((zd * zd).sum(0), (zd * zd).sum(0), npix, 0.0), "sum of z^2")
        _guard_ok(sb, nst, "sum of z")
        _guard_ok(qb, nst, "sum of z^2")


def run_bn_silu(gx, go, gr, k, s, seed=2, chunk=None):
    """yb200_conv2d_bn_silu_fwd: bf16(SiLU(conv * scale + shift)) [+ residual, after rounding the activation]"""
    capi, L = _lib()
    g = _g(seed)
    x = _in_view(gx, g)
    cin, cout = gx[3], go[3]
    w, wf, _ = _weights(capi, L, cout, cin, k, g, dgrad=False)
    scale = torch.rand(cout, generator=g, device="cuda") + 0.5
    shift = torch.randn(cout, generator=g, device="cuda") * 0.3
    res = _in_view(gr, g) if gr else None
    out, out0 = _out_view(go, g)
    xa, oa = _act(capi, x, gx), _act(capi, out, go)
    ra = _act(capi, res, gr) if gr else None
    capi.check(L.yb200_conv2d_bn_silu_fwd(ctypes.byref(xa), capi.ptr(wf), capi.ptr(scale), capi.ptr(shift), ctypes.byref(ra) if gr else None,
                                          ctypes.byref(oa), k, s, capi.stream_ptr()), "conv2d_bn_silu_fwd")
    zc, mag, kk = conv_ref(_sl(x, gx).double(), w, k, s, chunk)
    u = zc * scale.double() + shift.double()
    act = u * torch.sigmoid(u)
    mag = 1.1 * (mag * scale.double() + shift.double().abs())  # |SiLU'| <= 1.1
    ref = act
    if gr:
        rv = _sl(res, gr).double()
        ref, mag = act + rv, mag + rv.abs()
    check("bn_silu / affine fwd", _sl(out, go), ref, bound(ref, mag, kk, R_BF16, act if gr else None, R_BF16 * 1.02), "out")
    _outside_same(out, out0, go, "out")


def run_affine(gx, go, gr, k, s, with_scale=True, with_shift=True, seed=3, chunk=None):
    """yb200_conv2d_affine_fwd: bf16(conv * scale + shift [+ residual])"""
    capi, L = _lib()
    g = _g(seed)
    x = _in_view(gx, g)
    cin, cout = gx[3], go[3]
    w, wf, _ = _weights(capi, L, cout, cin, k, g, dgrad=False)
    scale = torch.rand(cout, generator=g, device="cuda") + 0.5 if with_scale else None
    shift = torch.randn(cout, generator=g, device="cuda") * 0.3 if with_shift else None
    res = _in_view(gr, g) if gr else None
    out, out0 = _out_view(go, g)
    xa, oa = _act(capi, x, gx), _act(capi, out, go)
    ra = _act(capi, res, gr) if gr else None
    capi.check(L.yb200_conv2d_affine_fwd(ctypes.byref(xa), capi.ptr(wf), capi.ptr(scale), capi.ptr(shift), ctypes.byref(ra) if gr else None,
                                         ctypes.byref(oa), k, s, capi.stream_ptr()), "conv2d_affine_fwd")
    ref, mag, kk = conv_ref(_sl(x, gx).double(), w, k, s, chunk)
    if scale is not None:
        ref, mag = ref * scale.double(), mag * scale.double()
    if shift is not None:
        ref, mag = ref + shift.double(), mag + shift.double().abs()
    if gr:
        rv = _sl(res, gr).double()
        ref, mag = ref + rv, mag + rv.abs()
    check("bn_silu / affine fwd", _sl(out, go), ref, bound(ref, mag, kk, R_BF16), "out")
    _outside_same(out, out0, go, "out")


def run_dgrad(gdz, gdx, ga, k, s, seed=4, chunk=None):
    """yb200_conv2d_dgrad: bf16(conv2d_input(dz, w) [+ addend])"""
    capi, L = _lib()
    g = _g(seed)
    dz = _in_view(gdz, g)
    cout, cin = gdz[3], gdx[3]
    w, _, wd = _weights(capi, L, cout, cin, k, g)
    add = _in_view(ga, g) if ga else None
    dx, dx0 = _out_view(gdx, g)
    dza, dxa = _act(capi, dz, gdz), _act(capi, dx, gdx)
    aa = _act(capi, add, ga) if ga else None
    capi.check(L.yb200_conv2d_dgrad(ctypes.byref(dza), capi.ptr(wd), ctypes.byref(dxa), ctypes.byref(aa) if ga else None, k, s,
                                    capi.stream_ptr()), "conv2d_dgrad")
    ref, mag, kk = dgrad_ref(_sl(dz, gdz).double(), w, k, s, (gdx[0], gdx[1], gdx[2], cin), chunk)
    if ga:
        av = _sl(add, ga).double()
        ref, mag = ref + av, mag + av.abs()
    check("dgrad (bf16)", _sl(dx, gdx), ref, bound(ref, mag, kk, R_BF16), "dx")
    _outside_same(dx, dx0, gdx, "dx")


def run_wgrad(gx, gdz, k, s, cin_real=None, accumulate=0, group=0, repeat=False, seed=5, chunk=None):
    """yb200_conv2d_wgrad (group > 1: _wgrad_grouped): fp32 [cout][cin_real][k][k], split-K partials reduced in a fixed order"""
    capi, L = _lib()
    g = _g(seed)
    x, dz = _in_view(gx, g), _in_view(gdz, g)
    cout, cin = gdz[3], gx[3]
    cin_real = cin_real or cin
    xa, dza = _act(capi, x, gx), _act(capi, dz, gdz)
    ws_bytes = L.yb200_conv2d_wgrad_workspace(ctypes.byref(xa), ctypes.byref(dza), k, s)
    assert ws_bytes > 0, L.yb200_last_error()
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device="cuda")
    shape = (cout, cin_real, k, k)
    g0 = torch.randn(shape, generator=g, device="cuda")
    buf, grad = _guarded(shape, g0 if accumulate else float("nan"))

    def call(dst, acc):
        if group:
            rc = L.yb200_conv2d_wgrad_grouped(ctypes.byref(xa), ctypes.byref(dza), k, s, cin_real, group, capi.ptr(dst), acc, capi.ptr(ws),
                                              ctypes.c_int64(ws_bytes), capi.stream_ptr())
        else:
            rc = L.yb200_conv2d_wgrad(ctypes.byref(xa), ctypes.byref(dza), k, s, cin_real, capi.ptr(dst), acc, capi.ptr(ws),
                                      ctypes.c_int64(ws_bytes), capi.stream_ptr())
        capi.check(rc, "conv2d_wgrad")

    call(grad, accumulate)
    ref, mag, kk = wgrad_ref(_sl(x, gx).double(), _sl(dz, gdz).double(), k, s, chunk)
    ref, mag = ref[:, :cin_real], mag[:, :cin_real]
    got = grad
    if accumulate:
        ref, mag = ref + g0.double(), mag + g0.double().abs()
    if group:  # only the positions the expansion fills are computed
        m = _fold_mask(cout, cin, group)[:, :cin_real].bool()
        got, ref, mag = got[m], ref[m], mag[m]
    check("wgrad (fp32)", got, ref, bound(ref, mag, kk, 0.0), "grad")
    _guard_ok(buf, math.prod(shape), "grad")
    if repeat:  # fixed summation order: the same call gives the same bits
        again = torch.full(shape, float("nan"), device="cuda")
        if accumulate:
            again.copy_(g0)
        call(again, accumulate)
        assert torch.equal(again, grad), "weight gradient is not bit-reproducible"


def run_linear_gelu(gx, gu, gh, seed=6):
    """yb200_linear_gelu_fwd: u = bf16(x W^T + b) (optional output), h = bf16(GELU(u)) of the stored u"""
    capi, L = _lib()
    g = _g(seed)
    x = _in_view(gx, g)
    cin, hid = gx[3], gh[3]
    w, wf, _ = _weights(capi, L, hid, cin, 1, g, dgrad=False)
    b = torch.rand(hid, generator=g, device="cuda") - 0.5
    u, u0 = _out_view(gu, g) if gu else (None, None)
    h, h0 = _out_view(gh, g)
    xa, ha = _act(capi, x, gx), _act(capi, h, gh)
    ua = _act(capi, u, gu) if gu else None
    capi.check(L.yb200_linear_gelu_fwd(ctypes.byref(xa), capi.ptr(wf), capi.ptr(b), ctypes.byref(ua) if gu else None, ctypes.byref(ha),
                                       capi.stream_ptr()), "linear_gelu_fwd")
    uref, mag, kk = conv_ref(_sl(x, gx).double(), w, 1, 1)
    uref, mag = uref + b.double(), mag + b.double().abs()
    if gu:
        check("linear + GELU", _sl(u, gu), uref, bound(uref, mag, kk, R_BF16), "u")
        _outside_same(u, u0, gu, "u")
        us = _sl(u, gu).double()
        href = gelu64(us)  # GELU of the stored u: only the evaluation and the storage rounding remain
        check("linear + GELU", _sl(h, gh), href, bound(href, us.abs(), 1, R_BF16), "h")
    else:
        href = gelu64(uref)  # |GELU'| <= 1.13 carries u's rounding inside the epilogue
        check("linear + GELU", _sl(h, gh), href, bound(href, 1.13 * mag, kk, R_BF16, uref, 1.13 * R_BF16), "h")
    _outside_same(h, h0, gh, "h")


def run_dgrad_gelu(gdz, gu, gdu, bias_sum=True, seed=7):
    """yb200_linear_dgrad_gelu: du = bf16((dz W) * GELU'(u)), and the column sums of the stored du into fp64"""
    capi, L = _lib()
    g = _g(seed)
    dz = _in_view(gdz, g)
    u = _in_view(gu, g, scale=1.5)
    c, hid = gdz[3], gdu[3]
    w, _, wd = _weights(capi, L, c, hid, 1, g)
    du, du0 = _out_view(gdu, g)
    sb, acc = _guarded((hid,), 0.0, torch.float64)
    dza, ua, dua = _act(capi, dz, gdz), _act(capi, u, gu), _act(capi, du, gdu)
    capi.check(L.yb200_linear_dgrad_gelu(ctypes.byref(dza), capi.ptr(wd), ctypes.byref(ua), ctypes.byref(dua), capi.ptr(acc) if bias_sum else None,
                                         capi.stream_ptr()), "linear_dgrad_gelu")
    d, mag, kk = dgrad_ref(_sl(dz, gdz).double(), w, 1, 1, (gdu[0], gdu[1], gdu[2], hid))
    uv = _sl(u, gu).double()
    gp = gelu_grad64(uv)
    ref = d * gp
    mag = mag * (gp.abs() + 1.0 + uv.abs())  # the GELU' evaluation error is a few 2^-24 of (1 + |u|)
    check("linear dgrad + GELU'", _sl(du, gdu), ref, bound(ref, mag, kk, R_BF16), "du")
    _outside_same(du, du0, gdu, "du")
    if bias_sum:
        dd = _sl(du, gdu).double().reshape(-1, hid)
        check("linear dgrad + GELU'", acc, dd.sum(0), bound(dd.sum(0), dd.abs().sum(0), dd.shape[0], 0.0), "bias-gradient sums")
        _guard_ok(sb, hid, "bias-gradient sums")


def run_pred(gx, cout, a_total, a_off, c_total, c_off, seed=8, chunk=None):
    """yb200_conv1x1_bias_f32: fp32 rows [n][a_total][c_total], block [a_off + pixel][c_off + c]"""
    capi, L = _lib()
    g = _g(seed)
    x = _in_view(gx, g)
    n, h, w_, cin = gx[0], gx[1], gx[2], gx[3]
    w, wf, _ = _weights(capi, L, cout, cin, 1, g, dgrad=False)
    b = torch.randn(cout, generator=g, device="cuda")
    out = torch.randn(n, a_total, c_total, generator=g, device="cuda")
    blk = (slice(None), slice(a_off, a_off + h * w_), slice(c_off, c_off + cout))
    out[blk] = float("nan")
    out0 = out.clone()
    xa = _act(capi, x, gx)
    capi.check(L.yb200_conv1x1_bias_f32(ctypes.byref(xa), capi.ptr(wf), capi.ptr(b), cout, capi.ptr(out), a_total, a_off, c_total, c_off,
                                        capi.stream_ptr()), "conv1x1_bias_f32")
    ref, mag, kk = conv_ref(_sl(x, gx).double(), w, 1, 1, chunk)
    ref, mag = (ref + b.double()).reshape(n, h * w_, cout), (mag + b.double().abs()).reshape(n, h * w_, cout)
    check("prediction conv (fp32)", out[blk], ref, bound(ref, mag, kk, 0.0), "out")
    out[blk] = 0
    out0[blk] = 0
    assert torch.equal(out, out0), "wrote outside its block of the prediction tensor"


# ------------------------------------------------------------------------------------------------------------------------------------
# section 2: every convolution geometry of both benchmarked plans, recorded from the plans
# ------------------------------------------------------------------------------------------------------------------------------------
def _geo(a):
    if a is None:
        return None
    v = a._obj
    return (v.n, v.h, v.w, v.c, v.c_pitch, v.c_off)


def _given(a):
    return a is not None and not (isinstance(a, ctypes.c_void_p) and not a.value)


def _pv(a):
    return a.value if isinstance(a, ctypes.c_void_p) else None


def _case_of(name, a):
    """(label, weight or gradient pointer, replay case) of one recorded call"""
    if name in ("yb200_conv2d_fwd", "yb200_conv2d_fwd_fold"):
        fold = a[7] if name.endswith("fold") else 0
        return ("fwd_fold" if fold else "fwd"), _pv(a[1]), dict(fn="fwd", gx=_geo(a[0]), gz=_geo(a[2]), k=a[3], s=a[4], stats=_given(a[5]),
                                                                fold=fold)
    if name == "yb200_conv2d_bn_silu_fwd":
        return "bn_silu_fwd", _pv(a[1]), dict(fn="bn_silu", gx=_geo(a[0]), go=_geo(a[5]), gr=_geo(a[4]), k=a[6], s=a[7])
    if name == "yb200_conv2d_affine_fwd":
        return "affine_fwd", _pv(a[1]), dict(fn="affine", gx=_geo(a[0]), go=_geo(a[5]), gr=_geo(a[4]), k=a[6], s=a[7], with_scale=_given(a[2]),
                                             with_shift=_given(a[3]))
    if name == "yb200_conv2d_dgrad":
        return "dgrad", _pv(a[1]), dict(fn="dgrad", gdz=_geo(a[0]), gdx=_geo(a[2]), ga=_geo(a[3]), k=a[4], s=a[5])
    if name == "yb200_conv2d_wgrad":
        return "wgrad", _pv(a[5]), dict(fn="wgrad", gx=_geo(a[0]), gdz=_geo(a[1]), k=a[2], s=a[3], cin_real=a[4], accumulate=a[6], group=0)
    if name == "yb200_conv2d_wgrad_grouped":
        return "wgrad_grouped", _pv(a[6]), dict(fn="wgrad", gx=_geo(a[0]), gdz=_geo(a[1]), k=a[2], s=a[3], cin_real=a[4], group=a[5],
                                                accumulate=a[7])
    if name == "yb200_linear_gelu_fwd":
        return "linear_gelu_fwd", _pv(a[1]), dict(fn="linear_gelu", gx=_geo(a[0]), gu=_geo(a[3]), gh=_geo(a[4]))
    if name == "yb200_linear_dgrad_gelu":
        return "linear_dgrad_gelu", _pv(a[1]), dict(fn="dgrad_gelu", gdz=_geo(a[0]), gu=_geo(a[2]), gdu=_geo(a[3]), bias_sum=_given(a[4]))
    if name == "yb200_conv1x1_bias_f32":
        return "conv1x1_bias_f32", _pv(a[1]), dict(fn="pred", gx=_geo(a[0]), cout=a[3], a_total=a[5], a_off=a[6], c_total=a[7], c_off=a[8])
    raise AssertionError(name)


RECORDED = ("yb200_conv2d_fwd", "yb200_conv2d_fwd_fold", "yb200_conv2d_bn_silu_fwd", "yb200_conv2d_affine_fwd", "yb200_conv2d_dgrad",
            "yb200_conv2d_wgrad", "yb200_conv2d_wgrad_grouped", "yb200_linear_gelu_fwd", "yb200_linear_dgrad_gelu", "yb200_conv1x1_bias_f32")

RUN = dict(fwd=run_fwd, bn_silu=run_bn_silu, affine=run_affine, dgrad=run_dgrad, wgrad=run_wgrad, linear_gelu=run_linear_gelu,
           dgrad_gelu=run_dgrad_gelu, pred=run_pred)


class _Recorder:
    """stands in for the library handle of an engine: records the convolution calls (as replay cases) and forwards every call"""

    def __init__(self, lib, log):
        self._lib, self._log = lib, log

    def __getattr__(self, name):
        fn = getattr(self._lib, name)
        if name not in RECORDED:
            return fn

        def rec(*a):
            self._log.append(_case_of(name, a))
            return fn(*a)
        return rec


def _yolox_names(eng):
    """weight / gradient pointer -> layer name; head pointers of merged convolutions separately (the fused eval epilogue uses them)"""
    from yolov7_d2_b200.engine import ConvOp, PredOp

    names, heads = {}, {}
    for op in eng.ops:
        if isinstance(op, ConvOp):
            nm = "+".join([op.prefixes[0]] + [p.rsplit(".", 1)[-1] for p in op.prefixes[1:]])
            for t in (op.w_fwd, getattr(op, "w_dgrad", None), getattr(op, "g_dst", None), getattr(op, "g_exp", None)):
                if t is not None:
                    names[t.data_ptr()] = nm
            if op.w_fwd is not None:
                for hd in op.heads:
                    heads[op.w_fwd.data_ptr() + 2 * hd.c0 * op.ksize * op.ksize * op.cin_pad] = hd.prefix
        elif isinstance(op, PredOp):
            for which, ts in (("cls_preds", (op.wc_fwd, op.wc_dgrad, op.gc_dst)), ("reg_obj_preds", (op.wr_fwd, op.wr_dgrad, op.gr_dst))):
                for t in ts:
                    names[t.data_ptr()] = f"head.{which}.{op.level}"
    return names, heads


def _convnext_names(cn):
    names = {cn.packed["stem"].data_ptr(): "backbone.downsample_layers.0.0"}
    for key, val in cn.packed.items():
        if key.startswith("ds"):
            for t in val:
                names[t.data_ptr()] = f"backbone.downsample_layers.{key[2:]}.1"
        elif key.startswith("b"):
            i, j = key[1:].split(".")
            for t, which in zip(val[:4], ("pwconv1", "pwconv1", "pwconv2", "pwconv2")):
                names[t.data_ptr()] = f"backbone.stages.{i}.{j}.{which}"
    for name, t in cn.grads.items():
        if name.endswith("weight") and t.dim() > 1:
            names.setdefault(t.data_ptr(), "backbone." + name[:-len(".weight")])
    for i, st in enumerate(cn.stage):
        names[st.raw.data_ptr()] = f"backbone.stages.{i} pwconv2"
    return names


def _record_plan(plan):
    """one train_step() and one eval_forward() of the plan at batch 2, 256 x 256; returns [(test id, replay case)], one per distinct case"""
    from yolov7_d2_b200 import synth
    from yolov7_d2_b200.engine import YoloxEngine
    from yolov7_d2_b200.yolox_convnext import YoloxConvNeXtEngine

    if plan == "yolox_convnext":
        eng = YoloxConvNeXtEngine(2, 256, 256)
        owners = [eng.cn, eng.yx]
        names, heads = _yolox_names(eng.yx)
        names.update(_convnext_names(eng.cn))
    else:
        eng = YoloxEngine(2, 256, 256)
        owners = [eng]
        names, heads = _yolox_names(eng)
    eng.init_weights(0)
    images, labels = synth.synthetic_batch(2, 256, seed=3)
    eng.images_u8.copy_(images.cuda())
    eng.labels.copy_(labels.cuda())
    log = []
    for o in owners:
        o.L = _Recorder(o.L, log)
    try:
        eng.train_step()
        eng.eval_forward()
        torch.cuda.synchronize()
    finally:
        for o in owners:
            o.L = o.L._lib
    seen, out = {}, []
    for label, p, case in log:
        key = tuple(sorted(case.items()))
        if key in seen:
            seen[key][1] += 1
            continue
        layer = (heads.get(p) if case["fn"] == "bn_silu" else None) or names.get(p, "?")
        seen[key] = [len(out), 1]
        out.append([f"{layer} {label}", case])
    ids = set()
    for k, (i, n) in seen.items():
        tid = out[i][0] + (f" (+{n - 1} more)" if n > 1 else "")
        while tid in ids:
            tid += "'"
        ids.add(tid)
        out[i][0] = tid
    del eng
    torch.cuda.empty_cache()
    return [tuple(x) for x in out]


PLANS = {}


def _plans():
    if not PLANS and torch.cuda.is_available():
        for plan in ("yolox_s", "yolox_convnext"):
            PLANS[plan] = _record_plan(plan)
    return PLANS


def pytest_generate_tests(metafunc):
    """the plan cases are the plans' own calls: recorded when the module is collected on a machine with a GPU"""
    if "plan_case" in metafunc.fixturenames:
        cases = [(plan, tid, case) for plan, lst in _plans().items() for tid, case in lst]
        metafunc.parametrize("plan_case", [c[2] for c in cases], ids=[f"{c[0]}: {c[1]}" for c in cases])


def test_plan_geometry(cuda, plan_case):
    case = dict(plan_case)
    RUN[case.pop("fn")](**case)


def test_plan_recording_is_not_trivial(cuda):
    plans = _plans()
    for plan, lst in plans.items():
        kinds = {c["fn"] for _, c in lst}
        assert len(lst) >= 40, f"{plan}: only {len(lst)} distinct convolution calls recorded"
        assert {"fwd", "dgrad", "wgrad", "bn_silu", "pred"} <= kinds, (plan, kinds)
    cnx = [c for _, c in plans["yolox_convnext"]]
    # the head's cr buffer [cls 192 | reg 192]: the data gradient of cls_convs.k.1 writes its first half, its weight gradient reads it
    assert any(c["fn"] == "dgrad" and c["gdx"][3:] == (192, 384, 0) for c in cnx), "no 192-channel dgrad output slice at c_off 0 of pitch 384"
    assert any(c["fn"] == "wgrad" and c["gx"][3:] == (192, 384, 0) for c in cnx), "no weight gradient reading a 192-channel slice of pitch 384"
    assert {"linear_gelu", "dgrad_gelu", "affine"} <= {c["fn"] for c in cnx}
    assert any(c["fn"] == "wgrad" and c["gdz"][3] == 192 for c in cnx), "no 192-wide dz: the second cout tile that overhangs the view"


# ------------------------------------------------------------------------------------------------------------------------------------
# section 3: planner branches at the edges the plans do not reach
# ------------------------------------------------------------------------------------------------------------------------------------
# Each width appears on each side once per kernel configuration.  What conv_api.cu picks for them:
#   forward / dgrad, pick_block_k(cin):  48 -> 16, 96 -> 32, 192 / 384 / 768 -> 64
#   forward / dgrad, pick_block_n(cout): 48 -> 64 (one partial tile), 96 -> 128 (partial), 192 -> 128 + a partial 64-of-128 tile,
#                                        320 -> two full tiles and a partial one, 384 / 768 -> full tiles
#   plan_wgrad, x side:  48 -> kc_b 16, bn 16, tpc 3;  96 -> kc_b 32, bn 32, cin_tiles 3, tpc 3;  192 -> kc_b 64, bn 64, tpc 3;
#                        384 / 768 -> bn 128, tpc 1 (one CTA per SM: the deeper ring)
#   plan_wgrad, dz side: 48 -> kc_a 32, ma 2 (the second box overhangs; legal because the view ends at its pitch);
#                        96 -> kc_a 64, ma 2 (same);  320 -> a third cout tile that covers 64 of its 128 rows
WIDTH_CIN = (48, 96, 192, 384, 768, 192)
WIDTH_COUT = (48, 96, 192, 320, 384, 768)
WIDTH_CFG = ((1, 1, (3, 13, 11)), (3, 1, (3, 13, 11)), (3, 2, (3, 14, 10)))  # small maps with ragged pixel tiles
WIDTH_CASES = [(k, s, hw, ci, WIDTH_COUT[(i + j) % 6]) for j, (k, s, hw) in enumerate(WIDTH_CFG) for i, ci in enumerate(WIDTH_CIN)]


@pytest.mark.parametrize("k,s,nhw,cin,cout", WIDTH_CASES, ids=[f"k{k}s{s}-{ci}to{co}" for k, s, _, ci, co in WIDTH_CASES])
def test_widths(cuda, k, s, nhw, cin, cout):
    n, h, w = nhw
    gx, gz = (n, h, w, cin, cin, 0), (n, h // s, w // s, cout, cout, 0)
    run_fwd(gx, gz, k, s)
    run_dgrad(gz, gx, None, k, s)
    run_wgrad(gx, gz, k, s)


# Output (and input) views at the first, a middle and the last position of a pitch three views wide.  96: one partial 128-wide column
# tile; 192: a full tile and a partial one whose upper half (64 channels) lies in the neighbouring view, which the epilogue's column mask
# must skip.  The weight gradient reads x and dz as slices; a dz of 96 channels that does not end at its pitch is refused (see below), so
# its dz is 192 wide: the second cout tile's boxes then read 64 channels of the neighbour, which the row mask drops.
SLICE_KINDS = ("fwd", "bn_silu", "affine", "dgrad", "wgrad")
SLICE_CASES = [(kind, c, pos) for kind in SLICE_KINDS for c in (96, 192) for pos in (0, 1, 2) if not (kind == "wgrad" and c == 96)]


@pytest.mark.parametrize("kind,c,pos", SLICE_CASES, ids=[f"{kd}-{c}-{('first', 'middle', 'last')[p]}" for kd, c, p in SLICE_CASES])
def test_slices(cuda, kind, c, pos):
    n, h, w, cin = 2, 13, 11, 96
    gx = (n, h, w, cin, 3 * cin, pos * cin)
    go = (n, h, w, c, 3 * c, pos * c)
    ga = (n, h, w, c, 3 * c, ((pos + 1) % 3) * c)  # residual / addend: a slice of another concat buffer
    if kind == "fwd":
        run_fwd(gx, go, 3, 1, stats=True)
    elif kind == "bn_silu":
        run_bn_silu(gx, go, ga, 3, 1)
    elif kind == "affine":
        run_affine(gx, go, ga, 3, 1)
    elif kind == "dgrad":
        run_dgrad(go, gx, (n, h, w, cin, 3 * cin, ((pos + 2) % 3) * cin), 3, 1)
    else:
        run_wgrad(gx, go, 3, 1)


# Weight-gradient split-K at bench sizes, twice each (fixed summation order), with accumulate = 1:
#   64x80x80 192->192 3x3: 18 CTAs per split (2 cout tiles x 3 cin tiles x 3 tap groups), one CTA per SM (tpc 3 x bn 64 registers) and so
#     the deeper ring; 7 splits of ~915 pixel blocks each: long fp32 accumulations per CTA, then the reduction of the splits.
#   64x20x20 768->768 3x3: the 128 MB workspace cap allows 6 splits, but 324 CTAs per split already exceed one wave, so splits == 1.  (With
#     132 SMs the cap cannot bind: splits * CTAs <= 2 * 132 while the cap allows >= 2048 / CTAs.)
#   1x8x24 192->192 3x3: 3 pixel blocks, fewer than 8 per split: splits == 1.
WGRAD_BENCH = [(64, 80, 80, 192, 192), (64, 20, 20, 768, 768), (1, 8, 24, 192, 192)]


@pytest.mark.parametrize("shape", WGRAD_BENCH, ids=lambda s: "%dx%dx%d-%dto%d" % s)
def test_wgrad_splits(cuda, shape):
    n, h, w, cin, cout = shape
    gx, gdz = (n, h, w, cin, cin, 0), (n, h, w, cout, cout, 0)
    run_wgrad(gx, gdz, 3, 1, repeat=True)
    run_wgrad(gx, gdz, 3, 1, accumulate=1, repeat=True)


# A dz slice whose k-boxes would overhang the view inside the buffer (conv_api.cu, plan_wgrad: dz->c % kc_a != 0 and the view does not
# end at its pitch) must be refused, not computed.
REFUSED = [((2, 8, 8, 96, 192, 0), "96-of-192"), ((2, 8, 8, 80, 96, 0), "80-of-96")]


@pytest.mark.parametrize("gdz", [r[0] for r in REFUSED], ids=[r[1] for r in REFUSED])
def test_wgrad_refuses_overhanging_dz_slice(cuda, gdz):
    capi, L = _lib()
    g = _g(9)
    gx = (2, 8, 8, 64, 64, 0)
    x, dz = _in_view(gx, g), _in_view(gdz, g)
    xa, dza = _act(capi, x, gx), _act(capi, dz, gdz)
    assert L.yb200_conv2d_wgrad_workspace(ctypes.byref(xa), ctypes.byref(dza), 3, 1) == capi.ERR_UNSUPPORTED
    grad = torch.randn(gdz[3], 64, 3, 3, generator=g, device="cuda")
    grad0 = grad.clone()
    ws = torch.zeros(1 << 20, dtype=torch.uint8, device="cuda")
    rc = L.yb200_conv2d_wgrad(ctypes.byref(xa), ctypes.byref(dza), 3, 1, 64, capi.ptr(grad), 0, capi.ptr(ws), ctypes.c_int64(ws.numel()),
                              capi.stream_ptr())
    assert rc == capi.ERR_UNSUPPORTED, (rc, L.yb200_last_error())
    torch.cuda.synchronize()
    assert torch.equal(grad, grad0) and not ws.any(), "a refused call wrote its outputs"


# ------------------------------------------------------------------------------------------------------------------------------------
# section 4: ConvNeXt kernels at bench pixel counts (stage 0 of a 640 x 640 image is 160 x 160 x 96)
# ------------------------------------------------------------------------------------------------------------------------------------
DW_BENCH = [(8, 160, 160, 96), (8, 80, 80, 192), (8, 40, 50, 192)]  # stage 0, stage 1, a width that is not a multiple of the 32-pixel tile


def _bf(n, h, w, c, g, scale=1.0, shift=0.0):
    return (torch.randn(n, h, w, c, generator=g, device="cuda") * scale + shift).to(torch.bfloat16)


@pytest.mark.parametrize("shape", DW_BENCH, ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("flip", [0, 1])
def test_dwconv7_bench(cuda, shape, flip):
    capi, L = _lib()
    n, h, w, c = shape
    g = _g(10)
    x, add = _bf(n, h, w, c, g), _bf(n, h, w, c, g)
    wt = torch.randn(c, 1, 7, 7, generator=g, device="cuda") * 0.15
    bias = torch.randn(c, generator=g, device="cuda") * 0.2
    out = torch.full_like(x, float("nan"))
    xa, aa, oa = capi.act(x), capi.act(add), capi.act(out)
    capi.check(L.yb200_dwconv7(ctypes.byref(xa), capi.ptr(wt), None if flip else capi.ptr(bias), ctypes.byref(aa) if flip else None,
                               ctypes.byref(oa), flip, capi.stream_ptr()), "dwconv7")
    ref, mag, kk = dw7_ref(x.double(), wt.double()[:, 0], flip)
    extra = add.double() if flip else bias.double()
    check("dwconv7", out, ref + extra, bound(ref + extra, mag + extra.abs(), kk + 2, R_BF16), "out")


@pytest.mark.parametrize("shape", DW_BENCH, ids=lambda s: "x".join(map(str, s)))
def test_dwconv7_wgrad_bench(cuda, shape):
    capi, L = _lib()
    n, h, w, c = shape
    g = _g(11)
    x, dy = _bf(n, h, w, c, g), _bf(n, h, w, c, g)
    xa, da = capi.act(x), capi.act(dy)
    ws = torch.empty(max(16, L.yb200_dwconv7_wgrad_workspace(ctypes.byref(xa))), dtype=torch.uint8, device="cuda")
    outs = []
    for _ in range(2):
        gbw, gw = _guarded((c, 7, 7), float("nan"))
        gbb, gb = _guarded((c,), float("nan"))
        capi.check(L.yb200_dwconv7_wgrad(ctypes.byref(xa), ctypes.byref(da), capi.ptr(gw), capi.ptr(gb), 0, capi.ptr(ws), capi.stream_ptr()),
                   "dwconv7_wgrad")
        outs.append((gw, gb))
        _guard_ok(gbw, c * 49, "dwconv7 weight gradient")
        _guard_ok(gbb, c, "dwconv7 bias gradient")
    ref, mag, kk = dw7_wgrad_ref(x.double(), dy.double())
    check("dwconv7 wgrad (fp32)", outs[0][0], ref, bound(ref, mag, kk, 0.0), "weight gradient")
    d2 = dy.double().reshape(-1, c)
    check("dwconv7 wgrad (fp32)", outs[0][1], d2.sum(0), bound(d2.sum(0), d2.abs().sum(0), kk, 0.0), "bias gradient")
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1]), "dwconv7_wgrad is not bit-reproducible"


LN_BENCH = [(8, 160, 160, 96), (8, 20, 20, 768)]


@pytest.mark.parametrize("shape", LN_BENCH, ids=lambda s: "x".join(map(str, s)))
def test_layernorm_and_colsum_bench(cuda, shape):
    """LayerNorm forward / backward and colsum: per-pixel reductions over C, per-channel reductions over every pixel (block partials)"""
    capi, L = _lib()
    n, h, w, c = shape
    g = _g(12)
    eps = 1e-6
    x, dy, add = _bf(n, h, w, c, g, 2.0, 0.5), _bf(n, h, w, c, g), _bf(n, h, w, c, g)
    gamma = torch.rand(c, generator=g, device="cuda") + 0.5
    beta = torch.rand(c, generator=g, device="cuda") - 0.5
    y = torch.full_like(x, float("nan"))
    stats = torch.full((n * h * w, 2), float("nan"), device="cuda")
    xa, ya, da, aa = capi.act(x), capi.act(y), capi.act(dy), capi.act(add)
    capi.check(L.yb200_layernorm_fwd(ctypes.byref(xa), capi.ptr(gamma), capi.ptr(beta), ctypes.c_float(eps), ctypes.byref(ya), capi.ptr(stats),
                                     capi.stream_ptr()), "layernorm_fwd")
    xd, gm, bt = x.double(), gamma.double(), beta.double()
    mean = xd.mean(-1, keepdim=True)
    var = ((xd - mean) ** 2).mean(-1, keepdim=True) + eps
    rstd = var.rsqrt()
    xh = (xd - mean) * rstd
    kappa = 1.0 + (xd * xd).mean(-1, keepdim=True) / var  # conditioning of the variance: its error relative to var is <= kappa * c(C) u
    ref = xh * gm + bt
    mag = gm.abs() * (xh.abs() + rstd * xd.abs().mean(-1, keepdim=True)) * kappa + bt.abs()
    check("LayerNorm", y, ref, bound(ref, mag, c, R_BF16), "y")
    ws = torch.empty(max(16, L.yb200_layernorm_bwd_workspace(ctypes.byref(xa))), dtype=torch.uint8, device="cuda")
    runs = []
    for _ in range(2):
        dx = torch.full_like(x, float("nan"))
        gg, gb = torch.full((c,), float("nan"), device="cuda"), torch.full((c,), float("nan"), device="cuda")
        dxa = capi.act(dx)
        capi.check(L.yb200_layernorm_bwd(ctypes.byref(da), ctypes.byref(xa), capi.ptr(stats), capi.ptr(gamma), ctypes.byref(aa), ctypes.byref(dxa),
                                         capi.ptr(gg), capi.ptr(gb), 0, capi.ptr(ws), capi.stream_ptr()), "layernorm_bwd")
        runs.append((dx, gg, gb))
    dyd = dy.double()
    gd = dyd * gm
    m1, m2 = gd.mean(-1, keepdim=True), (gd * xh).mean(-1, keepdim=True)
    ref = rstd * (gd - m1 - xh * m2) + add.double()
    mag = rstd * (gd.abs() + gd.abs().mean(-1, keepdim=True) + xh.abs() * (gd * xh).abs().mean(-1, keepdim=True)) * (1.0 + kappa) + add.double().abs()
    check("LayerNorm", runs[0][0], ref, bound(ref, mag, c, R_BF16), "dx")
    npix = n * h * w
    d2, x2, k2 = dyd.reshape(-1, c), xh.reshape(-1, c), kappa.reshape(-1, 1)
    rg = (d2 * x2).sum(0)
    check("LayerNorm / colsum parameter gradients (fp32)", runs[0][1], rg, bound(rg, ((d2 * x2).abs() * k2).sum(0), npix + c, 0.0), "grad gamma")
    check("LayerNorm / colsum parameter gradients (fp32)", runs[0][2], d2.sum(0), bound(d2.sum(0), d2.abs().sum(0), npix, 0.0), "grad beta")
    for a, b in zip(runs[0], runs[1]):
        assert torch.equal(a, b), "layernorm_bwd is not bit-reproducible"
    wsc = torch.empty(max(16, L.yb200_colsum_workspace(ctypes.byref(da))), dtype=torch.uint8, device="cuda")
    cs = []
    for _ in range(2):
        buf, out = _guarded((c,), float("nan"))
        capi.check(L.yb200_colsum(ctypes.byref(da), ctypes.c_float(0.5), capi.ptr(out), 0, capi.ptr(wsc), capi.stream_ptr()), "colsum")
        _guard_ok(buf, c, "colsum")
        cs.append(out)
    check("LayerNorm / colsum parameter gradients (fp32)", cs[0], 0.5 * d2.sum(0), bound(0.5 * d2.sum(0), 0.5 * d2.abs().sum(0), npix, 0.0), "colsum")
    assert torch.equal(cs[0], cs[1]), "colsum is not bit-reproducible"


def test_linear_gelu_bench(cuda):
    """pwconv1 + GELU and pwconv2's data gradient + GELU' of a stage-1 block at 8 x 80 x 80 (192 -> 768)"""
    n, h, w, c = 8, 80, 80, 192
    run_linear_gelu((n, h, w, c, c, 0), (n, h, w, 4 * c, 4 * c, 0), (n, h, w, 4 * c, 4 * c, 0))
    run_dgrad_gelu((n, h, w, c, c, 0), (n, h, w, 4 * c, 4 * c, 0), (n, h, w, 4 * c, 4 * c, 0))


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    if WORST:
        print("\nworst |err| / bound per case class: " + "; ".join(f"{k}: {v:.3g}" for k, v in sorted(WORST.items())))
