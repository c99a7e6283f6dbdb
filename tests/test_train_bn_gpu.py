"""Kernel parity, against fp64, of the C ABI calls the YOLOX training step makes around every BatchNorm and prediction layer:
yb200_bn_train_apply_silu (finalize folded into the apply), yb200_bn_silu_bwd in the engine's deferred mode followed by
yb200_bn_param_grads, yb200_head_bias_grad and yb200_pack_conv_weights_batched -- first on synthetic operands at every thread layout of
these kernels, then on every BatchNorm layer of a real YOLOX-s step, on the exact operands the engine gave it.

Every reference is fp64 torch on the stored operands the kernel read (fp16 z, bf16 gradients, fp32 per-channel constants, fp64 sums).
Every tolerance is derived from the kernel's arithmetic: one rounding to the stored type (unit roundoff 2^-8 for bf16), fp32 roundings
(2^-24 each), plus k * 2^-24 * sum|terms| for an fp32 sum whose longest addition path is k long (read from the launch configuration in
csrc/elementwise.cu).  SiLU runs on tanh.approx.f32, whose PTX-documented error is 2^-11: sigmoid_fast = 0.5 + 0.5 tanh(u/2) is then off
by at most 2^-12 absolute, so for u << 0 the SiLU error is about 2^-12 |u| -- absolute, not relative.
"""
import ctypes
import math

import pytest
import torch

from oracle import yolox_oracle as orc

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24   # fp32 unit roundoff
U_BF16 = 2.0 ** -8
D_SIG = 2.0 ** -12 + U32   # sigmoid_fast: 0.5 * (tanh.approx error 2^-11) + the rounding of fma(t, 0.5, 0.5)
EPS = orc.BN_EPS
MOM = orc.BN_MOMENTUM
EW_THREADS, BN_RED_ITERS = 256, 32   # kEwThreads, kBnRedIters (csrc/elementwise.cu)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _layout(c):
    """thread block of the BatchNorm kernels: (c / 8 channel vectors, 256 / (c / 8) pixel rows)"""
    cv = c // 8
    return cv, EW_THREADS // cv


def _red_iters(c, npix):
    """pixels per thread of the reduction pass of yb200_bn_silu_bwd"""
    _, by = _layout(c)
    return min(max(npix // (by * 6 * _sms()), 4), BN_RED_ITERS)


def _red_path(c, npix):
    """longest fp32 addition path of one channel's Σdu (or Σdu·z) before the fp64 atomics: red_iters per thread, the butterfly levels
    (blockDim.x a power of two below 32), then one sequential addition per shared-memory row; +1 for the fp64 atomics across blocks"""
    cv, by = _layout(c)
    shuf = cv < 32 and (cv & (cv - 1)) == 0
    levels = int(math.log2(32 // cv)) if shuf else 0
    rows = cv * by // 32 if shuf else by
    return _red_iters(c, npix) + levels + rows + 1


def _grid(spec):
    """(n, h, w) of a case; ("iters", c, r): a ragged grid on which a c-channel layer gets exactly r reduction iterations per thread"""
    if spec[0] != "iters":
        return spec
    _, c, r = spec
    _, by = _layout(c)
    n, h = 2, 13
    w = by * 6 * _sms() * r // (n * h) + 1
    assert _red_iters(c, n * h * w) == r
    return n, h, w


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


def _fail(name, what, err, tol):
    bad = err > tol
    if bad.any():
        i = int(torch.argmax((err - tol).flatten()))
        pytest.fail(f"{name}: {what}: {int(bad.sum())} of {bad.numel()} beyond the bound, worst {float(err.flatten()[i]):.4g} vs "
                    f"{float(tol.flatten()[i]):.4g} at flat index {i}")


def _p(t, off=0):
    return ctypes.c_void_p(t.data_ptr() + t.element_size() * off)


# ------------------------------------------------------------------------------------------------ forward checks (fp64 references)

def _check_stats(name, S, Q, count, gamma, beta, mean_k, invstd_k, scale_k, shift_k):
    """finalize folded into the apply: mean = S / count and var = Q / count - mean^2 in fp64; invstd = rsqrtf(fp32(var) + eps) plus one
    Newton step; scale = gamma * invstd, shift = beta - fp32(mean) * gamma * invstd in fp32.  Returns the fp64 mean and biased variance."""
    inv_count = 1.0 / count
    mean = S * inv_count
    # save_mean is fp32(S * fp64(1 / count)): bit for bit
    assert torch.equal(mean_k, mean.float()), f"{name}: save_mean"
    var = (Q * inv_count - mean * mean).clamp_min(0)
    r = 1.0 / torch.sqrt(var + float(torch.tensor(EPS, dtype=torch.float32)))
    # invstd: fp32(var) and + eps round twice (2^-24 each, halved by the square root: 1 ulp); rsqrtf is within 2 ulp, so the Newton
    # step's quadratic term is below 2^-43; its fp32 evaluation y0 (1.5 - (0.5 ve y0) y0) rounds three times (the two inside the
    # bracket halved): 3 ulp.  The fp64 fma of the kernel's variance differs from the reference's by < 2^-50 relative.  Total 5 * 2^-24.
    tol_i = 5 * U32 * r
    _fail(name, "save_invstd", (invstd_k.double() - r).abs(), tol_i)
    g, b = gamma.double(), beta.double()
    # scale = gamma * invstd: invstd's 5 ulp + one rounding
    _fail(name, "scale", (scale_k.double() - g * r).abs(), 6 * U32 * (g * r).abs())
    # shift: fp32(mean) (1 ulp), * gamma (1), * invstd (1 + invstd's 5), beta - that (1 ulp of the result)
    m_g_r = mean * g * r
    _fail(name, "shift", (shift_k.double() - (b - m_g_r)).abs(), 8 * U32 * m_g_r.abs() + U32 * (b - m_g_r).abs())
    return mean, var


def _ema(prev, prev_tol, new, new_rel):
    """running = (1 - m) running + m new in fp32, against fp64 with m = 0.03: (1 - fp32(m)) rounds once (and carries fp32(m)'s error),
    its product once, fp32(m) * new twice plus new's own error new_rel, the sum once"""
    ref = (1 - MOM) * prev + MOM * new
    tol = (1 - MOM) * prev_tol + 3 * U32 * (1 - MOM) * prev.abs() + MOM * new.abs() * (3 * U32 + new_rel) + U32 * ref.abs()
    return ref, tol


def _check_running(name, rm0, rv0, mean, var, count, rm_k, rv_k, calls):
    """running statistics after `calls` identical updates: momentum 0.03, the unbiased variance var * count / (count - 1)"""
    unb = var * count / (count - 1) if count > 1 else var
    rm, rv = rm0.double(), rv0.double()
    tm, tv = torch.zeros_like(rm), torch.zeros_like(rv)
    for _ in range(calls):
        # mean enters as fp32(mean) (1 ulp); the unbiased variance as fp32(var) * fp32(count / (count - 1)) (3 ulp)
        rm, tm = _ema(rm, tm, mean, U32)
        rv, tv = _ema(rv, tv, unb, 3 * U32)
    _fail(name, "running_mean", (rm_k.double() - rm).abs(), tm)
    _fail(name, "running_var", (rv_k.double() - rv).abs(), tv)


def _silu_err(u):
    """bound of |fp32 SiLU of the kernel - SiLU(u)| before storage: sigmoid_fast's D_SIG times |u|, the rounding of fma(z, s, t) (1 ulp of
    u) times max |SiLU'| < 1.1, and the rounding of u * sigmoid (1 ulp of the result)"""
    s = u * torch.sigmoid(u)
    return u.abs() * D_SIG + 1.1 * U32 * u.abs() + U32 * s.abs(), s


def _check_apply(name, z, scale_k, shift_k, out_k, res=None):
    """out = bf16(SiLU(fma(z, scale, shift))) [+ residual, added to the bf16-rounded activation, then rounded again], against fp64 with
    the scale / shift the kernel published.  z, res, out: [P, c].  Returns u, |out - SiLU(u)| and the worst error / bound, for reporting."""
    u = z * scale_k.double() + shift_k.double()
    e, silu = _silu_err(u)
    t1 = e + U_BF16 * (silu.abs() + e)   # bf16 rounding of the activation
    ref = silu
    if res is not None:
        ref = silu + res
        t1 = t1 + U32 * (ref.abs() + t1)  # fp32 addition of the residual
        t1 = t1 + U_BF16 * (ref.abs() + t1)
    err = (out_k.double() - ref).abs()
    _fail(name, "activation", err, t1)
    return u, (out_k.double() - silu).abs(), float((err / t1).max())


# ------------------------------------------------------------------------------------------------ backward reference

def _bwd_ref(z, d, d_abs, d_adds, scale, shift, mean, invstd, red_path):
    """fp64 BatchNorm + SiLU backward on the kernel's operands, and bounds for its outputs.

    z, d: [P, c] fp64 (d = the incoming gradient, exact sum of its bf16 sources; d_abs = sum of their magnitudes; d_adds = fp32 additions
    the kernel spends forming d).  scale / shift / mean / invstd: the fp32 per-channel constants the kernel reads.
    The kernel: du = d sig (1 + u (1 - sig)) with u = fma(z, s, t);  acc_dbeta += Σdu,  acc_dgamma += invstd (Σdu·z - mean Σdu), fp32
    per-thread and per-block partials, fp64 across blocks;  dz = bf16(s du + A z + B), A = -s invstd mg, B = -s mb - A mean with
    mg = fp32(acc_dgamma / M), mb = fp32(acc_dbeta / M)."""
    P = z.shape[0]
    s, t, mu, ist = (v.double() for v in (scale, shift, mean, invstd))
    u = z * s + t
    sg = torch.sigmoid(u)
    g = sg * (1 + u * (1 - sg))
    du = d * g
    zh = (z - mu) * ist
    db, dg = du.sum(0), (du * zh).sum(0)
    mb, mg = db / P, dg / P
    dz = s * (du - mb - zh * mg)
    # |du_kernel - du|: dSiLU/dsig = 1 + u - 2 u sig times sigmoid_fast's error; u's rounding times |SiLU''| <= 0.5; four fp32 roundings
    # of d * sg * fma(u, 1 - sg, 1) (1 - sg rounds absolutely, times |u|); the fp32 sum forming d (d_adds additions) times |SiLU'| < 1.1
    e_du = d.abs() * ((1 + u - 2 * u * sg).abs() * D_SIG + 0.5 * U32 * u.abs() + 4 * U32 * sg * (1 + u.abs() * (1 - sg)) + U32 * u.abs() * sg)
    e_du = e_du + 1.1 * d_adds * U32 * d_abs
    # accumulators: the kernel's per-element errors pass through exactly (Σ Δdu and Σ Δdu·zhat: the uncentred form is the same algebra),
    # the fp32 partial sums add red_path roundings of Σ|du| and of the UNCENTRED Σ|du·z|
    k = red_path
    e_db = e_du.sum(0) + k * U32 * du.abs().sum(0)
    e_dg = (e_du * zh.abs()).sum(0) + ist * k * U32 * ((du * z).abs().sum(0) + mu.abs() * du.abs().sum(0))
    # dz: mb, mg round once to fp32; A twice; B (s mb, A mean, difference) three times; fma(A, z, B) once; fma(s, du, .) once; bf16 once
    e_mb = e_db / P + U32 * mb.abs()
    e_mg = e_dg / P + U32 * mg.abs()
    A = -s * ist * mg
    B = -s * mb - A * mu
    e_A = (s * ist).abs() * e_mg + 2 * U32 * A.abs()
    e_B = s.abs() * e_mb + mu.abs() * e_A + 3 * U32 * ((s * mb).abs() + (A * mu).abs())
    e_in = e_A * z.abs() + e_B + U32 * (A * z + B).abs()
    e_o = s.abs() * e_du + e_in + U32 * dz.abs()
    tol_dz = e_o + U_BF16 * (dz.abs() + e_o)
    return dict(dz=dz, tol_dz=tol_dz, dg=dg, e_dg=e_dg, db=db, e_db=e_db, u=u, g=g, sg=sg)


def _check_param(name, what, got, ref, e_acc, prev=None):
    """parameter gradient = fp32(acc) [+ previous value, one more fp32 rounding]"""
    ref = ref if prev is None else prev.double() + ref
    tol = e_acc + U32 * ref.abs() + (0 if prev is None else U32 * ref.abs())
    _fail(name, what, (got.double() - ref).abs(), tol)


# ------------------------------------------------------------------------------------------------ synthetic operands

def _z_values(P, c, g, sweep=False):
    """fp16 pre-BatchNorm values [P, c]: per-channel offset and spread; channel 0 at |mean| / std = 30, channel 1 constant (var = 0,
    invstd = rsqrt(eps)).  sweep: uniform in [-1, 1] (with gamma 11.5 and beta 0, u = gamma * zhat sweeps about [-20, 20])."""
    if sweep:
        return (torch.rand(P, c, generator=g) * 2 - 1).to(torch.float16)
    mean = torch.randn(c, generator=g) * 2
    std = torch.exp(torch.randn(c, generator=g) * 0.7)
    std[0], mean[0] = 0.25, 7.5
    z = mean + std * torch.randn(P, c, generator=g)
    z[:, 1] = 0.75
    return z.to(torch.float16)


def _affine(c, g, sweep=False):
    if sweep:
        return torch.full((c,), 11.5), torch.zeros(c)
    gamma = torch.rand(c, generator=g) + 0.5
    gamma[2 % c] = -0.8  # a negative scale
    return gamma, torch.randn(c, generator=g) * 0.3


# (c, grid, residual, upsampled copy): every thread layout -- c / 8 a power of two below 32 (butterfly), non-powers of two and >= 32
# (shared-memory rows), c = 2048 (256 channel vectors, one pixel row per block); grids below one block row, ragged, odd and 32
# reduction iterations per thread, several waves
APPLY_CASES = [
    (16, (1, 1, 3), True, True),
    (48, (3, 13, 17), False, True),
    (96, ("iters", 96, 5), True, False),
    (192, (2, 9, 11), False, True),
    (256, (4, 10, 10), True, True),
    (320, (3, 13, 17), True, False),
    (768, (2, 7, 5), False, True),
    (2048, (2, 3, 5), True, False),
    (2048, ("iters", 2048, 7), False, False),
    (64, (64, 20, 20), False, False),
    (64, (8, 80, 80), False, True),
    (64, ("iters", 64, 32), True, False),
    (64, (4, 32, 32), False, False, "u_sweep"),
]


def _case_id(cs):
    grid = cs[1]
    gid = f"iters{grid[2]}" if grid[0] == "iters" else "x".join(map(str, grid))
    return f"c{cs[0]}-{gid}" + ("-res" if cs[2] else "") + ("-up" if cs[3] else "") + ("-" + cs[4] if len(cs) > 4 else "")


def _train_apply(L, capi, zv, S, Q, count, gamma, beta, rm, rv, outs, res_v, out_v, up_v):
    scale, shift, mean, invstd = outs
    return L.yb200_bn_train_apply_silu(ctypes.byref(zv), capi.ptr(S), capi.ptr(Q), ctypes.c_int64(count), capi.ptr(gamma), capi.ptr(beta),
                                       ctypes.c_float(EPS), ctypes.c_float(MOM), rm, rv, capi.ptr(scale), capi.ptr(shift), capi.ptr(mean),
                                       capi.ptr(invstd), ctypes.byref(res_v) if res_v is not None else None, ctypes.byref(out_v),
                                       ctypes.byref(up_v) if up_v is not None else None, capi.stream_ptr())


@pytest.mark.parametrize("case", APPLY_CASES, ids=_case_id)
def test_bn_train_apply_silu_against_fp64(cuda, case):
    """z, residual, out and out_up2x are channel slices of wider buffers; the sums come from the stored z in fp64.  Two successive calls:
    the published constants and the output repeat, the running statistics move twice, the sums are not cleared."""
    from yolov7_d2_b200 import capi

    L = capi.lib()
    c, spec, has_res, has_up = case[:4]
    sweep = len(case) > 4
    n, h, w = _grid(spec)
    P = n * h * w
    g = torch.Generator().manual_seed(c * 7 + P)
    zw = torch.randn(n, h, w, c + 24, generator=g).to(torch.float16).to(cuda)
    zw[..., 8:8 + c] = _z_values(P, c, g, sweep).view(n, h, w, c).to(cuda)
    z = zw[..., 8:8 + c].reshape(P, c).double()
    S, Q = z.sum(0), (z * z).sum(0)
    S0, Q0 = S.clone(), Q.clone()
    gamma, beta = (v.to(cuda) for v in _affine(c, g, sweep))
    # running statistics inside wider buffers: the neighbours must stay untouched
    rmw = torch.randn(c + 16, generator=g).to(cuda)
    rvw = (torch.rand(c + 16, generator=g) + 0.5).to(cuda)
    rm0, rv0 = rmw.clone(), rvw.clone()
    outs = [torch.full((c,), float("nan"), device=cuda) for _ in range(4)]
    ow = torch.full((n, h, w, c + 32), 7.0, dtype=torch.bfloat16, device=cuda)
    out_v = capi.act(ow, 16, c)
    resw = torch.randn(n, h, w, c + 8, generator=g).to(torch.bfloat16).to(cuda) if has_res else None
    res_v = capi.act(resw, 8, c) if has_res else None
    upw = torch.full((n, 2 * h, 2 * w, c + 16), 7.0, dtype=torch.bfloat16, device=cuda) if has_up else None
    up_v = capi.act(upw, 8, c) if has_up else None
    zv = capi.act(zw, 8, c)
    capi.check(_train_apply(L, capi, zv, S, Q, P, gamma, beta, _p(rmw, 8), _p(rvw, 8), outs, res_v, out_v, up_v), "bn_train_apply_silu")
    torch.cuda.synchronize()
    first = [o.clone() for o in outs] + [ow.clone()]
    name = _case_id(case)
    scale_k, shift_k, mean_k, invstd_k = outs
    mean, var = _check_stats(name, S, Q, P, gamma, beta, mean_k, invstd_k, scale_k, shift_k)
    _check_running(name, rm0[8:8 + c], rv0[8:8 + c], mean, var, P, rmw[8:8 + c], rvw[8:8 + c], 1)
    res = resw[..., 8:8 + c].reshape(P, c).double() if has_res else None
    out = ow[..., 16:16 + c]
    u, err, worst = _check_apply(name, z, scale_k, shift_k, out.reshape(P, c), res)
    assert (ow[..., :16] == 7).all() and (ow[..., 16 + c:] == 7).all(), "channels outside the output slice were written"
    if has_up:
        rep = out.repeat_interleave(2, 1).repeat_interleave(2, 2)
        assert torch.equal(upw[..., 8:8 + c].view(torch.int16), rep.view(torch.int16)), "out_up2x is not out replicated 2x2"
        assert (upw[..., :8] == 7).all() and (upw[..., 8 + c:] == 7).all(), "channels outside the upsampled slice were written"
    if sweep:
        neg = u < -4   # |SiLU| < 0.08: the bf16 rounding of the stored value is small against tanh.approx's absolute error
        bound = (u.abs() * D_SIG + 1.1 * U32 * u.abs())[neg]
        print(f"\nSiLU over u in [{float(u.min()):.1f}, {float(u.max()):.1f}]: worst |out - SiLU(u)| for u < -4 = {float(err[neg].max()):.3g} "
              f"(bound there {float(bound.max()):.3g}); worst error / |u| = {float((err[neg] / u.abs()[neg]).max()):.3g} vs 2^-12 = {2 ** -12:.3g}; "
              f"worst error / its bound over the whole sweep = {worst:.3g}")
        assert float(u.min()) < -19 and float(u.max()) > 19, "the sweep does not reach |u| = 19"
    # second call: same constants and output, running statistics updated again, sums still there
    capi.check(_train_apply(L, capi, zv, S, Q, P, gamma, beta, _p(rmw, 8), _p(rvw, 8), outs, res_v, out_v, up_v), "bn_train_apply_silu")
    torch.cuda.synchronize()
    for a, b in zip(first, outs + [ow]):
        assert torch.equal(a, b), f"{name}: the second call published different values"
    _check_running(name, rm0[8:8 + c], rv0[8:8 + c], mean, var, P, rmw[8:8 + c], rvw[8:8 + c], 2)
    assert torch.equal(S, S0) and torch.equal(Q, Q0), "stat_sum / stat_sqsum were modified"
    for full, full0 in ((rmw, rm0), (rvw, rv0)):
        assert torch.equal(full[:8], full0[:8]) and torch.equal(full[8 + c:], full0[8 + c:]), "running statistics outside the layer changed"


# (grid, channels of three layers sharing one accumulator run; layer 1 also receives an upsampled gradient)
BWD_CASES = [
    ((1, 1, 3), (16, 48, 2048)),
    ((3, 13, 17), (96, 192, 256)),
    (("iters", 96, 5), (96, 16, 320)),
    (("iters", 2048, 7), (2048, 16, 256)),
    ((64, 20, 20), (64, 768, 48)),
    ((8, 80, 80), (64, 16, 192)),
    (("iters", 64, 32), (64, 16, 48)),
    ((4, 32, 32), (64, 64, 64), "u_sweep"),
]


def _bwd_id(cs):
    gid = f"iters{cs[0][2]}c{cs[0][1]}" if cs[0][0] == "iters" else "x".join(map(str, cs[0]))
    return gid + "-" + "_".join(map(str, cs[1])) + ("-" + cs[2] if len(cs) > 2 else "")


@pytest.mark.parametrize("accumulate", [0, 1])
@pytest.mark.parametrize("case", BWD_CASES, ids=_bwd_id)
def test_bn_silu_bwd_deferred_and_param_grads_against_fp64(cuda, case, accumulate):
    """Three layers at their own channel offsets of one z / dz buffer, their sums deferred into one run of fp64 accumulators, then one
    yb200_bn_param_grads with an offset table that interleaves gamma and beta and skips padding, as engine.py builds it."""
    from yolov7_d2_b200 import capi

    L = capi.lib()
    spec, cs = case[0], case[1]
    sweep = len(case) > 2
    n, h, w = _grid(spec)
    P = n * h * w
    g = torch.Generator().manual_seed(P + sum(cs) + accumulate)
    offs = [8]
    for c in cs[:-1]:
        offs.append(offs[-1] + c + 8)
    pitch = offs[-1] + cs[-1] + 8
    zw = torch.randn(n, h, w, pitch, generator=g).to(torch.float16)
    daw = torch.randn(n, h, w, pitch, generator=g).to(torch.bfloat16)
    for o, c in zip(offs, cs):
        zw[..., o:o + c] = _z_values(P, c, g, sweep).view(n, h, w, c)
        if sweep:  # one pixel in 16 carries a gradient: there dz is s du, the mean terms are small, and dz's error shows SiLU''s
            daw[..., o:o + c] *= (torch.rand(n, h, w, 1, generator=g) < 1 / 16)
    zw, daw = zw.to(cuda), daw.to(cuda)
    c1 = cs[1]
    upw = torch.randn(n, 2 * h, 2 * w, c1 + 16, generator=g).to(torch.bfloat16).to(cuda)
    dzw = torch.full((n, h, w, pitch), float("nan"), dtype=torch.bfloat16, device=cuda)
    ctot = sum(cs)
    acc_g = torch.zeros(ctot + 16, dtype=torch.float64, device=cuda)
    acc_b = torch.zeros(ctot + 16, dtype=torch.float64, device=cuda)
    run = [8]
    for c in cs[:-1]:
        run.append(run[-1] + c)
    # the per-channel constants the forward would have published: from z's statistics and a random affine transform
    consts, refs = [], []
    for j, (o, c) in enumerate(zip(offs, cs)):
        z = zw[..., o:o + c].reshape(P, c).double()
        mean = z.mean(0)
        invstd = 1.0 / torch.sqrt(((z - mean) ** 2).mean(0) + EPS)
        gamma, beta = (v.to(cuda).double() for v in _affine(c, g, sweep))
        mean32, invstd32 = mean.float(), invstd.float()
        scale = (gamma * invstd32.double()).float()
        shift = (beta - mean32.double() * scale.double()).float()
        consts.append((scale, shift, mean32, invstd32))
        zv, dav, dzv = capi.act(zw, o, c), capi.act(daw, o, c), capi.act(dzw, o, c)
        upv = capi.act(upw, 8, c1) if j == 1 else None
        capi.check(L.yb200_bn_silu_bwd(ctypes.byref(zv), ctypes.byref(dav), None, ctypes.byref(upv) if upv is not None else None,
                                       capi.ptr(scale), capi.ptr(shift), capi.ptr(mean32), capi.ptr(invstd32), _p(acc_g, run[j]),
                                       _p(acc_b, run[j]), ctypes.byref(dzv), None, None, accumulate, capi.stream_ptr()), "bn_silu_bwd")
        d = daw[..., o:o + c].reshape(P, c).double()
        d_abs, d_adds = d.abs(), 0
        if j == 1:  # + the 2x2 sum-pool of the upsampled gradient: four fp32 additions
            up = upw[..., 8:8 + c].double().view(n, h, 2, w, 2, c)
            d = d + up.sum((2, 4)).reshape(P, c)
            d_abs, d_adds = d_abs + up.abs().sum((2, 4)).reshape(P, c), 4
        refs.append(_bwd_ref(z, d, d_abs, d_adds, scale, shift, mean32, invstd32, _red_path(c, P)))
    torch.cuda.synchronize()
    name = _bwd_id(case)
    acc_g_k, acc_b_k = acc_g.clone(), acc_b.clone()
    for j, (o, c) in enumerate(zip(offs, cs)):
        r = refs[j]
        dz = dzw[..., o:o + c].reshape(P, c).double()
        _fail(f"{name} layer {j}", "dz", (dz - r["dz"]).abs(), r["tol_dz"])
        _fail(f"{name} layer {j}", "acc_dgamma", (acc_g_k[run[j]:run[j] + c] - r["dg"]).abs(), r["e_dg"])
        _fail(f"{name} layer {j}", "acc_dbeta", (acc_b_k[run[j]:run[j] + c] - r["db"]).abs(), r["e_db"])
        if sweep and j != 1:
            # where |da| >= 1 (and no upsampled gradient) dz = s du + mean terms much smaller than s du: |dz - ref| / |s da| is the SiLU'
            # error plus dz's bf16 rounding (2^-8 |SiLU'|)
            s = consts[j][0].double()
            dd = daw[..., o:o + c].reshape(P, c).double()
            sel = dd.abs() >= 1
            ratio = ((dz - r["dz"]).abs() / (s * dd).abs())[sel]
            bound = ((1 + r["u"] - 2 * r["u"] * r["sg"]).abs() * D_SIG + U_BF16 * r["g"].abs())[sel]
            print(f"\nlayer {j}: SiLU' over u in [{float(r['u'][sel].min()):.1f}, {float(r['u'][sel].max()):.1f}]: worst |dz - ref| / |s da| = "
                  f"{float(ratio.max()):.3g}, worst ratio to |1 + u - 2 u sig| 2^-12 + 2^-8 |SiLU'| = {float((ratio / bound).max()):.3g}; "
                  f"worst dz error / its bound = {float(((dz - r['dz']).abs() / r['tol_dz']).max()):.3g}")
    assert torch.isnan(dzw[..., :8]).all() and all(torch.isnan(dzw[..., o + c:o + c + 8]).all() for o, c in zip(offs, cs)), \
        "dz written outside the layers' slices"
    # param grads: layer j's gamma at base_j + i, beta at base_j + c_j + i, 4 floats of padding after every layer (engine layout)
    g_off, b_off, base = [], [], 4
    for c in cs:
        g_off.append(torch.arange(base, base + c))
        b_off.append(torch.arange(base + c, base + 2 * c))
        base += 2 * c + 4
    g_off, b_off = torch.cat(g_off).int().to(cuda), torch.cat(b_off).int().to(cuda)
    gb = torch.randn(base + 8, generator=g).to(cuda)
    gb0 = gb.clone()
    capi.check(L.yb200_bn_param_grads(_p(acc_g, 8), _p(acc_b, 8), ctot, capi.ptr(g_off), capi.ptr(b_off), capi.ptr(gb), accumulate,
                                      capi.stream_ptr()), "bn_param_grads")
    torch.cuda.synchronize()
    assert (acc_g == 0).all() and (acc_b == 0).all(), "the accumulators are not zero after bn_param_grads"
    for j, c in enumerate(cs):
        r, ro = refs[j], run[j] - 8
        gi, bi = g_off[ro:ro + c].long(), b_off[ro:ro + c].long()
        # fp32(acc): the accumulator's own error is bounded by e_dg / e_db above
        _check_param(f"{name} layer {j}", "dgamma", gb[gi], r["dg"], r["e_dg"], gb0[gi] if accumulate else None)
        _check_param(f"{name} layer {j}", "dbeta", gb[bi], r["db"], r["e_db"], gb0[bi] if accumulate else None)
    untouched = torch.ones(gb.numel(), dtype=torch.bool, device=cuda)
    untouched[g_off.long()] = False
    untouched[b_off.long()] = False
    assert torch.equal(gb[untouched], gb0[untouched]), "bn_param_grads wrote outside its offset table"


def test_bn_kernels_refuse_2056_channels(cuda):
    """257 channel vectors do not fit the 256-thread block: both kernels refuse, neither launches"""
    from yolov7_d2_b200 import capi

    L = capi.lib()
    c = 2056
    z = torch.zeros(1, 2, 2, c, dtype=torch.float16, device=cuda)
    a = torch.zeros(1, 2, 2, c, dtype=torch.bfloat16, device=cuda)
    v = torch.zeros(c, device=cuda)
    s64 = torch.zeros(c, dtype=torch.float64, device=cuda)
    zv, av = capi.act(z), capi.act(a)
    rc = _train_apply(L, capi, zv, s64, s64, 4, v, v, capi.ptr(v), capi.ptr(v), [v, v, v, v], None, av, None)
    assert rc == capi.ERR_UNSUPPORTED, rc
    rc = L.yb200_bn_silu_bwd(ctypes.byref(zv), ctypes.byref(av), None, None, capi.ptr(v), capi.ptr(v), capi.ptr(v), capi.ptr(v), capi.ptr(s64),
                             capi.ptr(s64), ctypes.byref(av), None, None, 0, capi.stream_ptr())
    assert rc == capi.ERR_UNSUPPORTED, rc


# ------------------------------------------------------------------------------------------------ head bias gradients

@pytest.mark.parametrize("ch", [85, 6, 205], ids=["nc80", "nc1", "two_blocks"])
def test_head_bias_grad_exact(cuda, ch):
    """reg[4] / obj[1] / cls[nc] = fp32(bias_acc[level]) (or the previous value plus it, one fp32 addition): bit for bit.  Only that
    level's row of bias_acc is re-zeroed."""
    from yolov7_d2_b200 import capi

    L = capi.lib()
    g = torch.Generator().manual_seed(ch)
    acc0 = torch.randn(3, ch, dtype=torch.float64, generator=g) * 100
    for level in range(3):
        for accumulate in (0, 1):
            acc = acc0.to(cuda)
            gw = torch.randn(8 + 4 + 8 + 1 + 8 + ch - 5 + 8, generator=g).to(cuda)  # reg | obj | cls slices of one buffer, gaps between
            gw0 = gw.clone()
            capi.check(L.yb200_head_bias_grad(capi.ptr(acc), 3, ch, level, _p(gw, 8), _p(gw, 20), _p(gw, 29), accumulate, capi.stream_ptr()),
                       "head_bias_grad")
            torch.cuda.synchronize()
            v = acc0[level].float().to(cuda)
            exp = gw0.clone()
            for sl, cols in ((slice(8, 12), slice(0, 4)), (slice(20, 21), slice(4, 5)), (slice(29, 29 + ch - 5), slice(5, ch))):
                exp[sl] = gw0[sl] + v[cols] if accumulate else v[cols]
            assert torch.equal(gw, exp), f"level {level} accumulate {accumulate}: {(gw - exp).abs().max()}"
            assert (acc[level] == 0).all(), "the level's row is not re-zeroed"
            others = [i for i in range(3) if i != level]
            assert torch.equal(acc[others], acc0[others].to(cuda)), "another level's row changed"


# ------------------------------------------------------------------------------------------------ batched weight packing

def _pack_single(capi, d, ref_fwd, ref_dgrad):
    capi.check(capi.lib().yb200_pack_conv_weight(ctypes.c_void_p(d.w_oihw), d.cout, d.cin, d.ksize, d.cout_pad, d.cin_pad,
                                                 capi.ptr(ref_fwd), capi.ptr(ref_dgrad), capi.stream_ptr()), "pack_conv_weight")


def _nan_fill(t):
    t.view(torch.int16).fill_(0x7FC1)  # a bf16 NaN: a padding entry the batched pack leaves unwritten fails the comparison


def _compare_batched(capi, descs, outs, cuda):
    """outs[i] = (w_fwd tensor or None, w_dgrad tensor or None) of descs[i], filled by the batched pack: equal to one
    yb200_pack_conv_weight per layer, bit for bit"""
    for i, (d, (wf, wd)) in enumerate(zip(descs, outs)):
        kk = d.ksize * d.ksize
        rf = torch.empty(d.cout_pad, kk, d.cin_pad, dtype=torch.bfloat16, device=cuda)
        rd = torch.empty(d.cin_pad, kk, d.cout_pad, dtype=torch.bfloat16, device=cuda)
        _nan_fill(rf)
        _nan_fill(rd)
        _pack_single(capi, d, rf, rd)
        torch.cuda.synchronize()
        desc = f"layer {i}: cout {d.cout}/{d.cout_pad} cin {d.cin}/{d.cin_pad} k {d.ksize}"
        if wf is not None:
            assert torch.equal(wf.view(torch.int16).reshape(-1), rf.view(torch.int16).reshape(-1)), "w_fwd differs, " + desc
        if wd is not None:
            assert torch.equal(wd.view(torch.int16).reshape(-1), rd.view(torch.int16).reshape(-1)), "w_dgrad differs, " + desc


def test_pack_weights_batched_synthetic_table(cuda):
    """256 layers (the most one launch takes): w_fwd-only and w_dgrad-only layers, cout and cin padding, k = 1 and 3; 257 are refused"""
    from yolov7_d2_b200 import capi

    L = capi.lib()
    g = torch.Generator().manual_seed(5)
    descs, outs, keep = [], [], []
    prefix = [0]
    for i in range(257):
        k = 1 if i % 2 else 3
        cout, cin = int(torch.randint(1, 48, (1,), generator=g)), int(torch.randint(1, 48, (1,), generator=g))
        cop = cout + (0 if i % 4 == 0 else int(torch.randint(0, 17, (1,), generator=g)))
        cip = cin + (0 if i % 4 == 1 else int(torch.randint(0, 17, (1,), generator=g)))
        mode = i % 3   # 0: forward operand only, 1: data-gradient operand only, 2: both
        w = torch.randn(cout, cin, k, k, generator=g).to(cuda)
        wf = torch.empty(cop, k * k, cip, dtype=torch.bfloat16, device=cuda) if mode != 1 else None
        wd = torch.empty(cip, k * k, cop, dtype=torch.bfloat16, device=cuda) if mode != 0 else None
        for t in (wf, wd):
            if t is not None:
                _nan_fill(t)
        d = capi.PackDesc()
        d.w_oihw, d.w_fwd, d.w_dgrad = w.data_ptr(), wf.data_ptr() if wf is not None else None, wd.data_ptr() if wd is not None else None
        d.cout, d.cin, d.ksize, d.cout_pad, d.cin_pad = cout, cin, k, cop, cip
        descs.append(d)
        outs.append((wf, wd))
        keep.append(w)
        prefix.append(prefix[-1] + cop * k * k * cip)
    assert any(d.cin_pad > d.cin and d.w_fwd for d in descs[:256]) and any(d.cin_pad > d.cin and d.w_dgrad for d in descs[:256])
    arr = (capi.PackDesc * 257)(*descs)
    raw = torch.frombuffer(bytearray(bytes(arr)), dtype=torch.uint8).to(cuda)
    pre = torch.tensor(prefix, dtype=torch.int64, device=cuda)
    rc = L.yb200_pack_conv_weights_batched(capi.ptr(raw), capi.ptr(pre), 257, ctypes.c_int64(prefix[257]), capi.stream_ptr())
    assert rc == capi.ERR_INVALID, "257 layers must be refused"
    capi.check(L.yb200_pack_conv_weights_batched(capi.ptr(raw), capi.ptr(pre), 256, ctypes.c_int64(prefix[256]), capi.stream_ptr()),
               "pack_conv_weights_batched")
    torch.cuda.synchronize()
    _compare_batched(capi, descs[:256], outs[:256], cuda)
    assert all(t is None or bool((t.view(torch.int16) == 0x7FC1).all()) for t in outs[256]), "the refused call wrote"


# ------------------------------------------------------------------------------------------------ every BatchNorm of a real step

def build_step(cuda, batch, size):
    """YOLOX-s at batch x size^2 after one train_step(), non-trivial BatchNorm affine parameters and running statistics.  Snapshots of
    what a second step changes (running statistics, gradients) are kept, so the checks do not depend on each other's order."""
    from yolov7_d2_b200.engine import YoloxEngine

    sd = orc.yolox_state_dict(3)
    g = torch.Generator().manual_seed(9)
    for k in sd:
        if k.endswith(".bn.weight"):
            sd[k] = torch.rand(sd[k].shape, generator=g) * 0.5 + 0.75
        if k.endswith(".bn.bias"):
            sd[k] = torch.randn(sd[k].shape, generator=g) * 0.1
        if k.endswith(".bn.running_mean"):
            sd[k] = torch.randn(sd[k].shape, generator=g) * 0.2
        if k.endswith(".bn.running_var"):
            sd[k] = torch.rand(sd[k].shape, generator=g) + 0.5
    images, labels = orc.synthetic_batch(batch, size, 5, max_gt=6, empty_every=4)
    eng = YoloxEngine(batch, size, size, device=cuda)
    eng.load_state_dict(sd)
    eng.images_u8.copy_(images.to(cuda))
    eng.labels.copy_(labels.to(cuda))
    eng.train_step()
    torch.cuda.synchronize()
    return dict(eng=eng, sd=sd, rm=eng.flat_rm.clone(), rv=eng.flat_rv.clone(), grad=eng.flat_grad.clone(), stats=eng.flat_stats.clone(),
                images=images, labels=labels)


@pytest.fixture(scope="module")
def step(cuda):
    return build_step(cuda, 8, 256)


def _heads(eng):
    from yolov7_d2_b200.engine import ConvOp

    for op in eng.ops:
        if isinstance(op, ConvOp):
            for hd in op.heads:
                yield op, hd


def _layer_refs(eng, op, hd, stats):
    """fp64 references of one BatchNorm layer of the step just run, from the operands the engine passed"""
    nb, o, c = eng.nbn, hd.bn_off, hd.c
    zb = op.z.buf
    n, h, w = zb.n, zb.h, zb.w
    P = n * h * w
    z = zb.view(hd.c0, c).tensor().reshape(P, c).double()   # the stem too: its BatchNorm reads the plain [n, h, w, 32] view
    d = hd.out.grad_tensor().reshape(P, c).double()
    d_abs, d_adds = d.abs(), 0
    if hd.up is not None:
        up = hd.up.grad_tensor().double().reshape(n, h, 2, w, 2, c)
        d = d + up.sum((2, 4)).reshape(P, c)
        d_abs, d_adds = d_abs + up.abs().sum((2, 4)).reshape(P, c), 4
    sl = slice(o, o + c)
    consts = (eng.flat_scale[sl], eng.flat_shift[sl], eng.flat_mean[sl], eng.flat_invstd[sl])
    return z, P, (stats[o:o + c], stats[nb + o:nb + o + c]), consts, _bwd_ref(z, d, d_abs, d_adds, *consts, _red_path(c, P))


def _all_tiles(eng, op):
    """every 128-pixel tile of the layer's output grid (the stem's tiles cover its [n, h, w / 4] grouped grid): a bound on the tiles
    one CTA walks"""
    zb = op.z.buf
    return _choose_tile(zb.n, zb.h, zb.w // 4) if (op.first and eng.group4) else _choose_tile(zb.n, zb.h, zb.w)


def check_every_batchnorm(step, tiles_per_cta=_all_tiles, layers=None):
    """For every BatchNorm of the step (or those named in `layers`): the convolution epilogue's sums of the stored z, the published
    constants, the running statistics against the loaded ones, the activation (+ residual, + upsampled copy), dz, and the weight / bias
    gradients at the per-head parameter (gamma offset by hd.c0, bn_goff / bn_boff).  tiles_per_cta(eng, op): the most tiles one CTA
    of the layer's forward walks."""
    eng, sd = step["eng"], step["sd"]
    for op, hd in _heads(eng):
        name = hd.prefix
        if layers is not None and name not in layers:
            continue
        z, P, (S, Q), (scale, shift, mean_k, invstd_k), r = _layer_refs(eng, op, hd, step["stats"])
        c = hd.c
        # sums: fp32 per warp (32 pixels, 5 butterfly levels), one addition per 128-pixel tile the CTA walks, two levels for the four
        # 32-pixel quadrants, fp64 atomics (negligible); squares round once more
        k = 5 + tiles_per_cta(eng, op) + 2
        _fail(name, "stat_sum", (S - z.sum(0)).abs(), k * U32 * z.abs().sum(0))
        _fail(name, "stat_sqsum", (Q - (z * z).sum(0)).abs(), (k + 1) * U32 * (z * z).sum(0))
        gamma, beta = eng.params[name + ".bn.weight"], eng.params[name + ".bn.bias"]
        mean, var = _check_stats(name, S, Q, P, gamma, beta, mean_k, invstd_k, scale, shift)
        _check_running(name, sd[name + ".bn.running_mean"].to(z.device), sd[name + ".bn.running_var"].to(z.device), mean, var, P,
                       step["rm"][hd.bn_off:hd.bn_off + c], step["rv"][hd.bn_off:hd.bn_off + c], 1)
        out = hd.out.tensor()
        res = hd.residual.tensor().reshape(P, c).double() if hd.residual is not None else None
        _check_apply(name, z, scale, shift, out.reshape(P, c), res)
        if hd.up is not None:
            assert torch.equal(hd.up.tensor(), out.repeat_interleave(2, 1).repeat_interleave(2, 2)), f"{name}: upsampled copy"
        dz = eng._dz[id(op)].view(hd.c0, c).tensor().reshape(P, c).double()
        _fail(name, "dz", (dz - r["dz"]).abs(), r["tol_dz"])
        gofs = (eng.grads[name + ".bn.weight"].data_ptr() - eng.flat_grad.data_ptr()) // 4
        bofs = (eng.grads[name + ".bn.bias"].data_ptr() - eng.flat_grad.data_ptr()) // 4
        _check_param(name, "bn.weight grad", step["grad"][gofs:gofs + c], r["dg"], r["e_dg"])
        _check_param(name, "bn.bias grad", step["grad"][bofs:bofs + c], r["db"], r["e_db"])
        del z, r


def test_step_every_batchnorm_against_fp64(step):
    eng = step["eng"]
    nb = eng.nbn
    check_every_batchnorm(step)
    assert (step["stats"][2 * nb:] == 0).all(), "the dgamma / dbeta accumulators are not zero after backward"
    _check_head_bias(eng, step["grad"], None)
    hc = eng.hc
    for name, off, numel in eng.param_layout:
        if name.startswith("head.obj_preds") and name.endswith(".weight"):
            assert (step["grad"][off + numel:off + numel + 11 * hc] == 0).all(), f"padding rows after {name} are not zero"


def _check_head_bias(eng, flat_grad, prev):
    """prediction biases: Σ over anchors of the fp32 loss gradients, summed in fp32 tiles of at most 128 anchors (127 additions) and
    fp64 across tiles.  The stored d_cls / d_ro hold those gradients rounded to bf16 (2^-8 each), so against their fp64 sums the bound
    is (2^-8 + 127 * 2^-24) Σ|d| + one fp32 rounding (two with accumulate)."""
    base = eng.flat_grad.data_ptr()
    for k in range(len(eng.levels)):
        dc = eng.d_cls[k].double().sum((0, 1, 2))
        dca = eng.d_cls[k].double().abs().sum((0, 1, 2))
        dro = eng.d_ro[k][..., :5].double().sum((0, 1, 2))
        droa = eng.d_ro[k][..., :5].double().abs().sum((0, 1, 2))
        for leaf, ref, mag in (("cls_preds", dc, dca), ("reg_preds", dro[:4], droa[:4]), ("obj_preds", dro[4:], droa[4:])):
            name = f"head.{leaf}.{k}.bias"
            o = (eng.grads[name].data_ptr() - base) // 4
            got = flat_grad[o:o + ref.numel()]
            tol = (U_BF16 + 127 * U32) * mag
            _check_param(name, "gradient", got, ref, tol, prev[o:o + ref.numel()] if prev is not None else None)


def test_step_accumulated_gradients(step):
    """a second step with accumulate=True: BatchNorm and prediction-bias gradients = fp32 sum of the first step's values and the second
    step's fp64 references"""
    eng = step["eng"]
    prev = step["grad"]
    eng.train_step(accumulate=True)
    torch.cuda.synchronize()
    for op, hd in _heads(eng):
        name = hd.prefix
        _, _, _, _, r = _layer_refs(eng, op, hd, eng.flat_stats)
        for leaf, ref, e in ((".bn.weight", r["dg"], r["e_dg"]), (".bn.bias", r["db"], r["e_db"])):
            o = (eng.grads[name + leaf].data_ptr() - eng.flat_grad.data_ptr()) // 4
            _check_param(name, leaf + " grad (accumulated)", eng.flat_grad[o:o + hd.c], ref, e, prev[o:o + hd.c])
    _check_head_bias(eng, eng.flat_grad, prev)
    assert (eng.flat_stats[2 * eng.nbn:] == 0).all()


def test_pack_weights_batched_real_table(step, cuda):
    """the engine's own table: every convolution, the prediction rows (cout 5 -> 16 and 80) and the stem with no data-gradient operand"""
    from yolov7_d2_b200 import capi

    eng = step["eng"]
    raw, _, n, _, _ = eng._pack_table
    descs = list((capi.PackDesc * n).from_buffer_copy(bytes(raw.cpu().numpy())))
    by_ptr = {}
    for op in eng.ops:
        for attr in ("w_fwd", "w_dgrad", "wc_fwd", "wc_dgrad", "wr_fwd", "wr_dgrad"):
            t = getattr(op, attr, None)
            if t is not None:
                by_ptr[t.data_ptr()] = t
    assert any(d.cout == 5 and d.cout_pad == 16 for d in descs) and any(d.cout == 80 for d in descs)
    assert not descs[0].w_dgrad and descs[0].w_fwd == eng.ops[0].w_fwd.data_ptr()
    outs = [(by_ptr[d.w_fwd] if d.w_fwd else None, by_ptr[d.w_dgrad] if d.w_dgrad else None) for d in descs]
    for t in by_ptr.values():
        _nan_fill(t)
    eng.pack_weights()
    torch.cuda.synchronize()
    _compare_batched(capi, descs, outs, cuda)
