"""The DETR transformer's kernels, call by call, against fp64 at DETR-R50's sizes: d_model 256, 8 heads of 32, FFN 2048, dropout 0.1,
100 / 300 queries and a 25 x 42 = 1050-token memory (an 800 x 1333 image at stride 32).

tests/test_detr_gpu.py checks the layers end to end at small sizes; this module checks every kernel the layers and the DETR heads call, on
the geometries they call it with, each against a plain fp64 computation on exactly the operands the kernel read.

A. Recordings.  A stand-in for the library handle of every `_Kernels` instance records each call (entry point, arguments, return code)
   and forwards it, during (1) one training step of Transformer(256, 8, 6, 6, 2048, dropout 0.1, return_intermediate_dec) at B = 2 on a
   25 x 42 map with 100 queries -- image 0 unpadded, image 1 valid on 19 x 31, padded right and bottom as ImageList pads it -- with the
   DETR tail through `_linear_stack` (input_proj 2048 -> 256, class_embed 256 -> 81, bbox MLP 256 -> 256 -> 256 -> 4), (2) one decoder
   layer training step at 300 queries, (3) a no-grad forward of one encoder and one decoder layer (null lse, null LayerNorm statistics).
B. Each distinct geometry is replayed on fresh buffers with the conventions of tests/test_convnext_plan_gpu.py: input channels outside a
   view hold 2^14, output bits outside a view must not change, outputs inside a view start as NaN and must end finite.  The GEMMs use that
   module's bound; the rest is judged as stated in each replay's docstring.
C. The attention core at the shipped and benchmarked shapes, forward and backward, p = 0 and p = 0.1, with 2-D padding masks.

The attention bound.  Per (image, head) with s = scale * q k^T on the bf16 q / k, P = softmax(s) over the live keys, F the dropout
multiplier (0 or 1 / (1 - p), oracle/detr_oracle.py), A = P o F, U = 2^-24 and c(K) = 16 sqrt(K) + 16 as in the plan module:

  score error   the kernel's fp32 score differs from s by <= c(32) U scale sum_d |q_d||k_d| (the wgmma over 32 products); the exponent
                of ex2 is then formed with two fp32 roundings (scale * log2 e, the FMA with the running maximum or lse): <= 3 U (|s| + m),
                m = max_j |s_j| of the row (forward) or |lse| (backward).  An exponent error d moves p by the factor e^d.
  ex2           ex2.approx.ftz.f32: "maximum relative error 2 ulp across the full range" (PTX ISA, ex2), <= 2^-22; results below 2^-126
                flush to zero, an absolute error far below every other term.
  forward       o = A v.  With rho = the row's largest exponent error + 2^-22, the numerator's p and the normaliser l are each within
                rho (relative), so o moves by <= 2 rho mag, mag = A |v|.  The bf16 P tile adds <= 2^-8 mag (inner rounding: P~ feeds the
                P V wgmma).  Each 128-key tile rescales acc and l by one alpha = ex2(m_old - m_new); acc and l share the same alpha, so only
                the two products round, but we charge (2^-22 + 2 U) mag per tile.  fp32 accumulation of Lk terms (and l): c(Lk) U mag.
                The bf16 store: 2^-8 |o|.
                    bound_o = 2^-8 |o| + (2^-8 + 2 rho + tiles (2^-22 + 2 U) + c(Lk) U) mag
  lse           (m + log2f(l)) ln 2 in fp32, an absolute bound: rho + c(Lk) U (the relative error of l) + 2^-20 (log2f, 1 ulp of a value
                below 16) + 2 U (|m log2 e| + 16) + 2 U |lse|.
  backward      judged on its own, not through the forward: P = exp(s - lse) with the lse the kernel was given, D = rowsum(dO o O) of the
                bf16 O it was given.  eta = exponent error + 2^-22 per element.
                    dV = A^T dO:  2^-8 |dV| + 2^-8 mag + (eta o A)^T |dO| + c(Lq) U mag,  mag = A^T |dO|
                dS = P o (F o dP - D) scale with dP = dO v^T (fp32 over 32 products: c(32) U |dO||v|^T), D in fp32 (c(32) U sum |dO o O|),
                four fp32 roundings (4 U (|F dP| + |D|)) and the bf16 tile (2^-8 |dS|):
                    tau = 2^-8 |dS| + scale P (eta |F dP - D| + F c(32) U |dO||v|^T + c(32) U sum|dO o O| + 4 U (|F dP| + |D|))
                    dQ = dS k:    2^-8 |dQ| + tau |k| + c(Lk) U |dS| |k|
                    dK = dS^T q:  2^-8 |dK| + tau^T |q| + c(Lq) U |dS|^T |q|
                A masked key has P = 0 in every term, so its dK and dV must be exactly zero.

tests/test_detr_kernels_tol_cpu.py shows on the CPU that a faithful fp32 / bf16 emulation of the kernels passes these bounds and that a
dropped key tile, an ignored mask, a misread lse, a wrong normaliser, misplaced dropout, a neighbouring row's D or a neighbouring head's q
fail them, as does a LayerNorm with the unbiased variance (the rstd bound).
"""
import ctypes
import math

import pytest
import torch
import torch.nn as nn

from test_convnext_plan_gpu import (R_BF16, U, WORST, _act, _g, _geo, _given, _guard_ok, _guarded, _in_view, _lib, _out_view, _outside_same,
                                    _sl, _weights, acc_c, bound, check, conv_ref, dgrad_ref, run_affine, run_dgrad, run_wgrad)
from test_sparseinst_kernels_gpu import colsum_ref, run_pack

pytestmark = pytest.mark.gpu

EX2 = 2.0 ** -22      # ex2.approx.ftz.f32, PTX ISA: 2 ulp
LOG2E = 1.4426950408889634
TILE = 128            # keys per step of the attention kernels
SCALE = float(torch.tensor(32 ** -0.5, dtype=torch.float32))  # the fp32 softmax scale the layers pass
LN_EPS = float(torch.tensor(1e-5, dtype=torch.float32))
MAP = (25, 42)        # the stride-32 map of an 800 x 1333 image
VALID = [(25, 42), (19, 31), (1, 1), (25, 20), (6, 42), (13, 37), (25, 1), (20, 42)]  # valid (h, w) of the batch's images, cycled
SENT_KV = 64.0        # masked keys' k and v are scaled by this: a masked key that is read is a gross error


# ------------------------------------------------------------------------------------------------------------------------------------
# fp64 references of the attention core (also used on the CPU by tests/test_detr_kernels_tol_cpu.py)
# ------------------------------------------------------------------------------------------------------------------------------------
def attn_fwd_ref(q, k, v, dead, scale, mult=None):
    """q [H, Lq, 32], k / v [H, Lk, 32] (fp64 copies of the bf16 operands), dead [Lk] bool, mult [H, Lq, Lk] or None ->
    (o, bound of o, lse, bound of lse); every row has a live key"""
    s = scale * (q @ k.transpose(-1, -2))
    sa = scale * (q.abs() @ k.abs().transpose(-1, -2))
    s = s.masked_fill(dead, -math.inf)
    live = ~dead
    smax = torch.where(live, s.abs(), torch.zeros_like(s)).amax(-1, keepdim=True)
    mx = s.amax(-1, keepdim=True)
    lse = mx + torch.log(torch.exp(s - mx).sum(-1, keepdim=True))
    p = torch.exp(s - lse)
    a = p if mult is None else p * mult
    o, mag = a @ v, a @ v.abs()
    dexp = acc_c(32) * U * sa + 3 * U * (torch.where(live, s.abs(), torch.zeros_like(s)) + smax)
    rho = torch.where(live, dexp, torch.zeros_like(dexp)).amax(-1, keepdim=True) + EX2
    tiles = -(-k.shape[-2] // TILE)
    rel = R_BF16 + 2 * rho + tiles * (EX2 + 2 * U) + acc_c(k.shape[-2]) * U
    bnd_o = R_BF16 * o.abs() + rel * mag
    lse = lse[..., 0]
    bnd_lse = rho[..., 0] + acc_c(k.shape[-2]) * U + 2.0 ** -20 + 2 * U * (smax[..., 0] * LOG2E + 16) + 2 * U * lse.abs()
    return o, bnd_o, lse, bnd_lse


def attn_bwd_ref(q, k, v, o, do, lse, dead, scale, mult=None):
    """the backward of the attention core on the kernel's own o and lse -> {name: (ref, bound)} for dq, dk, dv"""
    s = scale * (q @ k.transpose(-1, -2))
    sa = scale * (q.abs() @ k.abs().transpose(-1, -2))
    live = (~dead).expand_as(s)
    p = torch.where(live, torch.exp(s - lse[..., None]), torch.zeros_like(s))
    f = torch.ones_like(s) if mult is None else mult
    a = p * f
    eta = torch.where(live, acc_c(32) * U * sa + 3 * U * (s.abs() + lse.abs()[..., None]) + EX2, torch.zeros_like(s))
    dv = a.transpose(-1, -2) @ do
    mdv = a.transpose(-1, -2) @ do.abs()
    bdv = R_BF16 * dv.abs() + (R_BF16 + acc_c(q.shape[-2]) * U) * mdv + (eta * a).transpose(-1, -2) @ do.abs()
    g = do @ v.transpose(-1, -2)
    ga = do.abs() @ v.abs().transpose(-1, -2)
    d = (do * o).sum(-1, keepdim=True)
    da = (do * o).abs().sum(-1, keepdim=True)
    fg = f * g
    ds = p * (fg - d) * scale
    tau = R_BF16 * ds.abs() + scale * p * (eta * (fg - d).abs() + f * acc_c(32) * U * ga + acc_c(32) * U * da + 4 * U * (fg.abs() + d.abs()))
    dq = ds @ k
    bdq = R_BF16 * dq.abs() + tau @ k.abs() + acc_c(k.shape[-2]) * U * (ds.abs() @ k.abs())
    dk = ds.transpose(-1, -2) @ q
    bdk = R_BF16 * dk.abs() + tau.transpose(-1, -2) @ q.abs() + acc_c(q.shape[-2]) * U * (ds.abs().transpose(-1, -2) @ q.abs())
    return dict(dq=(dq, bdq), dk=(dk, bdk), dv=(dv, bdv))


def ln_ref(x, gamma, beta, eps):
    """LayerNorm over the last dimension of fp64 rows x [R, C] -> y, its bound, mean and rstd with their bounds.
    The kernel sums in fp32 (two passes: the mean, then sum (x - mean)^2) and takes rsqrtf (2 ulp).  With the mean's error
    dm <= c(C) U mean|x| + U |mean|, sum (x - mean - dm)^2 = sum (x - mean)^2 + C dm^2 (the cross term vanishes), so
        |var~ - var| <= dm^2 + (c(C) + 3) U (var + dm^2),   rstd relative error <= |var~ - var| / (2 (var + eps)) + 2^-22 + U.
    y = ((x - mean~) rstd~) gamma + beta carries both: |gamma| (dm rstd + |x - mean| rstd drs) + 4 U (|gamma xhat| + |beta|), then bf16."""
    c = x.shape[-1]
    mean = x.mean(-1, keepdim=True)
    var = ((x - mean) ** 2).mean(-1, keepdim=True)
    rstd = (var + eps).rsqrt()
    xh = (x - mean) * rstd
    y = xh * gamma + beta
    dm = acc_c(c) * U * x.abs().mean(-1, keepdim=True) + U * mean.abs()
    dvar = dm * dm + (acc_c(c) + 3) * U * (var + dm * dm)
    drs = dvar / (2 * (var + eps)) + EX2 + U
    by = R_BF16 * y.abs() + gamma.abs() * (dm * rstd + (x - mean).abs() * rstd * drs) * 1.01 + 4 * U * (gamma.abs() * xh.abs() + beta.abs())
    return y, by, mean[:, 0], dm[:, 0], rstd[:, 0], (drs * rstd)[:, 0]


# ------------------------------------------------------------------------------------------------------------------------------------
# masks and buffers of the attention core
# ------------------------------------------------------------------------------------------------------------------------------------
def padding_mask(b, lk, dev):
    """uint8 [B, Lk], 1 = padding: at Lk = 25 x 42 image i is valid on VALID[i % 8] (image 0 unpadded, image 1 valid on 19 x 31, image 2
    only on key 0 -- key tiles 1-8 fully masked), padded right and bottom as ImageList pads a batch; other lengths: image i's last i * Lk / 8
    keys"""
    m = torch.zeros(b, lk, dtype=torch.uint8)
    for i in range(b):
        if lk == MAP[0] * MAP[1]:
            vh, vw = VALID[i % len(VALID)]
            mi = torch.ones(MAP, dtype=torch.uint8)
            mi[:vh, :vw] = 0
            m[i] = mi.flatten()
        else:
            m[i, lk - (i % 8) * lk // 8:] = 1
            m[i, 0] = 0
    return m.to(dev)


def _tok(b, l, pitch, g, scale=1.0):
    return (torch.randn(b, 1, l, pitch, generator=g, device="cuda") * scale).to(torch.bfloat16)


def _heads(t, geo):
    """[B][1][L][pitch] bf16 view -> fp64 [B, H, L, 32]"""
    b, _, l, c, _, off = geo
    return t[..., off:off + c].double().reshape(b, l, c // 32, 32).permute(0, 2, 1, 3)


def _attn_inputs(gq, gk, gv, masked, g):
    """q / k / v buffers of the views' pitches (channels outside the views: the 2^14 sentinel); q rows scaled by 1/4, 1 or 3 in turn (flat
    and peaked softmax rows); masked keys' k and v scaled by SENT_KV"""
    b, lq, lk = gq[0], gq[2], gk[2]
    mask = padding_mask(b, lk, "cuda") if masked else None
    bufs = {}
    for name, geo, ln in (("q", gq, lq), ("k", gk, lk), ("v", gv, lk)):
        key = (geo[4], ln)  # self-attention: q | k | v share one buffer, as in the layers
        t = bufs.get(key)
        if t is None:
            t = torch.full((b, 1, ln, geo[4]), 2.0 ** 14, dtype=torch.bfloat16, device="cuda")
            bufs[key] = t
        x = torch.randn(b, 1, ln, geo[3], generator=g, device="cuda")
        if name == "q":
            x = x * torch.tensor([0.25, 1.0, 3.0], device="cuda").repeat(ln // 3 + 1)[:ln, None]
        elif mask is not None:
            x = x * (1.0 + (SENT_KV - 1.0) * mask.float())[:, None, :, None]
        t[..., geo[5]:geo[5] + geo[3]] = x.to(torch.bfloat16)
    return bufs, mask


def _buf(bufs, geo, ln):
    return bufs[(geo[4], ln)]


def _attn_mult(p, seed, b, h, lq, lk):
    if p <= 0:
        return None
    from oracle import detr_oracle as dto

    return dto.attention_dropout_multiplier(seed, b, h, lq, lk, p, device="cuda")


def _out_buf(geo, ln, g):
    """bf16 [B][1][L][pitch]: random outside the view, NaN inside"""
    t = torch.randn(geo[0], 1, ln, geo[4], generator=g, device="cuda").to(torch.bfloat16)
    t[..., geo[5]:geo[5] + geo[3]] = float("nan")
    return t, t.clone()


def run_attention(gq, gk, gv, go, masked, p, lse=True, grads=None, seed=50):
    """yb200_attention_fwd_dropout [+ yb200_attention_bwd_dropout]: o and lse against attn_fwd_ref; with grads = (gdo, gdq, gdk, gdv) also
    dq / dk / dv against attn_bwd_ref on the kernel's own o and lse, exact zeros for every masked key's dk / dv, and a second backward
    that must give the same bits"""
    capi, L = _lib()
    g = _g(seed)
    b, lq, lk, e = gq[0], gq[2], gk[2], gq[3]
    h = e // 32
    bufs, mask = _attn_inputs(gq, gk, gv, masked, g)
    q, k, v = _buf(bufs, gq, lq), _buf(bufs, gk, lk), _buf(bufs, gv, lk)
    out, out0 = _out_buf(go, lq, g)
    lbuf, lv = _guarded((b, h, lq), float("nan")) if lse else (None, None)
    dseed = 0x2468ACE
    qa, ka, va, oa = _act(capi, q, gq), _act(capi, k, gk), _act(capi, v, gv), _act(capi, out, go)
    capi.check(L.yb200_attention_fwd_dropout(ctypes.byref(qa), ctypes.byref(ka), ctypes.byref(va), capi.ptr(mask), ctypes.c_float(SCALE), ctypes.byref(oa),
                                             capi.ptr(lv), ctypes.c_float(p), ctypes.c_uint32(dseed), capi.stream_ptr()), "attention_fwd_dropout")
    _outside_same(out, out0, (b, 1, lq, e, go[4], go[5]), "attention out")
    if lse:
        _guard_ok(lbuf, b * h * lq, "lse")
    mult = _attn_mult(p, dseed, b, h, lq, lk)
    dead = mask.bool() if masked else torch.zeros(b, lk, dtype=torch.bool, device="cuda")
    qd, kd, vd, od = _heads(q, gq), _heads(k, gk), _heads(v, gv), _heads(out, go)
    for i in range(b):
        mi = None if mult is None else mult[i].double()
        o_ref, bo, l_ref, bl = attn_fwd_ref(qd[i], kd[i], vd[i], dead[i], SCALE, mi)
        check("attention forward o (bf16)", od[i], o_ref, bo, f"image {i}: o")
        if lse:
            check("attention forward lse (fp32, absolute)", lv[i], l_ref, bl, f"image {i}: lse")
    if grads is None:
        return
    gdo, gdq, gdk, gdv = grads
    dbufs = {}
    dout = _tok(b, lq, gdo[4], g)
    ka_ = {}
    for name, geo, ln in (("dq", gdq, lq), ("dk", gdk, lk), ("dv", gdv, lk)):
        key = (geo[4], ln)
        if key not in dbufs:
            t = torch.randn(b, 1, ln, geo[4], generator=g, device="cuda").to(torch.bfloat16)
            dbufs[key] = t
        dbufs[key][..., geo[5]:geo[5] + geo[3]] = float("nan")
        ka_[name] = (dbufs[key], geo)
    before = {kk: t.clone() for kk, t in dbufs.items()}
    da = _act(capi, dout, gdo)
    dacts = [_act(capi, *ka_[n]) for n in ("dq", "dk", "dv")]
    ws = torch.empty(int(L.yb200_attention_bwd_workspace(ctypes.byref(qa))), dtype=torch.uint8, device="cuda")

    def bwd(acts):
        capi.check(L.yb200_attention_bwd_dropout(ctypes.byref(qa), ctypes.byref(ka), ctypes.byref(va), ctypes.byref(oa), ctypes.byref(da), capi.ptr(mask),
                                                 ctypes.c_float(SCALE), capi.ptr(lv), ctypes.byref(acts[0]), ctypes.byref(acts[1]), ctypes.byref(acts[2]),
                                                 capi.ptr(ws), ctypes.c_float(p), ctypes.c_uint32(dseed), capi.stream_ptr()), "attention_bwd_dropout")

    bwd(dacts)
    # every view of a gradient buffer written: the bits outside all of them must not change
    for key, t in dbufs.items():
        inside = torch.zeros(t.shape[-1], dtype=torch.bool, device="cuda")
        for n in ("dq", "dk", "dv"):
            bt, geo = ka_[n]
            if bt is t:
                inside[geo[5]:geo[5] + geo[3]] = True
        assert torch.equal(t[..., ~inside], before[key][..., ~inside]), "attention backward wrote outside its gradient views"
    got = {n: _heads(*ka_[n]) for n in ("dq", "dk", "dv")}
    dod = _heads(dout, gdo)
    for i in range(b):
        mi = None if mult is None else mult[i].double()
        refs = attn_bwd_ref(qd[i], kd[i], vd[i], od[i], dod[i], lv[i].double(), dead[i], SCALE, mi)
        for n, (r, bnd) in refs.items():
            check(f"attention backward {n} (bf16)", got[n][i], r, bnd, f"image {i}: {n}")
        if masked:
            for n in ("dk", "dv"):
                z = got[n][i][:, dead[i]]
                assert bool((z == 0).all()), f"image {i}: {n} of masked keys is not zero ({int((z != 0).sum())} elements, finite: {bool(z.isfinite().all())})"
    # the same call again: the same bits (no atomics)
    again = {kk: torch.full_like(t, float("nan")) for kk, t in dbufs.items()}
    for kk in again:
        again[kk].copy_(before[kk])
    acts2 = []
    for n in ("dq", "dk", "dv"):
        bt, geo = ka_[n]
        key = next(kk for kk, t in dbufs.items() if t is bt)
        acts2.append(_act(capi, again[key], geo))
    bwd(acts2)
    for kk in dbufs:
        assert torch.equal(again[kk], dbufs[kk]), "a repeated attention backward gives different bits"


# ------------------------------------------------------------------------------------------------------------------------------------
# B. replays of the kernels the plan module does not replay
# ------------------------------------------------------------------------------------------------------------------------------------
def run_pack2(cout, cin, k, cout_pad, cin_pad, dgrad, seed=51):
    """yb200_pack_conv_weight: the forward operand [cout_pad][k*k][cin_pad] (run_pack) and, with dgrad, also the data-gradient operand
    [cin_pad][k*k][cout_pad]: bf16 round to nearest even, padding rows / columns zero, nothing written past either"""
    run_pack(cout, cin, k, cout_pad, cin_pad, seed=seed)
    if not dgrad:
        return
    capi, L = _lib()
    g = _g(seed)
    w = torch.randn(cout, cin, k, k, generator=g, device="cuda") * 0.05
    n = cout_pad * k * k * cin_pad
    bf, wf = _guarded((cout_pad, k * k, cin_pad), float("nan"), torch.bfloat16)
    bd, wd = _guarded((cin_pad, k * k, cout_pad), float("nan"), torch.bfloat16)
    capi.check(L.yb200_pack_conv_weight(capi.ptr(w), cout, cin, k, cout_pad, cin_pad, capi.ptr(wf), capi.ptr(wd), capi.stream_ptr()), "pack_conv_weight")
    want = torch.zeros(cout_pad, k * k, cin_pad, dtype=torch.bfloat16, device="cuda")
    want[:cout, :, :cin] = w.permute(0, 2, 3, 1).reshape(cout, k * k, cin).to(torch.bfloat16)
    assert torch.equal(wf.view(torch.int16), want.view(torch.int16)), "forward operand differs from the bf16 rounding"
    assert torch.equal(wd.view(torch.int16), want.permute(2, 1, 0).contiguous().view(torch.int16)), \
        "data-gradient operand is not the transposed forward operand (padding included)"
    _guard_ok(bf, n, "forward operand")
    _guard_ok(bd, n, "data-gradient operand")


def run_linear_relu(gx, go, seed=52):
    """yb200_linear_relu_fwd: bf16(max(x W^T + b, 0)); ReLU is 1-Lipschitz, so the GEMM's bound carries over"""
    capi, L = _lib()
    g = _g(seed)
    x = _in_view(gx, g)
    cin, cout = gx[3], go[3]
    w, wf, _ = _weights(capi, L, cout, cin, 1, g, dgrad=False)
    b = torch.randn(cout, generator=g, device="cuda") * 0.5
    out, out0 = _out_view(go, g)
    xa, oa = _act(capi, x, gx), _act(capi, out, go)
    capi.check(L.yb200_linear_relu_fwd(ctypes.byref(xa), capi.ptr(wf), capi.ptr(b), ctypes.byref(oa), capi.stream_ptr()), "linear_relu_fwd")
    ref, mag, kk = conv_ref(_sl(x, gx).double(), w, 1, 1)
    ref, mag = (ref + b.double()).clamp_min(0.0), mag + b.double().abs()
    check("linear + ReLU (bf16)", _sl(out, go), ref, bound(ref, mag, kk, R_BF16), "h")
    _outside_same(out, out0, go, "h")


def run_dgrad_relu(gdz, gh, gdu, bias_sum=True, seed=53):
    """yb200_linear_dgrad_relu: du = bf16(h > 0 ? dz W : 0) -- h holds +-0, negatives and positives, as a dropped ReLU output and its
    sign tests see them -- and bias_grad_sum[c] += column sums of the STORED bf16 du (fp64 accumulator, already holding values)"""
    capi, L = _lib()
    g = _g(seed)
    dz = _in_view(gdz, g)
    h = _in_view(gh, g)
    hv = _sl(h, gh)
    hv[..., 0::5] = 0.0
    hv[..., 1::7] = -0.0
    c, hid = gdz[3], gdu[3]
    w, _, wd = _weights(capi, L, c, hid, 1, g)
    du, du0 = _out_view(gdu, g)
    a0 = torch.randn(hid, generator=g, device="cuda", dtype=torch.float64)
    sb, acc = _guarded((hid,), a0, torch.float64)
    dza, ha, dua = _act(capi, dz, gdz), _act(capi, h, gh), _act(capi, du, gdu)
    capi.check(L.yb200_linear_dgrad_relu(ctypes.byref(dza), capi.ptr(wd), ctypes.byref(ha), ctypes.byref(dua), capi.ptr(acc) if bias_sum else None,
                                         capi.stream_ptr()), "linear_dgrad_relu")
    d, mag, kk = dgrad_ref(_sl(dz, gdz).double(), w, 1, 1, (gdu[0], gdu[1], gdu[2], hid))
    on = (_sl(h, gh).float() > 0).double()
    check("linear dgrad + ReLU'", _sl(du, gdu), d * on, bound(d * on, mag * on, kk, R_BF16), "du")
    _outside_same(du, du0, gdu, "du")
    if bias_sum:
        dd = _sl(du, gdu).double().reshape(-1, hid)
        ref = a0 + dd.sum(0)
        check("linear dgrad + ReLU'", acc, ref, bound(ref, dd.abs().sum(0) + a0.abs(), dd.shape[0], 0.0), "bias-gradient sums of the stored du")
        _guard_ok(sb, hid, "bias-gradient sums")


def run_colsum(gx, scale, accumulate, seed=54):
    """yb200_colsum of a gradient (both signs): fp32 sums over every token, K = tokens"""
    capi, L = _lib()
    g = _g(seed)
    x = _in_view(gx, g)
    c = gx[3]
    o0 = torch.randn(c, generator=g, device="cuda")
    buf, out = _guarded((c,), o0 if accumulate else float("nan"))
    xa = _act(capi, x, gx)
    ws = torch.empty(max(16, L.yb200_colsum_workspace(ctypes.byref(xa))), dtype=torch.uint8, device="cuda")
    capi.check(L.yb200_colsum(ctypes.byref(xa), ctypes.c_float(scale), capi.ptr(out), accumulate, capi.ptr(ws), capi.stream_ptr()), "colsum")
    ref, mag, kk = colsum_ref(_sl(x, gx).double(), scale)
    if accumulate:
        ref, mag = ref + o0.double(), mag + o0.double().abs()
    check("column sums (fp32)", out, ref, bound(ref, mag, kk, 0.0), "sums")
    _guard_ok(buf, c, "sums")


def _ln_rows(gx, g):
    """LayerNorm input: N(0.5, 2^2) rows, and in turn rows with |mean| >> std (mean 64-200, std 1-2), constant rows (variance 0) and rows of
    variance below eps (std 2^-9)"""
    x = _in_view(gx, g, scale=2.0, shift=0.5)
    v = _sl(x, gx).reshape(-1, gx[3])
    r = v.shape[0]
    big = torch.rand(r, 1, generator=g, device="cuda") * 136 + 64
    v[1::4] = (torch.randn(v[1::4].shape, generator=g, device="cuda") * 1.5 + big[1::4]).to(torch.bfloat16)
    v[2::8] = (torch.full_like(v[2::8], 1.0) * big[2::8].floor()).to(torch.bfloat16)
    v[6::8] = (torch.randn(v[6::8].shape, generator=g, device="cuda") * 2.0 ** -9 + 0.25).to(torch.bfloat16)
    _sl(x, gx).copy_(v.view(_sl(x, gx).shape))
    return x


def run_ln_fwd(gx, gy, eps, stats, seed=55):
    """yb200_layernorm_fwd: bf16 y, and fp32 (mean, rstd) each against its own tight bound (ln_ref); the rstd bound is ~1e-5 relative, so
    the unbiased variance (a 1/510 change of rstd) cannot hide in it as it can under the bf16 rounding of y"""
    capi, L = _lib()
    g = _g(seed)
    x = _ln_rows(gx, g)
    c = gx[3]
    gamma = torch.rand(c, generator=g, device="cuda") + 0.5
    beta = torch.rand(c, generator=g, device="cuda") - 0.5
    y, y0 = _out_view(gy, g)
    rows = gx[0] * gx[1] * gx[2]
    sbuf, st = _guarded((rows, 2), float("nan")) if stats else (None, None)
    xa, ya = _act(capi, x, gx), _act(capi, y, gy)
    capi.check(L.yb200_layernorm_fwd(ctypes.byref(xa), capi.ptr(gamma), capi.ptr(beta), ctypes.c_float(eps), ctypes.byref(ya), capi.ptr(st),
                                     capi.stream_ptr()), "layernorm_fwd")
    xd = _sl(x, gx).double().reshape(-1, c)
    ref, by, mean, bm, rstd, br = ln_ref(xd, gamma.double(), beta.double(), float(torch.tensor(eps, dtype=torch.float32)))
    check("LayerNorm y (bf16)", _sl(y, gy).reshape(-1, c), ref, by, "y")
    _outside_same(y, y0, gy, "y")
    if stats:
        check("LayerNorm mean / rstd (fp32)", st[:, 0], mean, bm, "mean")
        check("LayerNorm mean / rstd (fp32)", st[:, 1], rstd, br, "rstd")
        _guard_ok(sbuf, 2 * rows, "statistics")


def run_ln_bwd(gdy, gx, gdx, addend, accumulate, seed=56):
    """yb200_layernorm_bwd on the statistics it is given (fp64 ones rounded to fp32): dx against fp64 on those statistics, grad gamma /
    beta (fp32 sums over every row) against fp64 sums; twice, the same bits"""
    capi, L = _lib()
    g = _g(seed)
    x = _ln_rows(gx, g)
    dy = _in_view(gdy, g)
    add = _in_view(addend, g) if addend else None
    c = gx[3]
    xd = _sl(x, gx).double().reshape(-1, c)
    eps = LN_EPS
    mean = xd.mean(-1)
    rstd = (((xd - mean[:, None]) ** 2).mean(-1) + eps).rsqrt()
    st = torch.stack([mean, rstd], -1).float().contiguous()
    gamma = torch.rand(c, generator=g, device="cuda") + 0.5
    g0 = torch.randn(2, c, generator=g, device="cuda")
    xa, da = _act(capi, x, gx), _act(capi, dy, gdy)
    aa = _act(capi, add, addend) if addend else None
    ws = torch.empty(max(16, L.yb200_layernorm_bwd_workspace(ctypes.byref(xa))), dtype=torch.uint8, device="cuda")
    runs = []
    for _ in range(2):
        dx, dx0 = _out_view(gdx, g)
        bg, gg = _guarded((c,), g0[0] if accumulate else float("nan"))
        bb, gb = _guarded((c,), g0[1] if accumulate else float("nan"))
        dxa = _act(capi, dx, gdx)
        capi.check(L.yb200_layernorm_bwd(ctypes.byref(da), ctypes.byref(xa), capi.ptr(st), capi.ptr(gamma), ctypes.byref(aa) if addend else None,
                                         ctypes.byref(dxa), capi.ptr(gg), capi.ptr(gb), accumulate, capi.ptr(ws), capi.stream_ptr()), "layernorm_bwd")
        _outside_same(dx, dx0, gdx, "dx")
        _guard_ok(bg, c, "grad gamma")
        _guard_ok(bb, c, "grad beta")
        runs.append((_sl(dx, gdx).clone(), gg.clone(), gb.clone()))
    m, r = st[:, 0:1].double(), st[:, 1:2].double()
    xh = (xd - m) * r
    dyd = _sl(dy, gdy).double().reshape(-1, c)
    gd = dyd * gamma.double()
    m1, m2 = gd.mean(-1, keepdim=True), (gd * xh).mean(-1, keepdim=True)
    ref = r * (gd - m1 - xh * m2)
    mag = r * (gd.abs() + gd.abs().mean(-1, keepdim=True) + xh.abs() * (gd * xh).abs().mean(-1, keepdim=True))
    if addend:
        av = _sl(add, addend).double().reshape(-1, c)
        ref, mag = ref + av, mag + av.abs()
    check("LayerNorm backward dx (bf16)", runs[0][0].reshape(-1, c), ref, bound(ref, mag, c, R_BF16), "dx")
    rows = xd.shape[0]
    rg, mg = (dyd * xh).sum(0), (dyd * xh).abs().sum(0)
    rb, mb = dyd.sum(0), dyd.abs().sum(0)
    if accumulate:
        rg, mg, rb, mb = rg + g0[0].double(), mg + g0[0].double().abs(), rb + g0[1].double(), mb + g0[1].double().abs()
    check("LayerNorm parameter gradients (fp32)", runs[0][1], rg, bound(rg, mg, rows, 0.0), "grad gamma")
    check("LayerNorm parameter gradients (fp32)", runs[0][2], rb, bound(rb, mb, rows, 0.0), "grad beta")
    for a, b in zip(runs[0], runs[1]):
        assert torch.equal(a, b), "layernorm_bwd is not bit-reproducible"


def run_add(ga, gb, go, seed=57):
    """yb200_add: bit-equal to (a.float() + b.float()).bfloat16()"""
    capi, L = _lib()
    g = _g(seed)
    a, b = _in_view(ga, g), _in_view(gb, g, scale=3.0)
    out, out0 = _out_view(go, g)
    aa, ba, oa = _act(capi, a, ga), _act(capi, b, gb), _act(capi, out, go)
    capi.check(L.yb200_add(ctypes.byref(aa), ctypes.byref(ba), ctypes.byref(oa), capi.stream_ptr()), "add")
    want = (_sl(a, ga).float() + _sl(b, gb).float()).bfloat16()
    assert torch.equal(_sl(out, go).view(torch.int16), want.view(torch.int16)), "add differs from the fp32 sum rounded to bf16"
    _outside_same(out, out0, go, "out")


def run_dropout(gx, gr, go, p, extra_scale, seed=58):
    """yb200_dropout: out = bf16(residual + x * keep / (1 - p) * extra_scale).  The keep pattern (read from a call without residual: x has no
    zeros, so out != 0 <=> kept) is bit-equal to oracle/detr_oracle.py's hash; the values are within one bf16 rounding of fp64 plus the fp32
    rounding of the factor and the FMA (2 U of the product)"""
    from oracle import detr_oracle as dto

    capi, L = _lib()
    g = _g(seed)
    x = _in_view(gx, g)
    xv = _sl(x, gx)
    xv.copy_(torch.where(xv == 0, torch.ones_like(xv), xv))
    res = _in_view(gr, g) if gr else None
    dseed = 0x13579BD
    b, _, l, c = gx[:4]
    mult = dto.dropout_multiplier(dseed, (b, l, c), p, device="cuda").double().view(b, 1, l, c) * float(torch.tensor(extra_scale, dtype=torch.float32))
    for with_res in ([True, False] if gr else [False]):
        out, out0 = _out_view(go, g)
        xa, oa = _act(capi, x, gx), _act(capi, out, go)
        ra = _act(capi, res, gr) if with_res else None
        capi.check(L.yb200_dropout(ctypes.byref(xa), ctypes.byref(ra) if with_res else None, ctypes.byref(oa), ctypes.c_float(p), ctypes.c_uint32(dseed),
                                   ctypes.c_float(extra_scale), capi.stream_ptr()), "dropout")
        _outside_same(out, out0, go, "out")
        got = _sl(out, go)
        prod = xv.double() * mult
        ref = prod + (_sl(res, gr).double() if with_res else 0.0)
        check("dropout (bf16)", got, ref, (R_BF16 + 2 * U) * ref.abs() + 2 * U * prod.abs(), "out")
        if not with_res:
            kept = got != 0
            want = mult != 0
            assert torch.equal(kept, want), f"keep pattern differs from the oracle's hash in {int((kept != want).sum())} of {kept.numel()} elements"


def run_f64_to_f32(n, accumulate, zero_src, seed=59):
    """yb200_f64_to_f32: dst = (accumulate ? dst : 0) + (float)src, exactly (one fp32 rounding of src, one fp32 addition); src zeroed when
    asked; nothing past n touched"""
    capi, L = _lib()
    g = _g(seed)
    src = torch.randn(n, generator=g, device="cuda", dtype=torch.float64) * 1e3
    sb, s = _guarded((n,), src, torch.float64)
    d0 = torch.randn(n, generator=g, device="cuda")
    db, d = _guarded((n,), d0)
    capi.check(L.yb200_f64_to_f32(capi.ptr(s), n, capi.ptr(d), accumulate, zero_src, capi.stream_ptr()), "f64_to_f32")
    want = (d0 + src.float()) if accumulate else src.float()
    assert torch.equal(d, want), "f64_to_f32 is not the exact fp32 conversion (and addition)"
    assert torch.equal(s, torch.zeros_like(src) if zero_src else src), "source not zeroed / changed"
    _guard_ok(sb, n, "source")
    _guard_ok(db, n, "destination")


RUN = dict(pack=run_pack2, affine=run_affine, linear_relu=run_linear_relu, dgrad=run_dgrad, dgrad_relu=run_dgrad_relu, wgrad=run_wgrad,
           colsum=run_colsum, ln_fwd=run_ln_fwd, ln_bwd=run_ln_bwd, add=run_add, dropout=run_dropout, f64_to_f32=run_f64_to_f32,
           attention=run_attention)


# ------------------------------------------------------------------------------------------------------------------------------------
# A. recordings
# ------------------------------------------------------------------------------------------------------------------------------------
QUERIES = ("yb200_conv2d_wgrad_workspace", "yb200_colsum_workspace", "yb200_layernorm_bwd_workspace", "yb200_attention_bwd_workspace")
ENTRY_POINTS = {"yb200_pack_conv_weight", "yb200_conv2d_affine_fwd", "yb200_linear_relu_fwd", "yb200_add", "yb200_attention_fwd_dropout",
                "yb200_dropout", "yb200_layernorm_fwd", "yb200_layernorm_bwd", "yb200_conv2d_dgrad", "yb200_conv2d_wgrad", "yb200_colsum",
                "yb200_linear_dgrad_relu", "yb200_f64_to_f32", "yb200_attention_bwd_dropout"} | set(QUERIES)


class _Recorder:
    """stands in for a `_Kernels` instance's library handle: records every call (entry point, arguments, return code) and forwards it"""

    def __init__(self, lib, log):
        self._lib, self.log = lib, log

    def __getattr__(self, name):
        fn = getattr(self._lib, name)
        if not name.startswith("yb200_") or name == "yb200_last_error":
            return fn

        def rec(*a):
            rc = fn(*a)
            self.log.append((name, a, rc))
            return rc
        return rec


def _v(a):
    return a.value if isinstance(a, (ctypes.c_void_p, ctypes.c_float, ctypes.c_int64, ctypes.c_uint32)) else a


def _case_of(name, a):
    """replay case of one recorded call (None for the workspace queries)"""
    if name == "yb200_pack_conv_weight":
        return dict(fn="pack", cout=a[1], cin=a[2], k=a[3], cout_pad=a[4], cin_pad=a[5], dgrad=_given(a[7]))
    if name == "yb200_conv2d_affine_fwd":
        return dict(fn="affine", gx=_geo(a[0]), go=_geo(a[5]), gr=_geo(a[4]), k=a[6], s=a[7], with_scale=_given(a[2]), with_shift=_given(a[3]))
    if name == "yb200_linear_relu_fwd":
        return dict(fn="linear_relu", gx=_geo(a[0]), go=_geo(a[3]))
    if name == "yb200_conv2d_dgrad":
        return dict(fn="dgrad", gdz=_geo(a[0]), gdx=_geo(a[2]), ga=_geo(a[3]), k=a[4], s=a[5])
    if name == "yb200_linear_dgrad_relu":
        return dict(fn="dgrad_relu", gdz=_geo(a[0]), gh=_geo(a[2]), gdu=_geo(a[3]), bias_sum=_given(a[4]))
    if name == "yb200_conv2d_wgrad":
        return dict(fn="wgrad", gx=_geo(a[0]), gdz=_geo(a[1]), k=a[2], s=a[3], cin_real=a[4], accumulate=a[6])
    if name == "yb200_colsum":
        return dict(fn="colsum", gx=_geo(a[0]), scale=_v(a[1]), accumulate=a[3])
    if name == "yb200_layernorm_fwd":
        return dict(fn="ln_fwd", gx=_geo(a[0]), gy=_geo(a[4]), eps=_v(a[3]), stats=_given(a[5]))
    if name == "yb200_layernorm_bwd":
        return dict(fn="ln_bwd", gdy=_geo(a[0]), gx=_geo(a[1]), gdx=_geo(a[5]), addend=_geo(a[4]), accumulate=a[8])
    if name == "yb200_add":
        return dict(fn="add", ga=_geo(a[0]), gb=_geo(a[1]), go=_geo(a[2]))
    if name == "yb200_dropout":
        return dict(fn="dropout", gx=_geo(a[0]), gr=_geo(a[1]), go=_geo(a[2]), p=_v(a[3]), extra_scale=_v(a[5]))
    if name == "yb200_f64_to_f32":
        return dict(fn="f64_to_f32", n=a[1], accumulate=a[3], zero_src=a[4])
    if name == "yb200_attention_fwd_dropout":
        return dict(fn="attention", gq=_geo(a[0]), gk=_geo(a[1]), gv=_geo(a[2]), go=_geo(a[5]), masked=_given(a[3]), lse=_given(a[6]), p=_v(a[7]))
    if name == "yb200_attention_bwd_dropout":
        return dict(fn="attention", gq=_geo(a[0]), gk=_geo(a[1]), gv=_geo(a[2]), go=_geo(a[3]), masked=_given(a[5]), lse=True, p=_v(a[12]),
                    grads=(_geo(a[4]), _geo(a[8]), _geo(a[9]), _geo(a[10])))
    if name in QUERIES:
        return None
    raise AssertionError(f"{name}: a DETR call this module does not replay")


def _kernels_of(*mods):
    from yolov7_d2_b200.detr import _Kernels

    out = []
    for mod in mods:
        for m in mod.modules():
            k = getattr(m, "k", None)
            if isinstance(k, _Kernels) and all(k is not o for o in out):
                out.append(k)
    return out


def _recorded(kns, fn):
    log = []
    for kn in kns:
        kn.L = _Recorder(kn.L, log)
    try:
        fn()
        torch.cuda.synchronize()
    finally:
        for kn in kns:
            kn.L = kn.L._lib
    return log


def _image_mask(b, dev):
    """[B, 25, 42] bool padding mask: image 0 unpadded, image 1 valid on 19 x 31 (padded right and bottom)"""
    m = torch.zeros(b, *MAP, dtype=torch.bool, device=dev)
    m[1, 19:, :] = True
    m[1, :, 31:] = True
    return m


def _record_training_step():
    """one training step of DETR-R50's transformer and tail at B = 2, 100 queries, a 25 x 42 map"""
    from yolov7_d2_b200.detr import MLP, Transformer, _Kernels, _linear_stack

    import types

    torch.manual_seed(0)
    dev = torch.device("cuda")
    tr = Transformer(256, 8, 6, 6, 2048, dropout=0.1, return_intermediate_dec=True).train()
    proj = nn.Conv2d(2048, 256, 1).to(dev)
    cls = nn.Linear(256, 81).to(dev)
    box = MLP(256, 256, 4, 3).to(dev)
    query = nn.Parameter(torch.randn(100, 256, device=dev))
    kn = _Kernels()
    b = 2
    feat = torch.randn(b, 2048, *MAP, device=dev).relu().requires_grad_(True)
    mask = _image_mask(b, dev)
    pos = torch.randn(b, 256, *MAP, device=dev)

    def step():
        lin = types.SimpleNamespace(weight=proj.weight.view(256, -1), bias=proj.bias)
        src = _linear_stack(kn, feat.permute(0, 2, 3, 1), [lin]).permute(0, 3, 1, 2)
        hs = tr(src, mask, query, pos)[0]
        logits = _linear_stack(kn, hs, [cls])
        boxes = box(hs).sigmoid()
        loss = (logits * torch.randn_like(logits)).sum() + (boxes * torch.randn_like(boxes)).sum()
        loss.backward()

    log = _recorded(_kernels_of(tr, box) + [kn], step)
    return tr, log


def _record_decoder_300():
    from yolov7_d2_b200.detr import TransformerDecoderLayer

    torch.manual_seed(1)
    dev = torch.device("cuda")
    layer = TransformerDecoderLayer(256, 8, 2048, 0.1).train()
    b, lk = 2, MAP[0] * MAP[1]
    tgt = torch.randn(300, b, 256, device=dev, requires_grad=True)
    mem = torch.randn(lk, b, 256, device=dev, requires_grad=True)
    pos = torch.randn(lk, b, 256, device=dev)
    qpos = torch.randn(300, b, 256, device=dev, requires_grad=True)
    mmask = _image_mask(b, dev).flatten(1)

    def step():
        out = layer(tgt, mem, memory_key_padding_mask=mmask, pos=pos, query_pos=qpos)
        (out * torch.randn_like(out)).sum().backward()

    return _recorded(_kernels_of(layer), step)


def _record_inference(tr):
    dev = torch.device("cuda")
    enc, dec = tr.encoder.layers[0], tr.decoder.layers[0]
    b, lk = 2, MAP[0] * MAP[1]
    src = torch.randn(lk, b, 256, device=dev)
    pos = torch.randn(lk, b, 256, device=dev)
    mmask = _image_mask(b, dev).flatten(1)

    def fwd():
        with torch.no_grad():
            mem = enc(src, src_key_padding_mask=mmask, pos=pos)
            dec(torch.zeros(100, b, 256, device=dev), mem, memory_key_padding_mask=mmask, pos=pos, query_pos=torch.randn(100, b, 256, device=dev))

    return _recorded(_kernels_of(enc, dec), fwd)


RECORDINGS = {}


def _recordings():
    """{recording: log}, recorded when the module is collected on a machine with a GPU"""
    if not RECORDINGS and torch.cuda.is_available():
        tr, log = _record_training_step()
        RECORDINGS["train"] = log
        RECORDINGS["decoder300"] = _record_decoder_300()
        tr.eval()
        RECORDINGS["no_grad"] = _record_inference(tr)
        del tr
        torch.cuda.empty_cache()
    return RECORDINGS


def _view(g):
    if g is None:
        return "-"
    return f"{g[0]}x{g[2]}x{g[3]}" + ("" if g[4] == g[3] and g[5] == 0 else f"@{g[5]}/{g[4]}")


def _describe(c):
    fn = c["fn"]
    if fn == "pack":
        return f"{c['cout']}x{c['cin']} -> {c['cout_pad']} rows" + (" +dgrad" if c["dgrad"] else "")
    if fn == "attention":
        s = f"{c['gq'][0]}x{c['gq'][2]}x{c['gk'][2]} q{_view(c['gq'])} k{_view(c['gk'])} v{_view(c['gv'])} p{c['p']:.1f}"
        return s + (" masked" if c["masked"] else "") + (" bwd" if c.get("grads") else "") + ("" if c["lse"] else " no-lse")
    views = [f"{k}={_view(v)}" for k, v in c.items() if k.startswith("g") and isinstance(v, tuple)]
    rest = [f"{k}={v}" for k, v in c.items() if k != "fn" and not (k.startswith("g") and (isinstance(v, tuple) or v is None))]
    return " ".join(views + rest)


def _distinct():
    """[(test id, case)]: each distinct call of the recordings once"""
    seen, out = {}, []
    for rec, log in _recordings().items():
        for name, a, _ in log:
            case = _case_of(name, a)
            if case is None:
                continue
            key = tuple(sorted(case.items()))
            if key in seen:
                seen[key][1] += 1
                continue
            seen[key] = [len(out), 1]
            out.append([f"{rec}: {name[len('yb200_'):]} {_describe(case)}", case])
    for i, n in seen.values():
        if n > 1:
            out[i][0] += f" (+{n - 1} more)"
    return [tuple(x) for x in out]


def pytest_generate_tests(metafunc):
    if "detr_case" in metafunc.fixturenames:
        cases = _distinct()
        metafunc.parametrize("detr_case", [c[1] for c in cases], ids=[c[0] for c in cases])


def test_detr_call(cuda, detr_case):
    case = dict(detr_case)
    RUN[case.pop("fn")](**case)


def test_recording_is_complete(cuda):
    """every entry point DETR calls is one this module replays, every call succeeded, and the shipped geometries are among the cases"""
    recs = _recordings()
    names = {name for log in recs.values() for name, _, _ in log}
    assert names == ENTRY_POINTS, f"entry points called {sorted(names)}, replayed {sorted(ENTRY_POINTS)}"
    assert all(rc >= 0 for log in recs.values() for _, _, rc in log)
    cases = [c for _, c in _distinct()]
    print(f"\n{len(cases)} distinct DETR kernel geometries replayed")
    att = [c for c in cases if c["fn"] == "attention"]
    # 100 queries x 1050 keys, masked cross-attention, forward and backward with dropout; its no-grad form without lse
    assert any(c["gq"][2] == 100 and c["gk"][2] == 1050 and c["masked"] and c.get("grads") and c["p"] > 0 for c in att), "no 100 x 1050 masked bwd"
    assert any(c["gq"][2] == 100 and c["gk"][2] == 1050 and not c["lse"] and c["p"] == 0 for c in att), "no no-grad 100 x 1050 forward"
    assert any(c["gq"][2] == 300 and c["gk"][2] == 300 and c.get("grads") for c in att), "no 300-query self-attention backward"
    assert any(c["gq"][2] == 1050 and c["gk"][2] == 1050 and c["masked"] and c.get("grads") for c in att), "no 1050-token encoder backward"
    # q|k|v packed at 768: the dz slice of the q|k rows (512 of 768) and the v rows (256 at 512)
    assert any(c["fn"] == "dgrad" and c["gdz"][3:] == (512, 768, 0) for c in cases), "no 512-of-768 dz slice"
    assert any(c["fn"] == "wgrad" and c["gdz"][3:] == (256, 768, 512) for c in cases), "no 256-at-512-of-768 dz slice"
    # K = 2048: linear2 forward and linear1's data gradient; the input projection
    assert any(c["fn"] == "affine" and c["gx"][3] == 2048 for c in cases), "no K = 2048 forward"
    assert any(c["fn"] == "dgrad" and c["gdz"][3] == 2048 for c in cases), "no K = 2048 data gradient"
    assert any(c["fn"] == "dgrad_relu" and c["gh"][3] == 2048 for c in cases), "no 2048-wide ReLU data gradient"
    # C = 256 LayerNorm with eps 1e-5, with and without statistics; its backward over the 2100 memory tokens
    assert any(c["fn"] == "ln_fwd" and c["gx"][3] == 256 and c["stats"] and abs(c["eps"] - 1e-5) < 1e-9 for c in cases)
    assert any(c["fn"] == "ln_fwd" and not c["stats"] for c in cases)
    assert any(c["fn"] == "ln_bwd" and c["gx"][0] * c["gx"][2] == 2100 for c in cases)
    # the heads' padded outputs: 81 -> 96 and 4 -> 16 rows
    assert any(c["fn"] == "pack" and (c["cout"], c["cout_pad"]) == (81, 96) for c in cases)
    assert any(c["fn"] == "pack" and (c["cout"], c["cout_pad"]) == (4, 16) for c in cases)
    assert any(c["fn"] == "dropout" and c["gr"] is not None for c in cases) and any(c["fn"] == "dropout" and c["gr"] is None for c in cases)


# ------------------------------------------------------------------------------------------------------------------------------------
# B'. calls the recordings make with one setting only
# ------------------------------------------------------------------------------------------------------------------------------------
def test_dropout_extra_scale(cuda):
    """the FFN backward's form: residual plus an extra scale that is not 1"""
    geo = (2, 1, 1050, 256, 256, 0)
    run_dropout(geo, geo, geo, 0.1, 0.75)


@pytest.mark.parametrize("n,accumulate,zero_src", [(2048, 0, 0), (2048, 1, 1), (81, 1, 0)])
def test_f64_to_f32_modes(cuda, n, accumulate, zero_src):
    run_f64_to_f32(n, accumulate, zero_src)


def test_layernorm_bwd_addend_accumulate(cuda):
    geo = (2, 1, 1050, 256, 256, 0)
    run_ln_bwd(geo, geo, geo, geo, 1)


# ------------------------------------------------------------------------------------------------------------------------------------
# C. the attention core at the shipped and benchmarked shapes
# ------------------------------------------------------------------------------------------------------------------------------------
SHAPES = [(2, 8, 1050, 1050), (2, 8, 100, 1050), (2, 8, 100, 100), (2, 8, 300, 300), (16, 8, 1050, 1050)]


def _layout(b, h, lq, lk):
    """the views the layers pass: self-attention q | k | v in one [.., 3E] buffer (and dq | dk | dv likewise), cross-attention q and dq on
    their own, k | v and dk | dv in [.., 2E] buffers; the memory (Lk = 1050) masked"""
    e = 32 * h
    if lq == lk:
        gq, gk, gv = (b, 1, lq, e, 3 * e, 0), (b, 1, lk, e, 3 * e, e), (b, 1, lk, e, 3 * e, 2 * e)
    else:
        gq, gk, gv = (b, 1, lq, e, e, 0), (b, 1, lk, e, 2 * e, 0), (b, 1, lk, e, 2 * e, e)
    go = (b, 1, lq, e, e, 0)
    return gq, gk, gv, go, (go, gq, gk, gv)


@pytest.mark.parametrize("p", [0.0, 0.1])
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "B%d_H%d_q%d_k%d" % s)
def test_attention_core(cuda, shape, p):
    gq, gk, gv, go, grads = _layout(*shape)
    run_attention(gq, gk, gv, go, shape[3] == MAP[0] * MAP[1], p, lse=True, grads=grads, seed=60 + shape[2] + shape[0])


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    saved = dict(WORST)
    WORST.clear()
    yield
    if WORST:
        print("\nworst |err| / bound per case class: " + "; ".join(f"{k}: {v:.3g}" for k, v in sorted(WORST.items())))
    for k, v in saved.items():
        WORST[k] = max(WORST.get(k, 0.0), v)
