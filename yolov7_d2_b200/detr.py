"""DETR transformer layers on the H100 kernels (forward path; SURVEY.md par.8a row T1).

Reference: yolov7/modeling/backbone/detr_backbone.py -- `TransformerEncoderLayer` :128-187 (forward_post :157-170), `TransformerDecoderLayer`
:190-279 (forward_post :221-242); both wrap torch's nn.MultiheadAttention (:140, :200-202).  The classes below keep the reference's
constructor arguments, parameter names / shapes (`self_attn.in_proj_weight` [3E,E], `linear1.weight`, `norm1.weight` ...) and the seq-first
`[L, B, E]` fp32 interface, and run

    x (+pos) -> in_proj GEMMs (bias epilogue, q|k|v packed in one [B, L, 3E] buffer) -> yb200_attention_fwd (wgmma, streaming softmax)
      -> out_proj GEMM (+bias +residual epilogue) -> LayerNorm -> linear1 GEMM (+bias +ReLU epilogue) -> linear2 GEMM (+bias +residual) -> LayerNorm

Internally tokens are batch-first bf16 `[B, 1, L, E]` views (yb200_act).  Forward and backward: with gradients enabled the layers run as one autograd node each
(`_EncoderLayerFn` / `_DecoderLayerFn`: attention backward, data / weight gradients and LayerNorm backward on the same kernels), validated on
hardware against the reference layer's autograd (tests/test_detr_gpu.py); YB200_DETR_TRAINING=0 forces the inference path.
Dropout (p = 0.1 in the reference: on the attention probabilities inside nn.MultiheadAttention and nn.Dropout on the residual branches / in the FFN) is
active in training mode: the masks are a counter-based hash of (seed, element index) evaluated inside the kernels (yb200_attention_*_dropout,
yb200_dropout), regenerated in the backward from the same seeds; seeds come from torch's CPU generator.  Same distribution as torch's Philox masks, not
the same bits: parity = the same computation given the same mask (tests/test_detr_dropout_gpu.py, oracle/detr_oracle.py).  `attn_mask` (never passed by the
reference's DETR) and `normalize_before=True` are not supported.  There is no CPU implementation.
"""
import ctypes
import os
import types

import torch
import torch.nn as nn

from . import capi

LN_EPS = 1e-5
# The layers' backward wiring (autograd.Function over the attention-backward / dgrad / wgrad / LayerNorm-backward kernels) is the default
# whenever autograd is recording; YB200_DETR_TRAINING=0 switches it off (inference-only modules)
TRAINING_PATH = os.environ.get("YB200_DETR_TRAINING", "1") == "1"


def _bl(t):
    """[L, B, E] (any float dtype, CUDA) -> contiguous bf16 [B, 1, L, E]"""
    return t.detach().permute(1, 0, 2).to(torch.bfloat16).contiguous().unsqueeze(1)


def _lb(t):
    """[B, 1, L, E] bf16 -> [L, B, E] fp32"""
    return t.squeeze(1).permute(1, 0, 2).float().contiguous()


class _Kernels:
    """thin wrappers: torch tensors in, C-ABI calls on the current stream"""

    def __init__(self):
        self.L = capi.lib()

    @staticmethod
    def _a(t, off=0, c=None):
        return capi.act(t, off, c)

    def pack(self, w):  # [out, in] fp32 -> bf16 GEMM operand
        out_f, in_f = w.shape
        wf = torch.empty(out_f, 1, in_f, dtype=torch.bfloat16, device=w.device)
        capi.check(self.L.yb200_pack_conv_weight(capi.ptr(w.detach().contiguous()), out_f, in_f, 1, out_f, in_f, capi.ptr(wf), None, capi.stream_ptr()), "pack")
        return wf

    def add(self, a, b):
        out = torch.empty_like(a)
        aa, ba, oa = self._a(a), self._a(b), self._a(out)
        capi.check(self.L.yb200_add(ctypes.byref(aa), ctypes.byref(ba), ctypes.byref(oa), capi.stream_ptr()), "add")
        return out

    def linear(self, x, w, bias, out=None, out_off=0, residual=None, relu=False):
        """out[..., out_off:out_off+N] = x W^T + bias (+ residual) (ReLU); x may be a (tensor, off, c) slice"""
        xt, xo, xc = x if isinstance(x, tuple) else (x, 0, None)
        n_out = w.shape[0]
        b, _, l, _ = xt.shape
        if out is None:
            out = torch.empty(b, 1, l, n_out, dtype=torch.bfloat16, device=xt.device)
        xa, oa = self._a(xt, xo, xc), self._a(out, out_off, n_out)
        wf = self.pack(w)
        bias = bias.detach().contiguous()
        if relu:
            capi.check(self.L.yb200_linear_relu_fwd(ctypes.byref(xa), capi.ptr(wf), capi.ptr(bias), ctypes.byref(oa), capi.stream_ptr()), "linear+relu")
        else:
            ra = self._a(residual) if residual is not None else None
            capi.check(self.L.yb200_conv2d_affine_fwd(ctypes.byref(xa), capi.ptr(wf), None, capi.ptr(bias), ctypes.byref(ra) if ra is not None else None,
                                                      ctypes.byref(oa), 1, 1, capi.stream_ptr()), "linear")
        return out

    def layernorm(self, x, weight, bias):
        y = torch.empty_like(x)
        xa, ya = self._a(x), self._a(y)
        capi.check(self.L.yb200_layernorm_fwd(ctypes.byref(xa), capi.ptr(weight.detach().contiguous()), capi.ptr(bias.detach().contiguous()), ctypes.c_float(LN_EPS),
                                              ctypes.byref(ya), None, capi.stream_ptr()), "layernorm")
        return y

    # ---- helpers of the training path ------------------------------------------------------------------------------------------
    def pack2(self, w):
        out_f, in_f = w.shape
        wf = torch.empty(out_f, 1, in_f, dtype=torch.bfloat16, device=w.device)
        wd = torch.empty(in_f, 1, out_f, dtype=torch.bfloat16, device=w.device)
        capi.check(self.L.yb200_pack_conv_weight(capi.ptr(w.detach().contiguous()), out_f, in_f, 1, out_f, in_f, capi.ptr(wf), capi.ptr(wd), capi.stream_ptr()), "pack")
        return wf, wd

    def _ws(self, nbytes, dev):
        return torch.empty(max(int(nbytes), 16), dtype=torch.uint8, device=dev)

    def layernorm_train(self, x, weight, bias):
        b, _, l, _ = x.shape
        y = torch.empty_like(x)
        stats = torch.empty(b * l, 2, device=x.device)
        xa, ya = self._a(x), self._a(y)
        capi.check(self.L.yb200_layernorm_fwd(ctypes.byref(xa), capi.ptr(weight.detach().contiguous()), capi.ptr(bias.detach().contiguous()), ctypes.c_float(LN_EPS),
                                              ctypes.byref(ya), capi.ptr(stats), capi.stream_ptr()), "layernorm")
        return y, stats

    def layernorm_bwd(self, dy, x, stats, weight):
        dx = torch.empty_like(x)
        c = x.shape[-1]
        gw, gb = torch.empty(c, device=x.device), torch.empty(c, device=x.device)
        da, xa, dxa = self._a(dy), self._a(x), self._a(dx)
        ws = self._ws(self.L.yb200_layernorm_bwd_workspace(ctypes.byref(xa)), x.device)
        capi.check(self.L.yb200_layernorm_bwd(ctypes.byref(da), ctypes.byref(xa), capi.ptr(stats), capi.ptr(weight.detach().contiguous()), None, ctypes.byref(dxa),
                                              capi.ptr(gw), capi.ptr(gb), 0, capi.ptr(ws), capi.stream_ptr()), "layernorm bwd")
        return dx, gw, gb

    def dgrad(self, dz, w_dgrad, cin, addend=None):
        """dx = dz W (+ addend); dz may be a (tensor, off, c) slice"""
        dt, do, dc = dz if isinstance(dz, tuple) else (dz, 0, None)
        b, _, l, _ = dt.shape
        dx = torch.empty(b, 1, l, cin, dtype=torch.bfloat16, device=dt.device)
        da, xa = self._a(dt, do, dc), self._a(dx)
        aa = self._a(addend) if addend is not None else None
        capi.check(self.L.yb200_conv2d_dgrad(ctypes.byref(da), capi.ptr(w_dgrad), ctypes.byref(xa), ctypes.byref(aa) if aa is not None else None, 1, 1, capi.stream_ptr()),
                   "dgrad")
        return dx

    def dgrad_relu(self, dz, w_dgrad, h):
        """du = (dz W) masked by h > 0, and its column sums (= bias gradient of the Linear that produced h)"""
        ff = h.shape[-1]
        du = torch.empty_like(h)
        acc = torch.zeros(ff, dtype=torch.float64, device=h.device)
        gb = torch.empty(ff, device=h.device)
        za, ha, dua = self._a(dz), self._a(h), self._a(du)
        capi.check(self.L.yb200_linear_dgrad_relu(ctypes.byref(za), capi.ptr(w_dgrad), ctypes.byref(ha), ctypes.byref(dua), capi.ptr(acc), capi.stream_ptr()),
                   "dgrad + relu bwd")
        capi.check(self.L.yb200_f64_to_f32(capi.ptr(acc), ff, capi.ptr(gb), 0, 1, capi.stream_ptr()), "bias grad")
        return du, gb

    def wgrad(self, x, dz, out):
        """out[cout, cin] (fp32, contiguous) = dz^T x"""
        xt, xo, xc = x if isinstance(x, tuple) else (x, 0, None)
        dt, do, dc = dz if isinstance(dz, tuple) else (dz, 0, None)
        xa, da = self._a(xt, xo, xc), self._a(dt, do, dc)
        ws = self._ws(self.L.yb200_conv2d_wgrad_workspace(ctypes.byref(xa), ctypes.byref(da), 1, 1), xt.device)
        assert out.is_contiguous() and out.shape == (da.c, xa.c)
        capi.check(self.L.yb200_conv2d_wgrad(ctypes.byref(xa), ctypes.byref(da), 1, 1, xa.c, capi.ptr(out), 0, capi.ptr(ws), ctypes.c_int64(ws.numel()), capi.stream_ptr()),
                   "wgrad")

    def colsum(self, dz, out):
        dt, do, dc = dz if isinstance(dz, tuple) else (dz, 0, None)
        da = self._a(dt, do, dc)
        ws = self._ws(self.L.yb200_colsum_workspace(ctypes.byref(da)), dt.device)
        capi.check(self.L.yb200_colsum(ctypes.byref(da), ctypes.c_float(1.0), capi.ptr(out), 0, capi.ptr(ws), capi.stream_ptr()), "colsum")

    def attention_train(self, q, k, v, mask, heads, p_drop=0.0, seed=0):
        """p_drop > 0: dropout on the attention probabilities (nn.MultiheadAttention(dropout=p), detr_backbone.py:140), mask = f(seed, b, h, q, k)"""
        qt, _, e = q
        b, _, lq, _ = qt.shape
        out = torch.empty(b, 1, lq, e, dtype=torch.bfloat16, device=qt.device)
        lse = torch.empty(b, heads, lq, device=qt.device)
        qa, ka, va, oa = self._a(*q), self._a(*k), self._a(*v), self._a(out)
        capi.check(self.L.yb200_attention_fwd_dropout(ctypes.byref(qa), ctypes.byref(ka), ctypes.byref(va), capi.ptr(mask), ctypes.c_float((e // heads) ** -0.5),
                                                      ctypes.byref(oa), capi.ptr(lse), ctypes.c_float(p_drop), ctypes.c_uint32(seed), capi.stream_ptr()), "attention")
        return out, lse

    def attention_bwd(self, q, k, v, out, dout, mask, heads, lse, dq, dk, dv, p_drop=0.0, seed=0):
        e = q[2]
        qa, ka, va, oa, da = self._a(*q), self._a(*k), self._a(*v), self._a(out), self._a(dout)
        dqa, dka, dva = self._a(*dq), self._a(*dk), self._a(*dv)
        ws = self._ws(self.L.yb200_attention_bwd_workspace(ctypes.byref(qa)), out.device)
        capi.check(self.L.yb200_attention_bwd_dropout(ctypes.byref(qa), ctypes.byref(ka), ctypes.byref(va), ctypes.byref(oa), ctypes.byref(da), capi.ptr(mask),
                                                      ctypes.c_float((e // heads) ** -0.5), capi.ptr(lse), ctypes.byref(dqa), ctypes.byref(dka), ctypes.byref(dva),
                                                      capi.ptr(ws), ctypes.c_float(p_drop), ctypes.c_uint32(seed), capi.stream_ptr()), "attention bwd")

    def dropout(self, x, p_drop, seed, residual=None, scale=1.0):
        """residual + x * keep(seed, element) / (1 - p) * scale  (nn.Dropout of the residual branches / the FFN, detr_backbone.py:147-152);
        the backward is the same call on the gradient with the same seed"""
        out = torch.empty_like(x)
        xa, oa = self._a(x), self._a(out)
        ra = self._a(residual) if residual is not None else None
        capi.check(self.L.yb200_dropout(ctypes.byref(xa), ctypes.byref(ra) if ra is not None else None, ctypes.byref(oa), ctypes.c_float(p_drop), ctypes.c_uint32(seed),
                                        ctypes.c_float(scale), capi.stream_ptr()), "dropout")
        return out

    def attention(self, q, k, v, mask, heads):
        """q, k, v: (tensor, channel offset, E) slices of [B,1,L,*] buffers; mask: uint8 [B, Lk] or None"""
        qt, qo, e = q
        b, _, lq, _ = qt.shape
        out = torch.empty(b, 1, lq, e, dtype=torch.bfloat16, device=qt.device)
        qa, ka, va, oa = self._a(*q), self._a(*k), self._a(*v), self._a(out)
        capi.check(self.L.yb200_attention_fwd(ctypes.byref(qa), ctypes.byref(ka), ctypes.byref(va), capi.ptr(mask), ctypes.c_float((e // heads) ** -0.5),
                                              ctypes.byref(oa), None, capi.stream_ptr()), "attention")
        return out


def _check_inputs(*tensors):
    for t in tensors:
        if t is None:
            continue
        if not t.is_cuda:
            raise capi.Yb200Error("DETR layers: inputs must be CUDA tensors (no CPU path)")
        if t.requires_grad and torch.is_grad_enabled():
            raise capi.Yb200Error("DETR layers: the attention backward kernel is not built yet -- run under torch.no_grad()")


def _mask_u8(mask):
    return None if mask is None else mask.to(torch.uint8).contiguous()


class _MhaParams(nn.Module):
    """parameter container with nn.MultiheadAttention's names (detr_backbone.py:140)"""

    def __init__(self, d_model, device):
        super().__init__()
        self.in_proj_weight = nn.Parameter(torch.empty(3 * d_model, d_model, device=device))
        self.in_proj_bias = nn.Parameter(torch.zeros(3 * d_model, device=device))
        self.out_proj = nn.Module()
        self.out_proj.weight = nn.Parameter(torch.empty(d_model, d_model, device=device))
        self.out_proj.bias = nn.Parameter(torch.zeros(d_model, device=device))
        nn.init.xavier_uniform_(self.in_proj_weight)
        nn.init.kaiming_uniform_(self.out_proj.weight, a=5 ** 0.5)


class _Norm(nn.Module):
    def __init__(self, d, device):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(d, device=device))
        self.bias = nn.Parameter(torch.zeros(d, device=device))


class _Lin(nn.Module):
    def __init__(self, i, o, device):
        super().__init__()
        lin = nn.Linear(i, o)
        self.weight = nn.Parameter(lin.weight.detach().to(device))
        self.bias = nn.Parameter(lin.bias.detach().to(device))


class _LayerBase(nn.Module):
    def __init__(self, d_model, nhead, dim_feedforward, dropout, activation, normalize_before, device):
        super().__init__()
        if d_model % nhead or d_model // nhead != 32:
            raise capi.Yb200Error(f"attention kernel is built for head dimension 32 (got d_model={d_model}, nhead={nhead})")
        if activation != "relu":
            raise capi.Yb200Error("only the reference's default activation (relu) is implemented")
        if normalize_before:
            raise capi.Yb200Error("normalize_before=True (forward_pre) is not implemented")
        self.d_model, self.nhead = d_model, nhead
        self.dropout_p = float(dropout)
        self._ctor = (d_model, nhead, dim_feedforward, dropout, activation, normalize_before, device)
        self.linear1 = _Lin(d_model, dim_feedforward, device)
        self.linear2 = _Lin(dim_feedforward, d_model, device)
        self.k = _Kernels()

    def _dropout_state(self, n):
        """(p, n seeds) of one training forward.  p = 0 in eval mode / with dropout=0 (every kernel then takes its dropout-free path).  The seeds come
        from torch's CPU generator (torch.manual_seed reproduces a run; no device synchronisation); the masks themselves are a counter-based hash of
        (seed, element index) evaluated inside the kernels (csrc/attention.cu) -- not torch's Philox stream: same distribution, different bits."""
        p = self.dropout_p if self.training else 0.0
        if p <= 0.0:
            return 0.0, (0,) * n
        return p, tuple(int(v) for v in torch.randint(0, 2 ** 31 - 1, (n,)))

    def _self_attention(self, x, qk, att, mask):
        """x: value source, qk: query/key source ([B,1,L,E] bf16); returns x + out_proj(attention)"""
        e, kn = self.d_model, self.k
        b, _, l, _ = x.shape
        qkv = torch.empty(b, 1, l, 3 * e, dtype=torch.bfloat16, device=x.device)
        w, bias = att.in_proj_weight, att.in_proj_bias
        kn.linear(qk, w[:2 * e], bias[:2 * e], out=qkv, out_off=0)
        kn.linear(x, w[2 * e:], bias[2 * e:], out=qkv, out_off=2 * e)
        a = kn.attention((qkv, 0, e), (qkv, e, e), (qkv, 2 * e, e), mask, self.nhead)
        return kn.linear(a, att.out_proj.weight, att.out_proj.bias, residual=x)

    def _ffn(self, x, norm):
        kn = self.k
        h = kn.linear(x, self.linear1.weight, self.linear1.bias, relu=True)
        y = kn.linear(h, self.linear2.weight, self.linear2.bias, residual=x)
        return kn.layernorm(y, norm.weight, norm.bias)


class _EncoderLayerFn(torch.autograd.Function):
    """forward_post (detr_backbone.py:157-170) with everything the backward needs kept in bf16; backward = the chain
    LayerNorm2 <- linear2 (+ReLU mask, fused) <- linear1 <- LayerNorm1 <- out_proj <- attention core <- in_proj on the H100 kernels"""

    NAMES = ("self_attn.in_proj_weight", "self_attn.in_proj_bias", "self_attn.out_proj.weight", "self_attn.out_proj.bias", "linear1.weight", "linear1.bias",
             "linear2.weight", "linear2.bias", "norm1.weight", "norm1.bias", "norm2.weight", "norm2.bias")

    @staticmethod
    def forward(ctx, layer, src, pos, mask, *params):
        kn, e, heads = layer.k, layer.d_model, layer.nhead
        w_in, b_in, w_o, b_o, w1, b1, w2, b2, g1, be1, g2, be2 = params
        x = _bl(src)
        qk = x if pos is None else kn.add(x, _bl(pos))
        b, _, l, _ = x.shape
        qkv = torch.empty(b, 1, l, 3 * e, dtype=torch.bfloat16, device=x.device)
        kn.linear(qk, w_in[:2 * e], b_in[:2 * e], out=qkv, out_off=0)
        kn.linear(x, w_in[2 * e:], b_in[2 * e:], out=qkv, out_off=2 * e)
        pd, sd = layer._dropout_state(4)  # (p, seeds): attention probabilities, dropout1, FFN dropout, dropout2 (detr_backbone.py:157-170)
        att, lse = kn.attention_train((qkv, 0, e), (qkv, e, e), (qkv, 2 * e, e), mask, heads, pd, sd[0])
        if pd > 0:
            y1 = kn.dropout(kn.linear(att, w_o, b_o), pd, sd[1], residual=x)
        else:
            y1 = kn.linear(att, w_o, b_o, residual=x)
        x1, st1 = kn.layernorm_train(y1, g1, be1)
        h = kn.linear(x1, w1, b1, relu=True)
        if pd > 0:
            h = kn.dropout(h, pd, sd[2])  # the dropped activation is what linear2 sees and what the backward needs (h > 0 and kept)
            y2 = kn.dropout(kn.linear(h, w2, b2), pd, sd[3], residual=x1)
        else:
            y2 = kn.linear(h, w2, b2, residual=x1)
        out, st2 = kn.layernorm_train(y2, g2, be2)
        ctx.drop = (pd, sd)
        ctx.layer, ctx.mask, ctx.has_pos = layer, mask, pos is not None
        ctx.saved = (x, qk, qkv, att, lse, y1, st1, x1, h, y2, st2)
        ctx.params = params
        return _lb(out)

    @staticmethod
    def backward(ctx, g_out):
        layer = ctx.layer
        kn, e, heads = layer.k, layer.d_model, layer.nhead
        x, qk, qkv, att, lse, y1, st1, x1, h, y2, st2 = ctx.saved
        w_in, b_in, w_o, b_o, w1, b1, w2, b2, g1, be1, g2, be2 = ctx.params
        dev = x.device
        ff = w1.shape[0]
        g = _bl(g_out)
        # LayerNorm 2
        pd, sd = ctx.drop
        g_y2, gg2, gb2 = kn.layernorm_bwd(g, y2, st2, g2)
        # linear2 (+ residual to x1) and the ReLU in front of it; with dropout: g_t = dropout2's mask on the branch gradient, and the saved h is the
        # dropped activation (positive <=> positive and kept), so the ReLU mask also applies the FFN dropout mask -- its 1 / (1 - p) follows
        g_t = kn.dropout(g_y2, pd, sd[3]) if pd > 0 else g_y2
        _, w2d = kn.pack2(w2)
        du, gb1 = kn.dgrad_relu(g_t, w2d, h)
        if pd > 0:
            du = kn.dropout(du, pd, sd[2])
            gb1 = gb1 / (1.0 - pd)
        gw2 = torch.empty(e, ff, device=dev)
        kn.wgrad(h, g_t, gw2)
        gb2_lin = torch.empty(e, device=dev)
        kn.colsum(g_t, gb2_lin)
        # linear1; the residual branch of x1 joins through the addend
        _, w1d = kn.pack2(w1)
        g_x1 = kn.dgrad(du, w1d, e, addend=g_y2)
        gw1 = torch.empty(ff, e, device=dev)
        kn.wgrad(x1, du, gw1)
        # LayerNorm 1
        g_y1, gg1, gb1n = kn.layernorm_bwd(g_x1, y1, st1, g1)
        # out_proj (+ residual to x)
        g_o = kn.dropout(g_y1, pd, sd[1]) if pd > 0 else g_y1
        _, wod = kn.pack2(w_o)
        g_att = kn.dgrad(g_o, wod, e)
        gwo = torch.empty(e, e, device=dev)
        kn.wgrad(att, g_o, gwo)
        gbo = torch.empty(e, device=dev)
        kn.colsum(g_o, gbo)
        # attention core
        dqkv = torch.empty_like(qkv)
        kn.attention_bwd((qkv, 0, e), (qkv, e, e), (qkv, 2 * e, e), att, g_att, ctx.mask, heads, lse, (dqkv, 0, e), (dqkv, e, e), (dqkv, 2 * e, e), pd, sd[0])
        # in_proj: q, k from qk = x + pos; v from x
        _, wqkd = kn.pack2(w_in[:2 * e])
        _, wvd = kn.pack2(w_in[2 * e:])
        g_qk = kn.dgrad((dqkv, 0, 2 * e), wqkd, e)
        g_x = kn.dgrad((dqkv, 2 * e, e), wvd, e, addend=g_y1)
        g_src = kn.add(g_x, g_qk)
        gw_in = torch.empty(3 * e, e, device=dev)
        kn.wgrad(qk, (dqkv, 0, 2 * e), gw_in[:2 * e])
        kn.wgrad(x, (dqkv, 2 * e, e), gw_in[2 * e:])
        gb_in = torch.empty(3 * e, device=dev)
        kn.colsum(dqkv, gb_in)
        grads = (gw_in, gb_in, gwo, gbo, gw1, gb1, gw2, gb2_lin, gg1, gb1n, gg2, gb2)
        return (None, _lb(g_src), _lb(g_qk) if ctx.has_pos else None, None) + grads


class _DecoderLayerFn(torch.autograd.Function):
    """TransformerDecoderLayer.forward_post (detr_backbone.py:221-242) and its backward on the same kernels as `_EncoderLayerFn`:
    self-attention block, cross-attention block (queries from the decoder stream, keys / values from the encoder memory), FFN block"""

    NAMES = ("self_attn.in_proj_weight", "self_attn.in_proj_bias", "self_attn.out_proj.weight", "self_attn.out_proj.bias",
             "multihead_attn.in_proj_weight", "multihead_attn.in_proj_bias", "multihead_attn.out_proj.weight", "multihead_attn.out_proj.bias",
             "linear1.weight", "linear1.bias", "linear2.weight", "linear2.bias", "norm1.weight", "norm1.bias", "norm2.weight", "norm2.bias", "norm3.weight", "norm3.bias")

    @staticmethod
    def forward(ctx, layer, tgt, memory, pos, query_pos, tgt_mask, mem_mask, *params):
        kn, e, heads = layer.k, layer.d_model, layer.nhead
        ws, bs, wso, bso, wc, bc, wco, bco, w1, b1, w2, b2, g1, be1, g2, be2, g3, be3 = params
        x = _bl(tgt)
        qp = None if query_pos is None else _bl(query_pos)
        qk = x if qp is None else kn.add(x, qp)
        b, _, lq, _ = x.shape
        qkv = torch.empty(b, 1, lq, 3 * e, dtype=torch.bfloat16, device=x.device)
        kn.linear(qk, ws[:2 * e], bs[:2 * e], out=qkv, out_off=0)
        kn.linear(x, ws[2 * e:], bs[2 * e:], out=qkv, out_off=2 * e)
        pd, sd = layer._dropout_state(6)  # self-attention probabilities, dropout1, cross-attention probabilities, dropout2, FFN dropout, dropout3
        att1, lse1 = kn.attention_train((qkv, 0, e), (qkv, e, e), (qkv, 2 * e, e), tgt_mask, heads, pd, sd[0])
        y1 = kn.dropout(kn.linear(att1, wso, bso), pd, sd[1], residual=x) if pd > 0 else kn.linear(att1, wso, bso, residual=x)
        x1, st1 = kn.layernorm_train(y1, g1, be1)
        mem = _bl(memory)
        memk = mem if pos is None else kn.add(mem, _bl(pos))
        q2 = x1 if qp is None else kn.add(x1, qp)
        qc = kn.linear(q2, wc[:e], bc[:e])
        lk = mem.shape[2]
        kv = torch.empty(b, 1, lk, 2 * e, dtype=torch.bfloat16, device=x.device)
        kn.linear(memk, wc[e:2 * e], bc[e:2 * e], out=kv, out_off=0)
        kn.linear(mem, wc[2 * e:], bc[2 * e:], out=kv, out_off=e)
        att2, lse2 = kn.attention_train((qc, 0, e), (kv, 0, e), (kv, e, e), mem_mask, heads, pd, sd[2])
        y2 = kn.dropout(kn.linear(att2, wco, bco), pd, sd[3], residual=x1) if pd > 0 else kn.linear(att2, wco, bco, residual=x1)
        x2, st2 = kn.layernorm_train(y2, g2, be2)
        h = kn.linear(x2, w1, b1, relu=True)
        if pd > 0:
            h = kn.dropout(h, pd, sd[4])
            y3 = kn.dropout(kn.linear(h, w2, b2), pd, sd[5], residual=x2)
        else:
            y3 = kn.linear(h, w2, b2, residual=x2)
        out, st3 = kn.layernorm_train(y3, g3, be3)
        ctx.drop = (pd, sd)
        ctx.layer, ctx.masks, ctx.has = layer, (tgt_mask, mem_mask), (pos is not None, query_pos is not None)
        ctx.saved = (x, qk, qkv, att1, lse1, y1, st1, x1, mem, memk, q2, qc, kv, att2, lse2, y2, st2, x2, h, y3, st3)
        ctx.params = params
        return _lb(out)

    @staticmethod
    def backward(ctx, g_out):
        layer = ctx.layer
        kn, e, heads = layer.k, layer.d_model, layer.nhead
        x, qk, qkv, att1, lse1, y1, st1, x1, mem, memk, q2, qc, kv, att2, lse2, y2, st2, x2, h, y3, st3 = ctx.saved
        ws, bs, wso, bso, wc, bc, wco, bco, w1, b1, w2, b2, g1, be1, g2, be2, g3, be3 = ctx.params
        tgt_mask, mem_mask = ctx.masks
        has_pos, has_qpos = ctx.has
        dev, ff = x.device, w1.shape[0]
        f32 = lambda *shape: torch.empty(*shape, device=dev)
        g = _bl(g_out)
        # FFN block
        pd, sd = ctx.drop
        g_y3, gg3, gbn3 = kn.layernorm_bwd(g, y3, st3, g3)
        g_t = kn.dropout(g_y3, pd, sd[5]) if pd > 0 else g_y3
        du, gb1 = kn.dgrad_relu(g_t, kn.pack2(w2)[1], h)
        if pd > 0:
            du = kn.dropout(du, pd, sd[4])
            gb1 = gb1 / (1.0 - pd)
        gw2, gb2 = f32(e, ff), f32(e)
        kn.wgrad(h, g_t, gw2)
        kn.colsum(g_t, gb2)
        g_x2 = kn.dgrad(du, kn.pack2(w1)[1], e, addend=g_y3)
        gw1 = f32(ff, e)
        kn.wgrad(x2, du, gw1)
        # cross-attention block
        g_y2, gg2, gbn2 = kn.layernorm_bwd(g_x2, y2, st2, g2)
        g_o2 = kn.dropout(g_y2, pd, sd[3]) if pd > 0 else g_y2
        g_att2 = kn.dgrad(g_o2, kn.pack2(wco)[1], e)
        gwco, gbco = f32(e, e), f32(e)
        kn.wgrad(att2, g_o2, gwco)
        kn.colsum(g_o2, gbco)
        dqc, dkv = torch.empty_like(qc), torch.empty_like(kv)
        kn.attention_bwd((qc, 0, e), (kv, 0, e), (kv, e, e), att2, g_att2, mem_mask, heads, lse2, (dqc, 0, e), (dkv, 0, e), (dkv, e, e), pd, sd[2])
        g_q2 = kn.dgrad(dqc, kn.pack2(wc[:e])[1], e)
        g_memk = kn.dgrad((dkv, 0, e), kn.pack2(wc[e:2 * e])[1], e)
        g_mem = kn.dgrad((dkv, e, e), kn.pack2(wc[2 * e:])[1], e, addend=g_memk)  # memory feeds keys (through + pos) and values
        gwc, gbc = f32(3 * e, e), f32(3 * e)
        kn.wgrad(q2, dqc, gwc[:e])
        kn.wgrad(memk, (dkv, 0, e), gwc[e:2 * e])
        kn.wgrad(mem, (dkv, e, e), gwc[2 * e:])
        kn.colsum(dqc, gbc[:e])
        kn.colsum(dkv, gbc[e:])
        g_x1 = kn.add(g_y2, g_q2)  # residual branch + query path
        # self-attention block
        g_y1, gg1, gbn1 = kn.layernorm_bwd(g_x1, y1, st1, g1)
        g_o1 = kn.dropout(g_y1, pd, sd[1]) if pd > 0 else g_y1
        g_att1 = kn.dgrad(g_o1, kn.pack2(wso)[1], e)
        gwso, gbso = f32(e, e), f32(e)
        kn.wgrad(att1, g_o1, gwso)
        kn.colsum(g_o1, gbso)
        dqkv = torch.empty_like(qkv)
        kn.attention_bwd((qkv, 0, e), (qkv, e, e), (qkv, 2 * e, e), att1, g_att1, tgt_mask, heads, lse1, (dqkv, 0, e), (dqkv, e, e), (dqkv, 2 * e, e), pd, sd[0])
        g_qk = kn.dgrad((dqkv, 0, 2 * e), kn.pack2(ws[:2 * e])[1], e)
        g_x = kn.dgrad((dqkv, 2 * e, e), kn.pack2(ws[2 * e:])[1], e, addend=g_y1)
        g_tgt = kn.add(g_x, g_qk)
        gws, gbs = f32(3 * e, e), f32(3 * e)
        kn.wgrad(qk, (dqkv, 0, 2 * e), gws[:2 * e])
        kn.wgrad(x, (dqkv, 2 * e, e), gws[2 * e:])
        kn.colsum(dqkv, gbs)
        g_qpos = _lb(kn.add(g_qk, g_q2)) if has_qpos else None
        grads = (gws, gbs, gwso, gbso, gwc, gbc, gwco, gbco, gw1, gb1, gw2, gb2, gg1, gbn1, gg2, gbn2, gg3, gbn3)
        return (None, _lb(g_tgt), _lb(g_mem), _lb(g_memk) if has_pos else None, g_qpos, None, None) + grads


class TransformerEncoderLayer(_LayerBase):
    """detr_backbone.py:128-187"""

    def __init__(self, d_model, nhead, dim_feedforward=2048, dropout=0.1, activation="relu", normalize_before=False, device="cuda"):
        super().__init__(d_model, nhead, dim_feedforward, dropout, activation, normalize_before, device)
        self.self_attn = _MhaParams(d_model, device)
        self.norm1, self.norm2 = _Norm(d_model, device), _Norm(d_model, device)

    def forward(self, src, src_mask=None, src_key_padding_mask=None, pos=None):
        if src_mask is not None:
            raise capi.Yb200Error("attn_mask is not supported (the reference's DETR never passes one)")
        if not src.is_cuda:
            raise capi.Yb200Error("DETR layers: inputs must be CUDA tensors (no CPU path)")
        if TRAINING_PATH and torch.is_grad_enabled():
            params = [dict(self.named_parameters())[n] for n in _EncoderLayerFn.NAMES]
            if src.requires_grad or any(p.requires_grad for p in params):
                return _EncoderLayerFn.apply(self, src, pos, _mask_u8(src_key_padding_mask), *params)
        with torch.no_grad():
            return self._forward_inference(src, src_key_padding_mask, pos)

    def _forward_inference(self, src, src_key_padding_mask, pos):
        _check_inputs(src, pos)
        x = _bl(src)
        qk = x if pos is None else self.k.add(x, _bl(pos))
        y = self._self_attention(x, qk, self.self_attn, _mask_u8(src_key_padding_mask))
        x1 = self.k.layernorm(y, self.norm1.weight, self.norm1.bias)
        return _lb(self._ffn(x1, self.norm2))


class TransformerDecoderLayer(_LayerBase):
    """detr_backbone.py:190-279"""

    def __init__(self, d_model, nhead, dim_feedforward=2048, dropout=0.1, activation="relu", normalize_before=False, device="cuda"):
        super().__init__(d_model, nhead, dim_feedforward, dropout, activation, normalize_before, device)
        self.self_attn = _MhaParams(d_model, device)
        self.multihead_attn = _MhaParams(d_model, device)
        self.norm1, self.norm2, self.norm3 = _Norm(d_model, device), _Norm(d_model, device), _Norm(d_model, device)

    def forward(self, tgt, memory, tgt_mask=None, memory_mask=None, tgt_key_padding_mask=None, memory_key_padding_mask=None, pos=None, query_pos=None):
        if tgt_mask is not None or memory_mask is not None:
            raise capi.Yb200Error("attn_mask is not supported (the reference's DETR never passes one)")
        if TRAINING_PATH and torch.is_grad_enabled():
            params = [dict(self.named_parameters())[n] for n in _DecoderLayerFn.NAMES]
            if tgt.requires_grad or memory.requires_grad or any(p.requires_grad for p in params):
                return _DecoderLayerFn.apply(self, tgt, memory, pos, query_pos, _mask_u8(tgt_key_padding_mask), _mask_u8(memory_key_padding_mask), *params)
        with torch.no_grad():
            return self._forward_inference(tgt, memory, tgt_key_padding_mask, memory_key_padding_mask, pos, query_pos)

    def _forward_inference(self, tgt, memory, tgt_key_padding_mask, memory_key_padding_mask, pos, query_pos):
        _check_inputs(tgt, memory, pos, query_pos)
        kn, e = self.k, self.d_model
        x = _bl(tgt)
        qp = None if query_pos is None else _bl(query_pos)
        qk = x if qp is None else kn.add(x, qp)
        x = kn.layernorm(self._self_attention(x, qk, self.self_attn, _mask_u8(tgt_key_padding_mask)), self.norm1.weight, self.norm1.bias)
        # cross attention: queries from the decoder stream, keys / values from the encoder memory
        mem = _bl(memory)
        memk = mem if pos is None else kn.add(mem, _bl(pos))
        att = self.multihead_attn
        w, bias = att.in_proj_weight, att.in_proj_bias
        q = kn.linear(x if qp is None else kn.add(x, qp), w[:e], bias[:e])
        b, _, lk, _ = mem.shape
        kv = torch.empty(b, 1, lk, 2 * e, dtype=torch.bfloat16, device=mem.device)
        kn.linear(memk, w[e:2 * e], bias[e:2 * e], out=kv, out_off=0)
        kn.linear(mem, w[2 * e:], bias[2 * e:], out=kv, out_off=e)
        a = kn.attention((q, 0, e), (kv, 0, e), (kv, e, e), _mask_u8(memory_key_padding_mask), self.nhead)
        x = kn.layernorm(kn.linear(a, att.out_proj.weight, att.out_proj.bias, residual=x), self.norm2.weight, self.norm2.bias)
        return _lb(self._ffn(x, self.norm3))


# ------------------------------------------------------------------------------------------------------------------------------------
# the stack: Transformer / TransformerEncoder / TransformerDecoder   (detr_backbone.py:25-126)
# ------------------------------------------------------------------------------------------------------------------------------------
class _LayerNormFn(torch.autograd.Function):
    """nn.LayerNorm over the last dimension of a seq-first [L, B, E] fp32 tensor on the LayerNorm kernels (forward + backward)"""

    @staticmethod
    def forward(ctx, k, x, weight, bias):
        xb = _bl(x)
        y, stats = k.layernorm_train(xb, weight, bias)
        ctx.k = k
        ctx.save_for_backward(xb, stats, weight)
        return _lb(y)

    @staticmethod
    def backward(ctx, g):
        xb, stats, weight = ctx.saved_tensors
        dx, gw, gb = ctx.k.layernorm_bwd(_bl(g), xb, stats, weight)
        return None, _lb(dx), gw, gb


class LayerNorm(nn.Module):
    """`nn.LayerNorm(d_model)` of the stack (the decoder's final / intermediate norm, detr_backbone.py:37-41,118-124)"""

    def __init__(self, d_model, device="cuda"):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(d_model, device=device))
        self.bias = nn.Parameter(torch.zeros(d_model, device=device))
        self.k = _Kernels()

    def forward(self, x):
        if not x.is_cuda:
            raise capi.Yb200Error("DETR layers: inputs must be CUDA tensors (no CPU path)")
        if TRAINING_PATH and torch.is_grad_enabled() and (x.requires_grad or self.weight.requires_grad):
            return _LayerNormFn.apply(self.k, x, self.weight, self.bias)
        with torch.no_grad():
            return _lb(self.k.layernorm(_bl(x), self.weight, self.bias))


def _clone_layer(layer):
    """`_get_clones` (detr_backbone.py:281-282): a new layer of the same shape carrying a copy of the prototype's parameters"""
    new = type(layer)(*layer._ctor)
    new.load_state_dict(layer.state_dict())
    return new


class TransformerEncoder(nn.Module):
    """detr_backbone.py:69-90; `layers` are independent TransformerEncoderLayer modules (the reference deep-copies one prototype)"""

    def __init__(self, encoder_layer, num_layers, norm=None):
        super().__init__()
        self.layers = nn.ModuleList([encoder_layer] + [_clone_layer(encoder_layer) for _ in range(num_layers - 1)])
        self.num_layers = num_layers
        self.norm = norm

    def forward(self, src, mask=None, src_key_padding_mask=None, pos=None):
        output = src
        for layer in self.layers:
            output = layer(output, src_mask=mask, src_key_padding_mask=src_key_padding_mask, pos=pos)
        if self.norm is not None:
            output = self.norm(output)
        return output


class TransformerDecoder(nn.Module):
    """detr_backbone.py:93-126: optional stack of the normalised intermediate outputs (auxiliary losses of DETR)"""

    def __init__(self, decoder_layer, num_layers, norm=None, return_intermediate=False):
        super().__init__()
        self.layers = nn.ModuleList([decoder_layer] + [_clone_layer(decoder_layer) for _ in range(num_layers - 1)])
        self.num_layers = num_layers
        self.norm = norm
        self.return_intermediate = return_intermediate

    def forward(self, tgt, memory, tgt_mask=None, memory_mask=None, tgt_key_padding_mask=None, memory_key_padding_mask=None, pos=None, query_pos=None):
        output = tgt
        intermediate = []
        for layer in self.layers:
            output = layer(output, memory, tgt_mask=tgt_mask, memory_mask=memory_mask, tgt_key_padding_mask=tgt_key_padding_mask,
                           memory_key_padding_mask=memory_key_padding_mask, pos=pos, query_pos=query_pos)
            if self.return_intermediate:
                intermediate.append(self.norm(output))
        if self.norm is not None:
            output = self.norm(output)
            if self.return_intermediate:
                intermediate.pop()
                intermediate.append(output)
        if self.return_intermediate:
            return torch.stack(intermediate)
        return output.unsqueeze(0)


class Transformer(nn.Module):
    """detr_backbone.py:25-66: encoder stack over the flattened feature map, decoder stack over the object queries.
    forward(src [B,C,H,W], mask [B,H,W] bool, query_embed [Q,C], pos_embed [B,C,H,W]) -> (hs [layers or 1, B, Q, C], memory [B,C,H,W]).
    Dropout (0.1 in the reference) is active in training mode (`_LayerBase._dropout_state`); normalize_before is not supported."""

    def __init__(self, d_model=512, nhead=8, num_encoder_layers=6, num_decoder_layers=6, dim_feedforward=2048, dropout=0.1, activation="relu",
                 normalize_before=False, return_intermediate_dec=False, device="cuda"):
        super().__init__()
        if normalize_before:
            raise capi.Yb200Error("normalize_before=True (pre-norm) is not implemented by the DETR layers of this package")
        enc = TransformerEncoderLayer(d_model, nhead, dim_feedforward, dropout, activation, normalize_before, device)
        self.encoder = TransformerEncoder(enc, num_encoder_layers, None)
        dec = TransformerDecoderLayer(d_model, nhead, dim_feedforward, dropout, activation, normalize_before, device)
        self.decoder = TransformerDecoder(dec, num_decoder_layers, LayerNorm(d_model, device), return_intermediate=return_intermediate_dec)
        self._reset_parameters()
        self.d_model, self.nhead = d_model, nhead

    def _reset_parameters(self):
        for p in self.parameters():
            if p.dim() > 1:
                nn.init.xavier_uniform_(p)

    def forward(self, src, mask, query_embed, pos_embed):
        bs, c, h, w = src.shape
        src = src.flatten(2).permute(2, 0, 1)
        pos_embed = pos_embed.flatten(2).permute(2, 0, 1)
        query_embed = query_embed.unsqueeze(1).repeat(1, bs, 1)
        mask = mask.flatten(1)
        tgt = torch.zeros_like(query_embed)
        memory = self.encoder(src, src_key_padding_mask=mask, pos=pos_embed)
        hs = self.decoder(tgt, memory, memory_key_padding_mask=mask, pos=pos_embed, query_pos=query_embed)
        return hs.transpose(1, 2), memory.permute(1, 2, 0).view(bs, c, h, w)


# ------------------------------------------------------------------------------------------------------------------------------------
# the DETR tail: input_proj, class_embed, bbox_embed   (yolov7/modeling/meta_arch/detr.py:282-294, 406-472)
# ------------------------------------------------------------------------------------------------------------------------------------
def _pad16(n):
    return (n + 15) // 16 * 16


class _LinearStackFn(torch.autograd.Function):
    """x [..., in] fp32 -> Linear (+ReLU) ... Linear -> [..., out] fp32, every row of x in one GEMM per layer (bf16 operands, fp32 bias and
    accumulation).  The last layer's output channels are padded to a multiple of 16 for the GEMMs and sliced off.  Backward: ReLU-masked data
    gradients with fused bias sums, weight gradients and column sums on the same kernels as the transformer layers."""

    @staticmethod
    def forward(ctx, kn, x, *params):
        ws, bs = params[0::2], params[1::2]
        lead, cin = x.shape[:-1], x.shape[-1]
        if cin % 16 or any(w.shape[0] % 16 for w in ws[:-1]):
            raise capi.Yb200Error(f"Linear stack: input {cin} and hidden widths {[w.shape[0] for w in ws[:-1]]} must be multiples of 16")
        n = x.numel() // cin
        h = x.detach().reshape(1, 1, n, cin).to(torch.bfloat16).contiguous()
        hs, wds = [h], []
        for i, (w, b) in enumerate(zip(ws, bs)):
            last = i == len(ws) - 1
            cout, cpad = w.shape[0], _pad16(w.shape[0])
            wf = torch.empty(cpad, 1, w.shape[1], dtype=torch.bfloat16, device=x.device)
            wd = torch.empty(w.shape[1], 1, cpad, dtype=torch.bfloat16, device=x.device)
            capi.check(kn.L.yb200_pack_conv_weight(capi.ptr(w.detach().contiguous()), cout, w.shape[1], 1, cpad, w.shape[1], capi.ptr(wf), capi.ptr(wd),
                                                   capi.stream_ptr()), "pack")
            bias = torch.zeros(cpad, device=x.device)
            bias[:cout] = b.detach()
            out = torch.empty(1, 1, n, cpad, dtype=torch.bfloat16, device=x.device)
            ha, oa = kn._a(h), kn._a(out)
            if last:
                capi.check(kn.L.yb200_conv2d_affine_fwd(ctypes.byref(ha), capi.ptr(wf), None, capi.ptr(bias), None, ctypes.byref(oa), 1, 1, capi.stream_ptr()),
                           "linear")
            else:
                capi.check(kn.L.yb200_linear_relu_fwd(ctypes.byref(ha), capi.ptr(wf), capi.ptr(bias), ctypes.byref(oa), capi.stream_ptr()), "linear+relu")
            wds.append(wd)
            h = out
            if not last:
                hs.append(h)
        ctx.kn, ctx.hs, ctx.wds, ctx.couts, ctx.lead, ctx.cin = kn, hs, wds, [w.shape[0] for w in ws], lead, cin
        cout = ws[-1].shape[0]
        return h[0, 0, :, :cout].float().reshape(*lead, cout)

    @staticmethod
    def backward(ctx, g):
        kn, hs, wds, couts = ctx.kn, ctx.hs, ctx.wds, ctx.couts
        n, dev = hs[0].shape[2], g.device
        d = torch.zeros(1, 1, n, _pad16(couts[-1]), dtype=torch.bfloat16, device=dev)
        d[0, 0, :, :couts[-1]] = g.reshape(n, couts[-1])
        grads = [None] * (2 * len(couts))
        gb = torch.empty(d.shape[-1], device=dev)
        kn.colsum(d, gb)
        grads[-1] = gb[:couts[-1]]
        for i in range(len(couts) - 1, -1, -1):
            gw = torch.empty(d.shape[-1], hs[i].shape[-1], device=dev)
            kn.wgrad(hs[i], d, gw)
            grads[2 * i] = gw[:couts[i]]
            if i > 0:
                d, grads[2 * i - 1] = kn.dgrad_relu(d, wds[i], hs[i])
            else:
                dx = kn.dgrad(d, wds[0], ctx.cin)
        return (None, dx.float().reshape(*ctx.lead, ctx.cin)) + tuple(grads)


def _linear_stack(kn, x, linears):
    if not x.is_cuda:
        raise capi.Yb200Error("DETR heads: inputs must be CUDA tensors (no CPU path)")
    return _LinearStackFn.apply(kn, x, *[p for lin in linears for p in (lin.weight, lin.bias)])


class MLP(nn.Module):
    """detr.py:282-294: Linear + ReLU ... Linear over the last dimension, all rows in one GEMM per layer"""

    def __init__(self, input_dim, hidden_dim, output_dim, num_layers):
        super().__init__()
        self.num_layers = num_layers
        h = [hidden_dim] * (num_layers - 1)
        self.layers = nn.ModuleList(nn.Linear(n, k) for n, k in zip([input_dim] + h, h + [output_dim]))
        self.k = _Kernels()

    def forward(self, x):
        return _linear_stack(self.k, x, self.layers)


class DETR(nn.Module):
    """detr.py:406-472.  `backbone` is the caller's module, called as the reference calls it (features, pos = backbone(samples);
    src, mask = features[-1].decompose()); `transformer` is this package's Transformer (return_intermediate_dec = deep supervision).
    input_proj (1x1 convolution) and the heads run as GEMMs over every pixel / every (layer, image, query) row at once; pred_logits and
    pred_boxes are fp32."""

    def __init__(self, backbone, transformer, num_classes, num_queries, aux_loss=False):
        super().__init__()
        self.num_queries = num_queries
        self.transformer = transformer
        hidden_dim = transformer.d_model
        self.class_embed = nn.Linear(hidden_dim, num_classes + 1)
        self.bbox_embed = MLP(hidden_dim, hidden_dim, 4, 3)
        self.query_embed = nn.Embedding(num_queries, hidden_dim)
        self.input_proj = nn.Conv2d(backbone.num_channels, hidden_dim, kernel_size=1)
        self.backbone = backbone
        self.aux_loss = aux_loss
        self.onnx_export = False
        self.k = self.bbox_embed.k

    def forward(self, samples):
        if isinstance(samples, (list, torch.Tensor)):
            raise capi.Yb200Error("DETR: pass a NestedTensor / ImageList with its padding mask (raw tensors and lists are not supported)")
        features, pos = self.backbone(samples)
        src, mask = features[-1].decompose()
        assert mask is not None
        conv = self.input_proj
        proj_lin = types.SimpleNamespace(weight=conv.weight.view(conv.weight.shape[0], -1), bias=conv.bias)
        proj = _linear_stack(self.k, src.permute(0, 2, 3, 1), [proj_lin]).permute(0, 3, 1, 2)
        hs = self.transformer(proj, mask, self.query_embed.weight, pos[-1])[0]
        outputs_class = _linear_stack(self.k, hs, [self.class_embed])
        outputs_coord = torch.sigmoid(self.bbox_embed(hs))
        out = {"pred_logits": outputs_class[-1], "pred_boxes": outputs_coord[-1]}
        if self.aux_loss:
            out["aux_outputs"] = [{"pred_logits": a, "pred_boxes": b} for a, b in zip(outputs_class[:-1], outputs_coord[:-1])]
        return out
