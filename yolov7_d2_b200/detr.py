"""DETR transformer layers on the H100 kernels (forward path; SURVEY.md par.8a row T1).

Reference: yolov7/modeling/backbone/detr_backbone.py -- `TransformerEncoderLayer` :128-187 (forward_post :157-170), `TransformerDecoderLayer`
:190-279 (forward_post :221-242); both wrap torch's nn.MultiheadAttention (:140, :200-202).  The classes below keep the reference's
constructor arguments, parameter names / shapes (`self_attn.in_proj_weight` [3E,E], `linear1.weight`, `norm1.weight` ...) and the seq-first
`[L, B, E]` fp32 interface, and run

    x (+pos) -> in_proj GEMMs (bias epilogue, q|k|v packed in one [B, L, 3E] buffer) -> yb200_attention_fwd (wgmma, streaming softmax)
      -> out_proj GEMM (+bias +residual epilogue) -> LayerNorm -> linear1 GEMM (+bias +ReLU epilogue) -> linear2 GEMM (+bias +residual) -> LayerNorm

Internally tokens are batch-first bf16 `[B, 1, L, E]` views (yb200_act).  Each layer is built from two blocks, each with one forward and one
backward: the attention block (`_attention_fwd` / `_attention_bwd`, self- or cross-attention) and the FFN block (`_ffn_fwd` / `_ffn_bwd`).
With gradients enabled the layers run as one autograd node each (`_EncoderLayerFn` / `_DecoderLayerFn`: attention backward, data / weight
gradients and LayerNorm backward on the same kernels), validated on hardware against the reference layer's autograd (tests/test_detr_gpu.py);
without autograd they run the same block forwards without keeping the log-sum-exp or the LayerNorm statistics.
Dropout (p = 0.1 in the reference: on the attention probabilities inside nn.MultiheadAttention and nn.Dropout on the residual branches / in the FFN) is
active in training mode: the masks are a counter-based hash of (seed, element index) evaluated inside the kernels (yb200_attention_*_dropout,
yb200_dropout), regenerated in the backward from the same seeds; seeds come from torch's CPU generator.  Same distribution as torch's Philox masks, not
the same bits: parity = the same computation given the same mask (tests/test_detr_dropout_gpu.py, oracle/detr_oracle.py).  `attn_mask` (never passed by the
reference's DETR) and `normalize_before=True` are not supported.  There is no CPU implementation.
"""
import ctypes
import operator
import types

import torch
import torch.nn as nn

from . import capi

LN_EPS = 1e-5
# (p, seeds) of a forward without autograd: it runs dropout-free, and draws no seeds from torch's generator
_NO_DROPOUT = (0.0, (0,) * 6)


def _bl(t):
    """[L, B, E] (any float dtype, CUDA) -> contiguous bf16 [B, 1, L, E]"""
    return t.detach().permute(1, 0, 2).to(torch.bfloat16).contiguous().unsqueeze(1)


def _lb(t):
    """[B, 1, L, E] bf16 -> [L, B, E] fp32"""
    return t.squeeze(1).permute(1, 0, 2).float().contiguous()


def _f32(*shape, device):
    return torch.empty(*shape, device=device)


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

    def pack2(self, w, rows=None):
        """[out, in] fp32 -> bf16 forward [rows, 1, in] and data-gradient [in, 1, rows] GEMM operands; rows > out pads with zero rows"""
        out_f, in_f = w.shape
        rows = out_f if rows is None else rows
        wf = torch.empty(rows, 1, in_f, dtype=torch.bfloat16, device=w.device)
        wd = torch.empty(in_f, 1, rows, dtype=torch.bfloat16, device=w.device)
        capi.check(self.L.yb200_pack_conv_weight(capi.ptr(w.detach().contiguous()), out_f, in_f, 1, rows, in_f, capi.ptr(wf), capi.ptr(wd), capi.stream_ptr()), "pack")
        return wf, wd

    def add(self, a, b):
        out = torch.empty_like(a)
        aa, ba, oa = self._a(a), self._a(b), self._a(out)
        capi.check(self.L.yb200_add(ctypes.byref(aa), ctypes.byref(ba), ctypes.byref(oa), capi.stream_ptr()), "add")
        return out

    def linear(self, x, w, bias, out=None, out_off=0, residual=None, relu=False):
        """out[..., out_off:out_off+N] = x W^T + bias (+ residual) (ReLU); x may be a (tensor, off, c) slice; w is an [N, in] fp32 weight or the
        forward operand from pack2"""
        xt, xo, xc = x if isinstance(x, tuple) else (x, 0, None)
        n_out = w.shape[0]
        b, _, l, _ = xt.shape
        if out is None:
            out = torch.empty(b, 1, l, n_out, dtype=torch.bfloat16, device=xt.device)
        xa, oa = self._a(xt, xo, xc), self._a(out, out_off, n_out)
        wf = w if w.dim() == 3 else self.pack(w)
        bias = bias.detach().contiguous()
        if relu:
            capi.check(self.L.yb200_linear_relu_fwd(ctypes.byref(xa), capi.ptr(wf), capi.ptr(bias), ctypes.byref(oa), capi.stream_ptr()), "linear+relu")
        else:
            ra = self._a(residual) if residual is not None else None
            capi.check(self.L.yb200_conv2d_affine_fwd(ctypes.byref(xa), capi.ptr(wf), None, capi.ptr(bias), ctypes.byref(ra) if ra is not None else None,
                                                      ctypes.byref(oa), 1, 1, capi.stream_ptr()), "linear")
        return out

    def layernorm(self, x, weight, bias, save=False):
        """save: also return the per-row (mean, rstd) that layernorm_bwd needs (else None)"""
        b, _, l, _ = x.shape
        y = torch.empty_like(x)
        stats = torch.empty(b * l, 2, device=x.device) if save else None
        xa, ya = self._a(x), self._a(y)
        capi.check(self.L.yb200_layernorm_fwd(ctypes.byref(xa), capi.ptr(weight.detach().contiguous()), capi.ptr(bias.detach().contiguous()), ctypes.c_float(LN_EPS),
                                              ctypes.byref(ya), capi.ptr(stats), capi.stream_ptr()), "layernorm")
        return y, stats

    def layernorm_train(self, x, weight, bias):
        """the forward of the autograd path: keeps the statistics"""
        return self.layernorm(x, weight, bias, save=True)

    def _ws(self, nbytes, dev):
        return torch.empty(max(int(nbytes), 16), dtype=torch.uint8, device=dev)

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

    def attention(self, q, k, v, mask, heads, p_drop=0.0, seed=0, save=False):
        """q, k, v: (tensor, channel offset, E) slices of [B,1,L,*] buffers; mask: uint8 [B, Lk] or None.  p_drop > 0: dropout on the attention
        probabilities (nn.MultiheadAttention(dropout=p), detr_backbone.py:140), mask = f(seed, b, h, q, k).  save: also return the log-sum-exp
        that attention_bwd needs (else None)"""
        qt, _, e = q
        b, _, lq, _ = qt.shape
        out = torch.empty(b, 1, lq, e, dtype=torch.bfloat16, device=qt.device)
        lse = torch.empty(b, heads, lq, device=qt.device) if save else None
        qa, ka, va, oa = self._a(*q), self._a(*k), self._a(*v), self._a(out)
        capi.check(self.L.yb200_attention_fwd_dropout(ctypes.byref(qa), ctypes.byref(ka), ctypes.byref(va), capi.ptr(mask), ctypes.c_float((e // heads) ** -0.5),
                                                      ctypes.byref(oa), capi.ptr(lse), ctypes.c_float(p_drop), ctypes.c_uint32(seed), capi.stream_ptr()), "attention")
        return out, lse

    def attention_train(self, q, k, v, mask, heads, p_drop=0.0, seed=0):
        """the forward of the autograd path: keeps the log-sum-exp"""
        return self.attention(q, k, v, mask, heads, p_drop, seed, save=True)

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


def _check_devices(*tensors):
    """the kernels take raw device pointers: every tensor argument of a layer is a CUDA tensor, all on one device"""
    devices = {t.device for t in tensors if t is not None}
    if any(d.type != "cuda" for d in devices):
        raise capi.Yb200Error("DETR layers: inputs must be CUDA tensors (no CPU path)")
    if len(devices) > 1:
        raise capi.Yb200Error(f"DETR layers: inputs on more than one device ({', '.join(sorted(map(str, devices)))})")


def _records(*tensors):
    """autograd is recording and one of the tensors requires grad: the layer runs as one autograd node"""
    return torch.is_grad_enabled() and any(t.requires_grad for t in tensors)


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


# ------------------------------------------------------------------------------------------------------------------------------------
# the blocks of forward_post (detr_backbone.py:157-170, 221-242).  A forward returns its output and, with save, what its backward needs
# (the block's parameters, dropout state and bf16 intermediates); a backward returns the input gradients and the parameter gradients.
# p = (in / linear1 weight, bias, out_proj / linear2 weight, bias, LayerNorm weight, bias); seeds = the block's two dropout seeds.
# ------------------------------------------------------------------------------------------------------------------------------------
def _linear_residual(kn, x, w, b, res, pd, seed):
    """res + dropout(x W^T + b): the residual joins in the GEMM epilogue, or in the dropout kernel when p > 0"""
    if pd > 0:
        return kn.dropout(kn.linear(x, w, b), pd, seed, residual=res)
    return kn.linear(x, w, b, residual=res)


def _attention_fwd(kn, heads, x, q_src, kv_src, mask, p, pd, seeds, save):
    """in-projection GEMMs -> attention core (dropout seeds[0]) -> out_proj (dropout seeds[1]) + residual x -> LayerNorm.
    Self-attention (kv_src None): q|k from q_src in one [.., 2E] GEMM and v from x, into one [.., 3E] buffer.
    Cross-attention (kv_src = (key source, value source)): q from q_src on its own, k and v into one [.., 2E] buffer."""
    w, b, w_o, b_o, g, be = p
    bs, _, lq, e = x.shape
    if kv_src is None:
        qkv = torch.empty(bs, 1, lq, 3 * e, dtype=torch.bfloat16, device=x.device)
        kn.linear(q_src, w[:2 * e], b[:2 * e], out=qkv, out_off=0)
        kn.linear(x, w[2 * e:], b[2 * e:], out=qkv, out_off=2 * e)
        qkv_s = ((qkv, 0, e), (qkv, e, e), (qkv, 2 * e, e))
    else:
        k_src, v_src = kv_src
        qc = kn.linear(q_src, w[:e], b[:e])
        kv = torch.empty(bs, 1, k_src.shape[2], 2 * e, dtype=torch.bfloat16, device=x.device)
        kn.linear(k_src, w[e:2 * e], b[e:2 * e], out=kv, out_off=0)
        kn.linear(v_src, w[2 * e:], b[2 * e:], out=kv, out_off=e)
        qkv_s = ((qc, 0, e), (kv, 0, e), (kv, e, e))
    att, lse = (kn.attention_train if save else kn.attention)(*qkv_s, mask, heads, pd, seeds[0])
    y = _linear_residual(kn, att, w_o, b_o, x, pd, seeds[1])
    out, st = (kn.layernorm_train if save else kn.layernorm)(y, g, be)
    return out, ((p, pd, seeds, mask, x, q_src, kv_src, qkv_s, att, lse, y, st) if save else None)


def _attention_bwd(kn, heads, g, saved):
    """-> (gradient of x, gradient of q_src, for cross-attention (gradient of the value source, gradient of the key source) else None,
    parameter gradients).  x feeds the residual and the queries (q_src = x + query / positional embedding), and self-attention's keys and
    values; the value source of cross-attention also feeds its keys (key source = value source + pos), so its gradient includes the key source's."""
    (w, _, w_o, _, g_ln, _), pd, seeds, mask, x, q_src, kv_src, (q, k, v), att, lse, y, st = saved
    e, dev = x.shape[-1], x.device
    g_y, gg, gbe = kn.layernorm_bwd(g, y, st, g_ln)
    g_o = kn.dropout(g_y, pd, seeds[1]) if pd > 0 else g_y
    g_att = kn.dgrad(g_o, kn.pack2(w_o)[1], e)
    gwo, gbo = _f32(e, e, device=dev), _f32(e, device=dev)
    kn.wgrad(att, g_o, gwo)
    kn.colsum(g_o, gbo)
    gw, gb = _f32(3 * e, e, device=dev), _f32(3 * e, device=dev)
    if kv_src is None:
        dqkv = torch.empty_like(q[0])
        kn.attention_bwd(q, k, v, att, g_att, mask, heads, lse, (dqkv, 0, e), (dqkv, e, e), (dqkv, 2 * e, e), pd, seeds[0])
        g_q = kn.dgrad((dqkv, 0, 2 * e), kn.pack2(w[:2 * e])[1], e)
        g_x = kn.add(kn.dgrad((dqkv, 2 * e, e), kn.pack2(w[2 * e:])[1], e, addend=g_y), g_q)
        kn.wgrad(q_src, (dqkv, 0, 2 * e), gw[:2 * e])
        kn.wgrad(x, (dqkv, 2 * e, e), gw[2 * e:])
        kn.colsum(dqkv, gb)
        g_kv = None
    else:
        k_src, v_src = kv_src
        dqc, dkv = torch.empty_like(q[0]), torch.empty_like(k[0])
        kn.attention_bwd(q, k, v, att, g_att, mask, heads, lse, (dqc, 0, e), (dkv, 0, e), (dkv, e, e), pd, seeds[0])
        g_q = kn.dgrad(dqc, kn.pack2(w[:e])[1], e)
        g_k = kn.dgrad((dkv, 0, e), kn.pack2(w[e:2 * e])[1], e)
        g_kv = (kn.dgrad((dkv, e, e), kn.pack2(w[2 * e:])[1], e, addend=g_k), g_k)
        kn.wgrad(q_src, dqc, gw[:e])
        kn.wgrad(k_src, (dkv, 0, e), gw[e:2 * e])
        kn.wgrad(v_src, (dkv, e, e), gw[2 * e:])
        kn.colsum(dqc, gb[:e])
        kn.colsum(dkv, gb[e:])
        g_x = kn.add(g_y, g_q)
    return g_x, g_q, g_kv, (gw, gb, gwo, gbo, gg, gbe)


def _ffn_fwd(kn, x, p, pd, seeds, save):
    """linear1 + ReLU (dropout seeds[0]) -> linear2 (dropout seeds[1]) + residual x -> LayerNorm"""
    w1, b1, w2, b2, g, be = p
    h = kn.linear(x, w1, b1, relu=True)
    if pd > 0:
        h = kn.dropout(h, pd, seeds[0])  # the dropped activation is what linear2 sees and what the backward needs (h > 0 and kept)
    y = _linear_residual(kn, h, w2, b2, x, pd, seeds[1])
    out, st = (kn.layernorm_train if save else kn.layernorm)(y, g, be)
    return out, ((p, pd, seeds, x, h, y, st) if save else None)


def _ffn_bwd(kn, g, saved):
    """-> (gradient of x, parameter gradients)"""
    (w1, _, w2, _, g_ln, _), pd, seeds, x, h, y, st = saved
    e, ff, dev = x.shape[-1], w1.shape[0], x.device
    g_y, gg, gbe = kn.layernorm_bwd(g, y, st, g_ln)
    # linear2 and the ReLU in front of it; with dropout: g_t = the output dropout's mask on the branch gradient, and the saved h is the dropped
    # activation (positive <=> positive and kept), so the ReLU mask also applies the FFN dropout mask -- its 1 / (1 - p) follows
    g_t = kn.dropout(g_y, pd, seeds[1]) if pd > 0 else g_y
    du, gb1 = kn.dgrad_relu(g_t, kn.pack2(w2)[1], h)
    if pd > 0:
        du = kn.dropout(du, pd, seeds[0])
        gb1 = gb1 / (1.0 - pd)
    gw2, gb2 = _f32(e, ff, device=dev), _f32(e, device=dev)
    kn.wgrad(h, g_t, gw2)
    kn.colsum(g_t, gb2)
    # linear1; the residual branch of x joins through the addend
    g_x = kn.dgrad(du, kn.pack2(w1)[1], e, addend=g_y)
    gw1 = _f32(ff, e, device=dev)
    kn.wgrad(x, du, gw1)
    return g_x, (gw1, gb1, gw2, gb2, gg, gbe)


class _EncoderLayerFn(torch.autograd.Function):
    """forward_post (detr_backbone.py:157-170) = attention block + FFN block, with everything the backward needs kept in bf16"""

    NAMES = ("self_attn.in_proj_weight", "self_attn.in_proj_bias", "self_attn.out_proj.weight", "self_attn.out_proj.bias", "linear1.weight", "linear1.bias",
             "linear2.weight", "linear2.bias", "norm1.weight", "norm1.bias", "norm2.weight", "norm2.bias")
    PARAMS = operator.attrgetter(*NAMES)  # layer -> its parameters in NAMES order

    @staticmethod
    def run(layer, src, pos, mask, params, drop, save):
        """drop = (p, 4 seeds): attention probabilities, dropout1, FFN dropout, dropout2"""
        kn = layer.k
        w_in, b_in, w_o, b_o, w1, b1, w2, b2, g1, be1, g2, be2 = params
        pd, sd = drop
        x = _bl(src)
        qk = x if pos is None else kn.add(x, _bl(pos))
        x1, s_att = _attention_fwd(kn, layer.nhead, x, qk, None, mask, (w_in, b_in, w_o, b_o, g1, be1), pd, sd[0:2], save)
        out, s_ffn = _ffn_fwd(kn, x1, (w1, b1, w2, b2, g2, be2), pd, sd[2:4], save)
        return _lb(out), (s_att, s_ffn)

    @staticmethod
    def forward(ctx, layer, src, pos, mask, *params):
        out, ctx.saved = _EncoderLayerFn.run(layer, src, pos, mask, params, layer._dropout_state(4), True)
        ctx.layer, ctx.has_pos = layer, pos is not None
        return out

    @staticmethod
    def backward(ctx, g_out):
        kn, heads = ctx.layer.k, ctx.layer.nhead
        s_att, s_ffn = ctx.saved
        g_x1, gf = _ffn_bwd(kn, _bl(g_out), s_ffn)
        g_src, g_qk, _, ga = _attention_bwd(kn, heads, g_x1, s_att)
        grads = ga[:4] + gf[:4] + ga[4:] + gf[4:]  # NAMES order: projections, then the norms
        return (None, _lb(g_src), _lb(g_qk) if ctx.has_pos else None, None) + grads


class _DecoderLayerFn(torch.autograd.Function):
    """TransformerDecoderLayer.forward_post (detr_backbone.py:221-242) = self-attention block + cross-attention block (queries from the decoder
    stream, keys / values from the encoder memory) + FFN block, and its backward on the same kernels as `_EncoderLayerFn`"""

    NAMES = ("self_attn.in_proj_weight", "self_attn.in_proj_bias", "self_attn.out_proj.weight", "self_attn.out_proj.bias",
             "multihead_attn.in_proj_weight", "multihead_attn.in_proj_bias", "multihead_attn.out_proj.weight", "multihead_attn.out_proj.bias",
             "linear1.weight", "linear1.bias", "linear2.weight", "linear2.bias", "norm1.weight", "norm1.bias", "norm2.weight", "norm2.bias", "norm3.weight", "norm3.bias")
    PARAMS = operator.attrgetter(*NAMES)

    @staticmethod
    def run(layer, tgt, memory, pos, query_pos, tgt_mask, mem_mask, params, drop, save):
        """drop = (p, 6 seeds): self-attention probabilities, dropout1, cross-attention probabilities, dropout2, FFN dropout, dropout3"""
        kn, heads = layer.k, layer.nhead
        ws, bs, wso, bso, wc, bc, wco, bco, w1, b1, w2, b2, g1, be1, g2, be2, g3, be3 = params
        pd, sd = drop
        x = _bl(tgt)
        qp = None if query_pos is None else _bl(query_pos)
        qk = x if qp is None else kn.add(x, qp)
        x1, s_self = _attention_fwd(kn, heads, x, qk, None, tgt_mask, (ws, bs, wso, bso, g1, be1), pd, sd[0:2], save)
        mem = _bl(memory)
        memk = mem if pos is None else kn.add(mem, _bl(pos))
        q2 = x1 if qp is None else kn.add(x1, qp)
        x2, s_cross = _attention_fwd(kn, heads, x1, q2, (memk, mem), mem_mask, (wc, bc, wco, bco, g2, be2), pd, sd[2:4], save)
        out, s_ffn = _ffn_fwd(kn, x2, (w1, b1, w2, b2, g3, be3), pd, sd[4:6], save)
        return _lb(out), (s_self, s_cross, s_ffn)

    @staticmethod
    def forward(ctx, layer, tgt, memory, pos, query_pos, tgt_mask, mem_mask, *params):
        out, ctx.saved = _DecoderLayerFn.run(layer, tgt, memory, pos, query_pos, tgt_mask, mem_mask, params, layer._dropout_state(6), True)
        ctx.layer, ctx.has = layer, (pos is not None, query_pos is not None)
        return out

    @staticmethod
    def backward(ctx, g_out):
        kn, heads = ctx.layer.k, ctx.layer.nhead
        s_self, s_cross, s_ffn = ctx.saved
        has_pos, has_qpos = ctx.has
        g_x2, gf = _ffn_bwd(kn, _bl(g_out), s_ffn)
        g_x1, g_q2, (g_mem, g_memk), gc = _attention_bwd(kn, heads, g_x2, s_cross)
        g_tgt, g_qk, _, gs = _attention_bwd(kn, heads, g_x1, s_self)
        g_qpos = _lb(kn.add(g_qk, g_q2)) if has_qpos else None
        grads = gs[:4] + gc[:4] + gf[:4] + gs[4:] + gc[4:] + gf[4:]  # NAMES order: projections, then the norms
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
        _check_devices(src, pos, src_key_padding_mask)
        params = _EncoderLayerFn.PARAMS(self)
        mask = _mask_u8(src_key_padding_mask)
        if _records(src, *params):
            return _EncoderLayerFn.apply(self, src, pos, mask, *params)
        return _EncoderLayerFn.run(self, src, pos, mask, params, _NO_DROPOUT, False)[0]


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
        _check_devices(tgt, memory, pos, query_pos, tgt_key_padding_mask, memory_key_padding_mask)
        params = _DecoderLayerFn.PARAMS(self)
        masks = _mask_u8(tgt_key_padding_mask), _mask_u8(memory_key_padding_mask)
        if _records(tgt, memory, *params):
            return _DecoderLayerFn.apply(self, tgt, memory, pos, query_pos, *masks, *params)
        return _DecoderLayerFn.run(self, tgt, memory, pos, query_pos, *masks, params, _NO_DROPOUT, False)[0]


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
        if _records(x, self.weight):
            return _LayerNormFn.apply(self.k, x, self.weight, self.bias)
        return _lb(self.k.layernorm(_bl(x), self.weight, self.bias)[0])


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
            cpad = _pad16(w.shape[0])
            wf, wd = kn.pack2(w, cpad)
            bias = torch.zeros(cpad, device=x.device)
            bias[:w.shape[0]] = b.detach()
            h = kn.linear(h, wf, bias, relu=not last)
            wds.append(wd)
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
