"""TEST INFRASTRUCTURE -- CPU restatement (plain torch fp32) of the reference's DETR transformer layers (SURVEY.md par.8a row T1).

Pinned by tests/golden/detr.npz, produced by oracle/gen_golden_detr.py from the UNMODIFIED reference classes
(yolov7/modeling/backbone/detr_backbone.py:140-242, which wrap torch's nn.MultiheadAttention); tests/test_detr_oracle_golden.py
re-checks this file against those vectors on every CPU run.  Only tests/, __graft_entry__.smoke() and bench.py's CPU legs may import it.
Dropout (0.1 in the reference, active in training) is an RNG-driven regulariser: parity runs use eval mode / p = 0 (SURVEY.md par.8a T1).
"""
import math

import torch
import torch.nn.functional as F

LN_EPS = 1e-5  # nn.LayerNorm default (detr_backbone.py:146-147)
# True: round every tensor the CUDA path stores in bf16 (activations and the packed weights) -- the yardstick for judging the 16-bit path
# against this fp32 restatement (same idea as oracle/yolox_oracle.py).  Rounding has an identity gradient, so autograd still works.
EMULATE_STORAGE = False


def _q(t):
    return t.to(torch.bfloat16).to(torch.float32) if EMULATE_STORAGE else t


# ---- the kernels' dropout masks, restated: a counter-based hash of (seed, element index) (csrc/attention.cu: mix32 / drop_row_key / drop_factor and
# dropout_bf16_kernel).  NOT torch's Philox stream (nn.Dropout / nn.MultiheadAttention(dropout=p), detr_backbone.py:140-152): the reference's masks
# are random, so parity is "same computation given the same mask" + the keep probability; these functions give the tests the kernels' mask.
_M = 0xFFFFFFFF


def _mix32(h):
    h = h ^ (h >> 16)
    h = (h * 0x85EBCA6B) & _M
    h = h ^ (h >> 13)
    h = (h * 0xC2B2AE35) & _M
    return h ^ (h >> 16)


def _thr24(p):
    return int(float(torch.tensor(p, dtype=torch.float32)) * 16777216.0)


def dropout_multiplier(seed, shape_blc, p, device=None):
    """[B, L, C] multiplier (0 or 1/(1-p)) of yb200_dropout for a [B][1][L][C] activation: element index ((b*L + l)*C + c).  device: where
    to evaluate the hash (default: the CPU)"""
    n = 1
    for d in shape_blc:
        n *= d
    e = torch.arange(n, dtype=torch.int64, device=device)
    keep = (_mix32(seed ^ ((e * 0x9E3779B1) & _M)) >> 8) >= _thr24(p)
    inv = float(torch.tensor(1.0, dtype=torch.float32) / (torch.tensor(1.0, dtype=torch.float32) - torch.tensor(p, dtype=torch.float32)))
    return (keep.to(torch.float32) * inv).view(*shape_blc)


def attention_dropout_multiplier(seed, b, heads, lq, lk, p, device=None):
    """[B, H, Lq, Lk] multiplier of yb200_attention_fwd_dropout: row key from (seed, b*H + h, q), element from the key index.  device: where
    to evaluate the hash (default: the CPU; B = 16 at 1050 x 1050 tokens is 141 M elements)"""
    bh = torch.arange(b * heads, dtype=torch.int64, device=device)[:, None]
    q = torch.arange(lq, dtype=torch.int64, device=device)[None, :]
    row = _mix32(seed ^ _mix32((bh * 0x9E3779B1 + q + 0x7F4A7C15) & _M))
    col = (torch.arange(lk, dtype=torch.int64, device=device) * 0x9E3779B1) & _M
    keep = (_mix32(row[..., None] ^ col) >> 8) >= _thr24(p)
    inv = float(torch.tensor(1.0, dtype=torch.float32) / (torch.tensor(1.0, dtype=torch.float32) - torch.tensor(p, dtype=torch.float32)))
    return (keep.to(torch.float32) * inv).view(b, heads, lq, lk)


def _drop_seq(x_lbe, mult_blc):
    """apply a [B, L, C] multiplier to a seq-first [L, B, C] tensor (None = identity)"""
    return x_lbe if mult_blc is None else x_lbe * mult_blc.permute(1, 0, 2)


def mha(query, key, value, sd, prefix, nhead, key_padding_mask=None, need_probs=False, attn_drop=None):
    """nn.MultiheadAttention.forward (detr_backbone.py:140,160-161,200-202) for seq-first inputs [L, B, E]:
    packed in_proj (q | k | v rows of in_proj_weight), q scaled by head_dim^-0.5, softmax over keys with key_padding_mask (True = ignore)
    as -inf, out_proj.  Returns [Lq, B, E]."""
    lq, b, e = query.shape
    lk = key.shape[0]
    dh = e // nhead
    w, bias = sd[prefix + "in_proj_weight"], sd[prefix + "in_proj_bias"]
    q = _q(F.linear(query, _q(w[:e]), bias[:e])) * (dh ** -0.5)
    k = _q(F.linear(key, _q(w[e:2 * e]), bias[e:2 * e]))
    v = _q(F.linear(value, _q(w[2 * e:]), bias[2 * e:]))
    q = q.reshape(lq, b * nhead, dh).transpose(0, 1)          # [B*H, Lq, dh]
    k = k.reshape(lk, b * nhead, dh).transpose(0, 1)
    v = v.reshape(lk, b * nhead, dh).transpose(0, 1)
    s = torch.bmm(q, k.transpose(1, 2))                        # [B*H, Lq, Lk]
    if key_padding_mask is not None:
        s = s.view(b, nhead, lq, lk).masked_fill(key_padding_mask[:, None, None, :], float("-inf")).view(b * nhead, lq, lk)
    p = torch.softmax(s, dim=-1)
    if attn_drop is not None:  # dropout on the attention probabilities: [B, H, Lq, Lk] multiplier
        p = p * attn_drop.reshape(b * nhead, lq, lk)
    o = _q(torch.bmm(_q(p), v)).transpose(0, 1).reshape(lq, b, e)
    out = F.linear(o, _q(sd[prefix + "out_proj.weight"]), sd[prefix + "out_proj.bias"])
    return (out, p) if need_probs else out


def _ln(x, sd, name):
    return F.layer_norm(x, (x.shape[-1],), sd[name + ".weight"], sd[name + ".bias"], LN_EPS)


def _pos(t, pos):
    return t if pos is None else t + pos


def encoder_layer_post(src, sd, prefix, nhead, key_padding_mask=None, pos=None, drop=None):
    """TransformerEncoderLayer.forward_post, detr_backbone.py:157-170.  drop = None: dropout is the identity (eval / p = 0); else
    (attention-probability multiplier [B,H,L,L], dropout1 [B,L,E], FFN dropout [B,L,F], dropout2 [B,L,E]) -- the explicit masks of one training step"""
    da, d1, df, d2 = drop if drop is not None else (None, None, None, None)
    src = _q(src)
    qk = _q(_pos(src, pos))
    src = _q(_ln(_q(src + _drop_seq(mha(qk, qk, src, sd, prefix + "self_attn.", nhead, key_padding_mask, attn_drop=da), d1)), sd, prefix + "norm1"))
    h = _q(_drop_seq(F.relu(F.linear(src, _q(sd[prefix + "linear1.weight"]), sd[prefix + "linear1.bias"])), df))
    ff = _drop_seq(F.linear(h, _q(sd[prefix + "linear2.weight"]), sd[prefix + "linear2.bias"]), d2)
    return _q(_ln(_q(src + ff), sd, prefix + "norm2"))


def decoder_layer_post(tgt, memory, sd, prefix, nhead, memory_key_padding_mask=None, pos=None, query_pos=None, drop=None):
    """TransformerDecoderLayer.forward_post, detr_backbone.py:221-242.  drop = None: dropout = identity; else the explicit multipliers
    (self-attention probabilities, dropout1, cross-attention probabilities, dropout2, FFN dropout, dropout3)"""
    a1, d1, a2, d2, df, d3 = drop if drop is not None else (None,) * 6
    tgt, memory = _q(tgt), _q(memory)
    qk = _q(_pos(tgt, query_pos))
    tgt = _q(_ln(_q(tgt + _drop_seq(mha(qk, qk, tgt, sd, prefix + "self_attn.", nhead, attn_drop=a1), d1)), sd, prefix + "norm1"))
    cross = mha(_q(_pos(tgt, query_pos)), _q(_pos(memory, pos)), memory, sd, prefix + "multihead_attn.", nhead, memory_key_padding_mask, attn_drop=a2)
    tgt = _q(_ln(_q(tgt + _drop_seq(cross, d2)), sd, prefix + "norm2"))
    h = _q(_drop_seq(F.relu(F.linear(tgt, _q(sd[prefix + "linear1.weight"]), sd[prefix + "linear1.bias"])), df))
    ff = _drop_seq(F.linear(h, _q(sd[prefix + "linear2.weight"]), sd[prefix + "linear2.bias"]), d3)
    return _q(_ln(_q(tgt + ff), sd, prefix + "norm3"))


def attention_core(q, k, v, key_padding_mask=None, scale=None, attn_drop=None):
    """softmax(q k^T * scale + mask) v for [B, H, L, dh] tensors: the part of nn.MultiheadAttention between in_proj and out_proj; attn_drop = the
    [B, H, Lq, Lk] dropout multiplier on the probabilities (None = no dropout)"""
    scale = q.shape[-1] ** -0.5 if scale is None else scale
    s = torch.matmul(q, k.transpose(-1, -2)) * scale
    if key_padding_mask is not None:
        s = s.masked_fill(key_padding_mask[:, None, None, :], float("-inf"))
    p = torch.softmax(s, -1)
    if attn_drop is not None:
        p = p * attn_drop
    return torch.matmul(p, v)


def layer_state_dict(kind, d_model, ffn, seed=0):
    """parameters of one layer under the reference's names (nn.MultiheadAttention: in_proj_weight [3E,E], in_proj_bias, out_proj.*)"""
    g = torch.Generator().manual_seed(seed)

    def rn(*s, std):
        return torch.randn(*s, generator=g) * std

    sd = {}
    for att in (["self_attn"] if kind == "encoder" else ["self_attn", "multihead_attn"]):
        sd[att + ".in_proj_weight"] = rn(3 * d_model, d_model, std=d_model ** -0.5)
        sd[att + ".in_proj_bias"] = rn(3 * d_model, std=0.1)
        sd[att + ".out_proj.weight"] = rn(d_model, d_model, std=d_model ** -0.5)
        sd[att + ".out_proj.bias"] = rn(d_model, std=0.1)
    sd["linear1.weight"], sd["linear1.bias"] = rn(ffn, d_model, std=d_model ** -0.5), rn(ffn, std=0.1)
    sd["linear2.weight"], sd["linear2.bias"] = rn(d_model, ffn, std=ffn ** -0.5), rn(d_model, std=0.1)
    for n in (["norm1", "norm2"] if kind == "encoder" else ["norm1", "norm2", "norm3"]):
        sd[n + ".weight"] = torch.rand(d_model, generator=g) + 0.5
        sd[n + ".bias"] = rn(d_model, std=0.1)
    return sd
