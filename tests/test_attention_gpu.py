"""GPU parity of the wgmma attention core (yb200_attention_fwd) against the oracle's attention_core (= the arithmetic inside
torch's nn.MultiheadAttention that detr_backbone.py:140,200-202 instantiates) on the same bf16-rounded q, k, v.
Tolerance: probabilities and the output are rounded to bf16 (rel 2^-8 each) => 2^-6 of the output's max; the log-sum-exp is fp32 => 2e-3 abs."""
import ctypes

import pytest
import torch

from oracle import detr_oracle as dto

pytestmark = pytest.mark.gpu


def _run(capi, q, k, v, mask, scale, out, lse):
    qa, ka, va, oa = (capi.act(*t) if isinstance(t, tuple) else capi.act(t) for t in (q, k, v, out))
    capi.check(capi.lib().yb200_attention_fwd(ctypes.byref(qa), ctypes.byref(ka), ctypes.byref(va), capi.ptr(mask), ctypes.c_float(scale), ctypes.byref(oa),
                                              capi.ptr(lse), capi.stream_ptr()), "attention_fwd")


CASES = [  # (B, heads, Lq, Lk, masked)
    (2, 2, 150, 150, True),     # one full + one partial tile, ragged padding (the golden layer's shape)
    (1, 1, 128, 128, False),    # exactly one tile
    (3, 8, 100, 1050, True),    # decoder cross-attention at 800x1333
    (2, 8, 1050, 1050, True),   # encoder self-attention at 800x1333
    (2, 4, 17, 5, False),       # tiny
    (1, 8, 300, 300, False),    # DetrD2go query count
]


@pytest.mark.parametrize("case", CASES, ids=lambda c: "B%d_H%d_q%d_k%d_%s" % (c[0], c[1], c[2], c[3], "mask" if c[4] else "nomask"))
def test_attention_core(cuda, case):
    from yolov7_d2_b200 import capi

    b, heads, lq, lk, masked = case
    e = heads * 32
    g = torch.Generator().manual_seed(lq * 7 + lk)
    q = (torch.randn(b, 1, lq, e, generator=g) * 1.5).to(cuda).to(torch.bfloat16)
    k = (torch.randn(b, 1, lk, e, generator=g) * 1.5).to(cuda).to(torch.bfloat16)
    v = torch.randn(b, 1, lk, e, generator=g).to(cuda).to(torch.bfloat16)
    mask = None
    if masked:
        mask = torch.zeros(b, lk, dtype=torch.uint8)
        mask[0, lk - lk // 3:] = 1
        if b > 1:
            mask[1, 1:max(2, lk // 5)] = 1
        mask = mask.to(cuda)
    out = torch.full((b, 1, lq, e), float("nan"), dtype=torch.bfloat16, device=cuda)
    lse = torch.full((b, heads, lq), float("nan"), device=cuda)
    scale = 32 ** -0.5
    _run(capi, q, k, v, mask, scale, out, lse)

    def heads_first(t, l):
        return t.float().view(b, l, heads, 32).permute(0, 2, 1, 3)

    qh, kh, vh = heads_first(q, lq), heads_first(k, lk), heads_first(v, lk)
    ref = dto.attention_core(qh, kh, vh, mask.bool() if masked else None, scale)          # [B,H,Lq,32]
    got = out.float().view(b, lq, heads, 32).permute(0, 2, 1, 3)
    assert torch.isfinite(got).all()
    err = (got - ref).abs().max().item()
    assert err <= 2.0 ** -6 * ref.abs().max().item(), f"attention output: max err {err:.4e} (max |ref| {ref.abs().max().item():.3f})"
    s = torch.matmul(qh, kh.transpose(-1, -2)) * scale
    if masked:
        s = s.masked_fill(mask.bool()[:, None, None, :], float("-inf"))
    assert (lse - torch.logsumexp(s, -1)).abs().max().item() <= 2e-3


def test_attention_on_packed_qkv_slices(cuda):
    """q, k, v as channel slices of one [B, L, 3E] buffer (the packed in_proj output) and the output into a slice of a wider buffer"""
    from yolov7_d2_b200 import capi

    b, heads, l = 2, 8, 200
    e = heads * 32
    g = torch.Generator().manual_seed(5)
    qkv = torch.randn(b, 1, l, 3 * e, generator=g).to(cuda).to(torch.bfloat16)
    out = torch.zeros(b, 1, l, e + 64, dtype=torch.bfloat16, device=cuda)
    _run(capi, (qkv, 0, e), (qkv, e, e), (qkv, 2 * e, e), None, 32 ** -0.5, (out, 64, e), None)
    hf = lambda t: t.float().view(b, l, heads, 32).permute(0, 2, 1, 3)
    ref = dto.attention_core(hf(qkv[..., :e]), hf(qkv[..., e:2 * e]), hf(qkv[..., 2 * e:]))
    got = out[..., 64:].float().view(b, l, heads, 32).permute(0, 2, 1, 3)
    assert (got - ref).abs().max().item() <= 2.0 ** -6 * ref.abs().max().item()
    assert not out[..., :64].any()


def test_fully_masked_rows_give_zeros(cuda):
    from yolov7_d2_b200 import capi

    q = torch.randn(1, 1, 40, 64, device=cuda).to(torch.bfloat16)
    k = torch.randn(1, 1, 30, 64, device=cuda).to(torch.bfloat16)
    v = torch.randn(1, 1, 30, 64, device=cuda).to(torch.bfloat16)
    mask = torch.ones(1, 30, dtype=torch.uint8, device=cuda)
    out = torch.full((1, 1, 40, 64), float("nan"), dtype=torch.bfloat16, device=cuda)
    _run(capi, q, k, v, mask, 32 ** -0.5, out, None)
    assert not out.any()
