"""Attention core and whole encoder layer at the DETR-R50 800x1333 bs=16 shape (BASELINE.json configs[3]): L = 1050 tokens, 8 heads x 32."""
import ctypes, json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from yolov7_d2_b200 import capi
from yolov7_d2_b200.detr import TransformerEncoderLayer, TransformerDecoderLayer

dev = torch.device("cuda:0")
L_ = capi.lib()
b, l, heads = 16, 1050, 8
e = heads * 32

def timeit(fn, iters=20):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters

res = {}
for name, lq in (("encoder self-attention", l), ("decoder cross-attention (100 queries)", 100), ("decoder cross-attention (300 queries)", 300)):
    qkv = torch.randn(b, 1, l, 3 * e, device=dev).to(torch.bfloat16)
    q = torch.randn(b, 1, lq, e, device=dev).to(torch.bfloat16)
    out = torch.empty(b, 1, lq, e, dtype=torch.bfloat16, device=dev)
    mask = torch.zeros(b, l, dtype=torch.uint8, device=dev)
    qa, ka, va, oa = capi.act(q), capi.act(qkv, e, e), capi.act(qkv, 2 * e, e), capi.act(out)
    ms = timeit(lambda: capi.check(L_.yb200_attention_fwd(ctypes.byref(qa), ctypes.byref(ka), ctypes.byref(va), capi.ptr(mask), ctypes.c_float(32 ** -0.5),
                                                          ctypes.byref(oa), None, capi.stream_ptr()), "att"))
    flops = 4.0 * b * heads * lq * l * 32
    exps = 1.0 * b * heads * ((lq + 127) // 128 * 128) * ((l + 127) // 128 * 128)
    res[name] = {"us": ms * 1e3, "tflops": flops / ms / 1e9, "gexp_per_s": exps / ms / 1e6}
    # backward of the same core: P recomputed from the saved log-sum-exp; 2.5x the forward FLOPs (S, dP, dV, dK, dQ) and 2x the exponentials
    lse = torch.empty(b, heads, lq, device=dev)
    capi.check(L_.yb200_attention_fwd(ctypes.byref(qa), ctypes.byref(ka), ctypes.byref(va), capi.ptr(mask), ctypes.c_float(32 ** -0.5), ctypes.byref(oa),
                                      capi.ptr(lse), capi.stream_ptr()), "att")
    dout = torch.randn(b, 1, lq, e, device=dev).to(torch.bfloat16)
    dq = torch.empty_like(q)
    dkv = torch.empty(b, 1, l, 2 * e, dtype=torch.bfloat16, device=dev)
    da, dqa, dka, dva = capi.act(dout), capi.act(dq), capi.act(dkv, 0, e), capi.act(dkv, e, e)
    ws = torch.empty(max(int(L_.yb200_attention_bwd_workspace(ctypes.byref(qa))), 16), dtype=torch.uint8, device=dev)
    msb = timeit(lambda: capi.check(L_.yb200_attention_bwd(ctypes.byref(qa), ctypes.byref(ka), ctypes.byref(va), ctypes.byref(oa), ctypes.byref(da), capi.ptr(mask),
                                                           ctypes.c_float(32 ** -0.5), capi.ptr(lse), ctypes.byref(dqa), ctypes.byref(dka), ctypes.byref(dva),
                                                           capi.ptr(ws), capi.stream_ptr()), "att bwd"))
    res[name + " backward"] = {"us": msb * 1e3, "tflops": 2.5 * flops / msb / 1e9, "gexp_per_s": 2 * exps / msb / 1e6}
enc = TransformerEncoderLayer(e, heads, dim_feedforward=2048).eval()
dec = TransformerDecoderLayer(e, heads, dim_feedforward=2048).eval()
src, pos = torch.randn(l, b, e, device=dev), torch.randn(l, b, e, device=dev)
tgt, qpos = torch.randn(100, b, e, device=dev), torch.randn(100, b, e, device=dev)
mask = torch.zeros(b, l, dtype=torch.bool, device=dev)
res["encoder layer forward (bs16, 1050 tokens, FFN 2048)"] = {"us": timeit(lambda: enc(src, src_key_padding_mask=mask, pos=pos), 10) * 1e3}
res["decoder layer forward (100 queries)"] = {"us": timeit(lambda: dec(tgt, src, memory_key_padding_mask=mask, pos=pos, query_pos=qpos), 10) * 1e3}
# inference: the same layers without autograd (no log-sum-exp or LayerNorm statistics kept)
with torch.no_grad():
    res["encoder layer forward, no grad"] = {"us": timeit(lambda: enc(src, src_key_padding_mask=mask, pos=pos), 10) * 1e3}
    res["decoder layer forward, no grad (100 queries)"] = {"us": timeit(lambda: dec(tgt, src, memory_key_padding_mask=mask, pos=pos, query_pos=qpos), 10) * 1e3}
# training: layer forward + backward through autograd (the kernels' own backward wiring, detr._EncoderLayerFn / _DecoderLayerFn), and the 6 + 6 stack
from yolov7_d2_b200.detr import Transformer
enc.train(); dec.train()
src_g, tgt_g = src.clone().requires_grad_(True), tgt.clone().requires_grad_(True)
def enc_step():
    enc(src_g, src_key_padding_mask=mask, pos=pos).sum().backward()
def dec_step():
    dec(tgt_g, src, memory_key_padding_mask=mask, pos=pos, query_pos=qpos).sum().backward()
res["encoder layer forward + backward (dropout 0.1)"] = {"us": timeit(enc_step, 10) * 1e3}
res["decoder layer forward + backward (100 queries, dropout 0.1)"] = {"us": timeit(dec_step, 10) * 1e3}
tr = Transformer(d_model=e, nhead=heads, num_encoder_layers=6, num_decoder_layers=6, dim_feedforward=2048, dropout=0.1, return_intermediate_dec=True).to(dev).train()
feat = torch.randn(b, e, 25, 42, device=dev, requires_grad=True)
pos_map = torch.randn(b, e, 25, 42, device=dev)
m2 = torch.zeros(b, 25, 42, dtype=torch.bool, device=dev)
query = torch.randn(100, e, device=dev)
def stack_step():
    hs, mem = tr(feat, m2, query, pos_map)
    (hs.sum() + mem.sum()).backward()
res["Transformer 6+6 (bs16, 25x42 memory, 100 queries, dropout 0.1) forward + backward"] = {"us": timeit(stack_step, 5) * 1e3}
print(json.dumps(res))
