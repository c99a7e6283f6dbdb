"""DETR transformer layers (yolov7_d2_b200.detr) against the outputs of the unmodified reference layers (tests/golden/detr.npz).
The CUDA path stores every intermediate in bf16 (the reference is fp32): tolerance 4e-2 of the output's max and correlation > 0.999
(LayerNorm outputs are O(1); each of the ~8 stored intermediates contributes rel 2^-8 rounding)."""
import os

import numpy as np
import pytest
import torch

from oracle import detr_oracle as dto

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "detr.npz")


def _check(got, ref, what):
    got, ref = got.float().cpu(), torch.as_tensor(np.asarray(ref)).float()
    assert torch.isfinite(got).all(), what
    err = (got - ref).abs().max().item()
    cos = torch.dot(got.flatten(), ref.flatten()) / (got.norm() * ref.norm())
    assert err <= 4e-2 * ref.abs().max().item() and cos > 0.999, f"{what}: max err {err:.4f} (max |ref| {ref.abs().max().item():.3f}), cos {cos:.5f}"


def test_encoder_layer_matches_reference(cuda):
    from yolov7_d2_b200.detr import TransformerEncoderLayer

    gold = np.load(GOLD, allow_pickle=False)
    d, nhead, ffn, b, L = (int(v) for v in gold["dims"])
    layer = TransformerEncoderLayer(d, nhead, dim_feedforward=ffn, dropout=0.0)
    layer.load_state_dict({k: v.to(cuda) for k, v in dto.layer_state_dict("encoder", d, ffn, seed=2).items()}, strict=True)
    layer.eval()
    args = torch.tensor(gold["enc_src"]).to(cuda), torch.tensor(gold["enc_mask"]).to(cuda), torch.tensor(gold["enc_pos"]).to(cuda)
    out = layer(args[0], src_key_padding_mask=args[1], pos=args[2])
    assert out.shape == (L, b, d) and out.dtype == torch.float32
    _check(out, gold["enc_out"], "encoder layer output")
    with torch.no_grad():
        _check(layer(args[0], src_key_padding_mask=args[1], pos=args[2]), gold["enc_out"], "encoder layer output (no grad)")
    # without mask / positional embedding: against the oracle (pinned to the reference by tests/test_detr_oracle_golden.py)
    sd = {"l." + k: v for k, v in dto.layer_state_dict("encoder", d, ffn, seed=2).items()}
    src = torch.tensor(gold["enc_src"])
    _check(layer(src.to(cuda)), dto.encoder_layer_post(src, sd, "l.", nhead), "encoder layer, no mask / pos")


def test_decoder_layer_matches_reference(cuda):
    from yolov7_d2_b200.detr import TransformerDecoderLayer

    gold = np.load(GOLD, allow_pickle=False)
    d, nhead, ffn, b, L = (int(v) for v in gold["dims"])
    layer = TransformerDecoderLayer(d, nhead, dim_feedforward=ffn, dropout=0.0)
    layer.load_state_dict({k: v.to(cuda) for k, v in dto.layer_state_dict("decoder", d, ffn, seed=3).items()}, strict=True)
    layer.eval()
    t = lambda k: torch.tensor(gold[k]).to(cuda)
    out = layer(t("dec_tgt"), t("dec_mem"), memory_key_padding_mask=t("enc_mask"), pos=t("enc_pos"), query_pos=t("dec_qpos"))
    _check(out, gold["dec_out"], "decoder layer output")
    with torch.no_grad():
        out = layer(t("dec_tgt"), t("dec_mem"), memory_key_padding_mask=t("enc_mask"), pos=t("enc_pos"), query_pos=t("dec_qpos"))
    _check(out, gold["dec_out"], "decoder layer output (no grad)")


def test_layers_refuse_what_is_not_built(cuda):
    from yolov7_d2_b200 import capi
    from yolov7_d2_b200.detr import TransformerDecoderLayer, TransformerEncoderLayer

    with pytest.raises(capi.Yb200Error):
        TransformerEncoderLayer(96, 2)  # head dimension 48
    layer = TransformerEncoderLayer(64, 2, dim_feedforward=128)
    with pytest.raises(capi.Yb200Error):
        layer(torch.randn(10, 1, 64))  # CPU tensor
    with pytest.raises(capi.Yb200Error):
        layer(torch.randn(10, 1, 64, device=cuda), src_mask=torch.zeros(10, 10, device=cuda))
    # every tensor argument is checked before any kernel sees its pointer, with and without autograd
    src = torch.randn(10, 1, 64, device=cuda)
    with pytest.raises(capi.Yb200Error, match="CUDA tensors"):
        layer(src, pos=torch.randn(10, 1, 64))
    with pytest.raises(capi.Yb200Error, match="CUDA tensors"):
        layer(src, src_key_padding_mask=torch.zeros(1, 10, dtype=torch.bool))
    dec = TransformerDecoderLayer(64, 2, dim_feedforward=128)
    tgt, mem = torch.randn(6, 1, 64, device=cuda), torch.randn(10, 1, 64, device=cuda)
    with pytest.raises(capi.Yb200Error, match="CUDA tensors"):
        dec(tgt, torch.randn(10, 1, 64))
    with pytest.raises(capi.Yb200Error, match="CUDA tensors"):
        dec(tgt, mem, query_pos=torch.randn(6, 1, 64))
    with torch.no_grad(), pytest.raises(capi.Yb200Error, match="CUDA tensors"):
        dec(tgt, mem, memory_key_padding_mask=torch.zeros(1, 10, dtype=torch.bool))


def test_relu_epilogues(cuda):
    """Linear + ReLU forward and the ReLU-masked data gradient with bias-gradient sums (FFN of detr_backbone.py:167)"""
    import ctypes
    import torch.nn.functional as F
    from yolov7_d2_b200 import capi

    L_ = capi.lib()
    b, l, e, ff = 2, 150, 64, 256
    g = torch.Generator().manual_seed(3)
    x = torch.randn(b, 1, l, e, generator=g).to(cuda).to(torch.bfloat16)
    w1 = (torch.randn(ff, e, generator=g) / e ** 0.5).to(cuda).to(torch.bfloat16).float()
    b1 = (torch.randn(ff, generator=g) * 0.3).to(cuda)
    wf = torch.empty(ff, 1, e, dtype=torch.bfloat16, device=cuda)
    capi.check(L_.yb200_pack_conv_weight(capi.ptr(w1), ff, e, 1, ff, e, capi.ptr(wf), None, capi.stream_ptr()), "pack")
    h = torch.full((b, 1, l, ff), float("nan"), dtype=torch.bfloat16, device=cuda)
    xa, ha = capi.act(x), capi.act(h)
    capi.check(L_.yb200_linear_relu_fwd(ctypes.byref(xa), capi.ptr(wf), capi.ptr(b1), ctypes.byref(ha), capi.stream_ptr()), "linear_relu")
    ref = F.relu(F.linear(x.float(), w1, b1))
    assert (h.float() - ref).abs().max() <= 2.0 ** -7 * ref.abs().max()
    dz = torch.randn(b, 1, l, e, generator=g).to(cuda).to(torch.bfloat16)
    w2 = (torch.randn(e, ff, generator=g) / ff ** 0.5).to(cuda).to(torch.bfloat16).float()
    wd = torch.empty(ff, 1, e, dtype=torch.bfloat16, device=cuda)
    capi.check(L_.yb200_pack_conv_weight(capi.ptr(w2), e, ff, 1, e, ff, None, capi.ptr(wd), capi.stream_ptr()), "pack")
    du = torch.full_like(h, float("nan"))
    acc = torch.zeros(ff, dtype=torch.float64, device=cuda)
    dza, dua = capi.act(dz), capi.act(du)
    capi.check(L_.yb200_linear_dgrad_relu(ctypes.byref(dza), capi.ptr(wd), ctypes.byref(ha), ctypes.byref(dua), capi.ptr(acc), capi.stream_ptr()), "dgrad_relu")
    refd = F.linear(dz.float(), w2.t()) * (h.float() > 0)
    assert (du.float() - refd).abs().max() <= 2.0 ** -7 * refd.abs().max()
    assert (acc.float() - du.float().sum((0, 1, 2))).abs().max() <= 1e-4 * du.float().sum((0, 1, 2)).abs().max() + 1e-4


def test_encoder_layer_backward_matches_reference(cuda):
    """training path: gradients w.r.t. the input and every parameter of the encoder layer against the reference layer's autograd
    (tests/golden/detr.npz).  bf16 storage of every saved tensor: cosine > 0.995 and at most 2.5x the error of the oracle's own
    bf16-storage emulation (+2 % of the gradient's max)."""
    from yolov7_d2_b200.detr import TransformerEncoderLayer

    gold = np.load(GOLD, allow_pickle=False)
    d, nhead, ffn, b, L = (int(v) for v in gold["dims"])
    layer = TransformerEncoderLayer(d, nhead, dim_feedforward=ffn, dropout=0.0)
    layer.load_state_dict({k: v.to(cuda) for k, v in dto.layer_state_dict("encoder", d, ffn, seed=2).items()}, strict=True)
    src = torch.tensor(gold["enc_src"]).to(cuda).requires_grad_(True)
    out = layer(src, src_key_padding_mask=torch.tensor(gold["enc_mask"]).to(cuda), pos=torch.tensor(gold["enc_pos"]).to(cuda))
    _check(out.detach(), gold["enc_out"], "encoder layer output (training path)")
    out.backward(torch.tensor(gold["enc_gout"]).to(cuda))

    # yardstick: the oracle with every stored tensor rounded to bf16.  Rounding the FFN hidden activations flips ReLU masks near zero,
    # which alone moves linear1's gradients by ~10 % of their max on this layer (fp32 vs bf16 storage, both on the CPU).
    dto.EMULATE_STORAGE = True
    try:
        sde = {"l." + k: v.clone().requires_grad_(True) for k, v in dto.layer_state_dict("encoder", d, ffn, seed=2).items()}
        se = torch.tensor(gold["enc_src"]).requires_grad_(True)
        dto.encoder_layer_post(se, sde, "l.", nhead, torch.tensor(gold["enc_mask"]), torch.tensor(gold["enc_pos"])).backward(torch.tensor(gold["enc_gout"]))
    finally:
        dto.EMULATE_STORAGE = False

    def chk(got, ref, emu, what):
        got, ref, emu = got.float().cpu(), torch.as_tensor(np.asarray(ref)).float(), emu.float()
        assert torch.isfinite(got).all(), what
        scale = ref.abs().max().item()
        err, yard = (got - ref).abs().max().item() / scale, (emu - ref).abs().max().item() / scale
        cos = torch.dot(got.flatten(), ref.flatten()) / (got.norm() * ref.norm())
        assert cos > 0.995 and err <= 2.5 * yard + 2e-2, f"{what}: cos {cos:.4f}, rel err {err:.4f} vs emulated-storage yardstick {yard:.4f}"

    chk(src.grad, gold["enc_gsrc"], se.grad, "src gradient")
    for name, p in layer.named_parameters():
        chk(p.grad, gold["enc_grad/" + name], sde["l." + name].grad, name)


def test_decoder_layer_backward_matches_oracle(cuda):
    """training path of the decoder layer against the autograd of the oracle (forward pinned to the reference layer), judged with the oracle's
    bf16-storage emulation as yardstick (see the encoder test)"""
    import torch.nn.functional as F
    from yolov7_d2_b200.detr import TransformerDecoderLayer

    gold = np.load(GOLD, allow_pickle=False)
    d, nhead, ffn, b, L = (int(v) for v in gold["dims"])
    sd = dto.layer_state_dict("decoder", d, ffn, seed=3)
    layer = TransformerDecoderLayer(d, nhead, dim_feedforward=ffn, dropout=0.0)
    layer.load_state_dict({k: v.to(cuda) for k, v in sd.items()}, strict=True)
    names = ("dec_tgt", "dec_mem", "enc_pos", "dec_qpos")
    mask = torch.tensor(gold["enc_mask"])
    gout = torch.randn(gold["dec_out"].shape, generator=torch.Generator().manual_seed(4))

    def oracle_run(emulate):
        dto.EMULATE_STORAGE = emulate
        try:
            ins = [torch.tensor(gold[k]).requires_grad_(True) for k in names]
            sdr = {"l." + k: v.clone().requires_grad_(True) for k, v in sd.items()}
            dto.decoder_layer_post(ins[0], ins[1], sdr, "l.", nhead, mask, ins[2], ins[3]).backward(gout)
        finally:
            dto.EMULATE_STORAGE = False
        return ins, sdr

    ref_in, ref_sd = oracle_run(False)
    emu_in, emu_sd = oracle_run(True)
    ours = [torch.tensor(gold[k]).to(cuda).requires_grad_(True) for k in names]
    out = layer(ours[0], ours[1], memory_key_padding_mask=mask.to(cuda), pos=ours[2], query_pos=ours[3])
    _check(out.detach(), gold["dec_out"], "decoder layer output (training path)")
    out.backward(gout.to(cuda))

    def chk(got, ref, emu, what):
        got, ref, emu = got.float().cpu(), ref.float(), emu.float()
        scale = ref.abs().max().item()
        err, yard = (got - ref).abs().max().item() / scale, (emu - ref).abs().max().item() / scale
        cos = torch.dot(got.flatten(), ref.flatten()) / (got.norm() * ref.norm())
        assert torch.isfinite(got).all() and cos > 0.995 and err <= 2.5 * yard + 2e-2, f"{what}: cos {cos:.4f}, rel err {err:.4f} vs yardstick {yard:.4f}"

    for k, a, r, m in zip(names, ours, ref_in, emu_in):
        chk(a.grad, r.grad, m.grad, k + " gradient")
    for name, p in layer.named_parameters():
        chk(p.grad, ref_sd["l." + name].grad, emu_sd["l." + name].grad, name)


def test_transformer_stack_forward_and_backward(cuda):
    """`Transformer` (detr_backbone.py:25-126): encoder stack -> decoder stack with the final LayerNorm and return_intermediate, against
    the composed oracle layers (oracle/detr_oracle.py, pinned to the reference layers by tests/golden/detr.npz); gradients flow to every
    parameter and to the inputs."""
    from yolov7_d2_b200.detr import Transformer

    d, nhead, ffn, bs, h, w, nq = 256, 8, 512, 2, 6, 9, 20
    torch.manual_seed(0)
    model = Transformer(d, nhead, num_encoder_layers=2, num_decoder_layers=2, dim_feedforward=ffn, dropout=0.0, return_intermediate_dec=True)
    g = torch.Generator().manual_seed(3)
    src = torch.randn(bs, d, h, w, generator=g).to(cuda).requires_grad_(True)
    pos = torch.randn(bs, d, h, w, generator=g).to(cuda)
    mask = torch.zeros(bs, h, w, dtype=torch.bool)
    mask[1, :, 6:] = True
    query = torch.randn(nq, d, generator=g).to(cuda)
    hs, memory = model(src, mask.to(cuda), query, pos)
    assert tuple(hs.shape) == (2, bs, nq, d) and tuple(memory.shape) == (bs, d, h, w)
    # oracle composition with the same parameters
    sd = {k: v.detach().cpu().float() for k, v in model.state_dict().items()}
    s = src.detach().cpu().flatten(2).permute(2, 0, 1)
    p = pos.cpu().flatten(2).permute(2, 0, 1)
    q = query.cpu().unsqueeze(1).repeat(1, bs, 1)
    m = mask.flatten(1)
    mem = s
    for i in range(2):
        mem = dto.encoder_layer_post(mem, sd, f"encoder.layers.{i}.", nhead, m, p)
    out, inter = torch.zeros_like(q), []
    for i in range(2):
        out = dto.decoder_layer_post(out, mem, sd, f"decoder.layers.{i}.", nhead, m, p, q)
        inter.append(torch.nn.functional.layer_norm(out, (d,), sd["decoder.norm.weight"], sd["decoder.norm.bias"]))
    ref_hs = torch.stack(inter).transpose(1, 2)
    err = (hs.detach().cpu() - ref_hs).abs().max().item() / ref_hs.abs().max().item()
    assert err <= 0.05, err  # bf16 storage through 4 layers
    merr = (memory.detach().cpu() - mem.permute(1, 2, 0).view(bs, d, h, w)).abs().max().item() / mem.abs().max().item()
    assert merr <= 0.05, merr
    (hs.float().square().mean() + memory.float().mean()).backward()
    assert src.grad is not None and torch.isfinite(src.grad).all() and float(src.grad.abs().sum()) > 0
    missing = [n for n, prm in model.named_parameters() if prm.grad is None or not torch.isfinite(prm.grad).all()]
    assert not missing, missing[:5]
