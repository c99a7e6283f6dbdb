"""GPU: the SparseInst meta-architecture (yolov7_d2_b200/sparseinst_model.py) and its kernels (csrc/sparseinst_infer.cu).

A. yb200_normalize_pad is bit-identical to torch's `(image - mean) / std` and ImageList's zero padding, uint8 and fp32, mixed sizes; nothing
   outside the output is written.
B. yb200_sparseinst_infer_scores against the reference arithmetic in torch on the same GPU tensors and against fp64: labels exact, keep flags
   exact except where the fp64 score lies within 1e-6 of the threshold, scores and rescored scores within 1e-5 relative; the compact lists.
C. yb200_sparseinst_paste_masks at the shipped geometry (16 images x 100 queries, 160x216 -> 640x864 -> crop 640x853 -> 480x640) and on a
   mixed-size batch: the bool masks equal the reference's torch-CUDA chain except at pixels whose fp64 composite lies within 1e-6 of
   MASK_THRESHOLD (their count is reported); two calls give the same bits.
D. The whole model with a stand-in torch backbone (oracle/sparseinst_infer_oracle.StandInBackbone, registered as
   "build_sparseinst_standin_backbone"): its state_dict matches the reference's keys and shapes; eval Instances match the reference's
   `inference` in torch on the same decoder outputs; a training step's losses and every parameter's gradient, the backbone's included, against
   the fp64 composition of the oracles on the engine's match (<= 2.5 x the bf16-storage oracle's relative L2 error + 2 %); bit-reproducible
   steps; an image without instances trains; errors raise before any kernel runs."""
import ctypes
import os
import types

import numpy as np
import pytest
import torch

from test_sparseinst_bwd_gpu import _judge

pytestmark = pytest.mark.gpu

MEAN, STD = (123.675, 116.280, 103.530), (58.395, 57.120, 57.375)
MASK_THRESHOLD, CLS_THRESHOLD = 0.45, 0.005
NEAR = 1e-6
BACKBONE_NAME = "build_sparseinst_standin_backbone"


def _lib():
    from yolov7_d2_b200 import capi

    return capi.lib()


def _sp():
    from yolov7_d2_b200 import capi

    return capi.stream_ptr()


def _p(t, byte_off=0):
    return ctypes.c_void_p(t.data_ptr() + byte_off)


# ------------------------------------------------------------------------------------------------------------------------------------
# A. normalize_pad
# ------------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("f32", [False, True], ids=["uint8", "fp32"])
def test_normalize_pad_is_bit_identical(cuda, f32):
    from oracle import sparseinst_infer_oracle as sio

    g = torch.Generator().manual_seed(1 + f32)
    sizes = [(480, 640), (427, 640), (640, 501), (33, 17)]
    imgs = [torch.randint(0, 256, (3, h, w), generator=g, dtype=torch.uint8) for h, w in sizes]
    if f32:
        imgs = [(im.float() + torch.rand(im.shape, generator=g) - 0.5) for im in imgs]  # non-integer values too
    imgs = [im.cuda() for im in imgs]
    ref, _ = sio.preprocess(imgs, MEAN, STD)
    B, _, hp, wp = ref.shape
    assert (hp, wp) == (640, 640)
    staged = torch.cat([im.reshape(-1) for im in imgs])
    offs = np.concatenate([[0], np.cumsum([im.numel() for im in imgs])])
    table = torch.tensor([(int(o), h, w) for o, (h, w) in zip(offs, sizes)], dtype=torch.int64, device=cuda)
    mean, std = torch.tensor(MEAN, device=cuda), torch.tensor(STD, device=cuda)
    guard = 4096
    buf = torch.full((ref.numel() + 2 * guard,), float("nan"), device=cuda)
    rc = _lib().yb200_normalize_pad(_p(staged), int(f32), _p(table), B, _p(mean), _p(std), hp, wp, _p(buf, 4 * guard), _sp())
    assert rc == 0
    torch.cuda.synchronize()
    out = buf[guard:guard + ref.numel()].view(ref.shape)
    assert torch.equal(out, ref), f"{int((out != ref).sum())} values differ"
    assert buf[:guard].isnan().all() and buf[-guard:].isnan().all(), "written outside the output"


# ------------------------------------------------------------------------------------------------------------------------------------
# B. scores
# ------------------------------------------------------------------------------------------------------------------------------------
def _scores(logits, obj, masks, cls_thr=CLS_THRESHOLD, mask_thr=MASK_THRESHOLD):
    from yolov7_d2_b200 import capi

    B, N, K = logits.shape
    HW = masks.shape[-2] * masks.shape[-1]
    dev = logits.device
    o = dict(score=torch.empty(B, N, device=dev), label=torch.empty(B, N, dtype=torch.int32, device=dev),
             keep=torch.empty(B, N, dtype=torch.uint8, device=dev), rescored=torch.empty(B, N, device=dev),
             counts=torch.empty(B, dtype=torch.int32, device=dev), offsets=torch.empty(B + 1, dtype=torch.int32, device=dev),
             kept_query=torch.empty(B * N, dtype=torch.int32, device=dev), kept_score=torch.empty(B * N, device=dev),
             kept_label=torch.empty(B * N, dtype=torch.int64, device=dev))
    capi.check(_lib().yb200_sparseinst_infer_scores(_p(logits), _p(obj), _p(masks), B, N, K, HW, ctypes.c_float(cls_thr), ctypes.c_float(mask_thr),
                                                    _p(o["score"]), _p(o["label"]), _p(o["keep"]), _p(o["rescored"]), _p(o["counts"]),
                                                    _p(o["offsets"]), _p(o["kept_query"]), _p(o["kept_score"]), _p(o["kept_label"]), _sp()),
               "infer_scores")
    torch.cuda.synchronize()
    return o


def _shipped_outputs(B=16, N=100, K=80, hm=160, wm=216, seed=3):
    g = torch.Generator().manual_seed(seed)
    logits = torch.randn(B, N, K, generator=g) * 2 - 3
    logits[:, :7, 11] = logits[:, :7, 40] = 8.0  # exact ties: the lower class wins
    obj = torch.randn(B, N, 1, generator=g)
    masks = torch.randn(B, N, hm, wm, generator=g) * 2
    return logits.cuda(), obj.cuda(), masks.cuda()


def test_scores_against_torch_and_fp64(cuda):
    logits, obj, masks = _shipped_outputs()
    logits[3] -= 40  # an image without kept queries
    B, N, _ = logits.shape
    o = _scores(logits, obj, masks)
    # the reference's arithmetic in torch, fp32, same tensors (sparseinst.py:182-206)
    s32, l32 = torch.sqrt(logits.sigmoid() * obj.sigmoid()).max(dim=-1)
    s64, _ = torch.sqrt(logits.double().sigmoid() * obj.double().sigmoid()).max(dim=-1)
    assert torch.equal(o["label"].long(), l32), "labels differ from torch's max(dim)"
    assert (o["label"][:, :7] == 11).all()
    keep64 = s64 > CLS_THRESHOLD
    near = (s64 - CLS_THRESHOLD).abs() < NEAR
    assert torch.equal(o["keep"].bool()[~near], keep64[~near]) and torch.equal(o["keep"].bool(), s32 > CLS_THRESHOLD)
    assert not o["keep"][3].any() and o["keep"].sum() > B * N // 4
    torch.testing.assert_close(o["score"].double(), s64, rtol=1e-5, atol=0)
    keep = o["keep"].bool()
    m32 = masks.sigmoid()
    p = m32 > MASK_THRESHOLD  # the decisions both sides make in fp32
    m64 = masks.double().sigmoid()
    r64 = s64 * ((m64 * p).sum([2, 3]) / (p.sum([2, 3]).double() + 1e-6))
    r32 = s32 * ((m32 * p.float()).sum([2, 3]) / (p.float().sum([2, 3]) + 1e-6))
    torch.testing.assert_close(o["rescored"].double()[keep], r64[keep], rtol=1e-5, atol=0)
    torch.testing.assert_close(o["rescored"][keep], r32[keep], rtol=1e-5, atol=0)
    assert (o["rescored"][~keep] == 0).all()
    # compact lists: image-major, ascending queries
    counts = keep.sum(1)
    assert torch.equal(o["counts"].long(), counts) and torch.equal(o["offsets"].long(), torch.cat([counts.new_zeros(1), counts.cumsum(0)]))
    total = int(counts.sum())
    assert torch.equal(o["kept_query"][:total].long(), keep.nonzero()[:, 1])
    assert torch.equal(o["kept_score"][:total], o["rescored"][keep]) and torch.equal(o["kept_label"][:total], o["label"][keep].long())
    again = _scores(logits, obj, masks)
    assert all(torch.equal(again[k], o[k]) for k in ("score", "label", "keep", "rescored", "counts", "offsets"))


# ------------------------------------------------------------------------------------------------------------------------------------
# C. paste
# ------------------------------------------------------------------------------------------------------------------------------------
def _paste(masks, images, counts, ori, hp, wp, thr=MASK_THRESHOLD, kept=None):
    """images: per image (h, w); counts: kept masks per image (its first `count` queries unless `kept` gives the compact query list)"""
    from yolov7_d2_b200 import capi
    from yolov7_d2_b200.sparseinst_model import PasteImage

    B, N, hm, wm = masks.shape
    first = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    sizes = [c * h * w for c, (h, w) in zip(counts, ori)]
    off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    if kept is None:
        kept = torch.cat([torch.arange(c, dtype=torch.int32) for c in counts]).cuda()
    table = (PasteImage * B)(*[PasteImage(h, w, oh, ow, int(first[b]), c, int(off[b])) for b, ((h, w), (oh, ow), c) in enumerate(zip(images, ori, counts))])
    guard = 4096
    buf = torch.full((int(off[-1]) + 2 * guard,), 7, dtype=torch.uint8, device=masks.device)
    capi.check(_lib().yb200_sparseinst_paste_masks(_p(masks), N, hm, wm, _p(kept), table, B, hp, wp, ctypes.c_float(thr), _p(buf, guard), _sp()),
               "paste")
    torch.cuda.synchronize()
    assert (buf[:guard] == 7).all() and (buf[-guard:] == 7).all(), "written outside the output"
    out = buf[guard:guard + int(off[-1])]
    return [out[int(off[b]):int(off[b + 1])].view(c, *ori[b]) for b, c in enumerate(counts)]


def _taps(n_in, n_out, dev):
    """ATen's upsample_bilinear2d index arithmetic in fp32 (align_corners=False, size given): scale = (float)in / out, src = max(scale (dst + 0.5)
    - 0.5, 0) rounded once (the contracted multiply-add of the CUDA kernel), i1 = i0 + (i0 < in - 1), l1 = src - i0, l0 = 1 - l1"""
    scale = (torch.tensor(n_in, dtype=torch.float32) / n_out).double()
    s = (scale * (torch.arange(n_out, dtype=torch.float64) + 0.5) - 0.5).float().clamp_min(0)
    i0 = s.long()
    i1 = i0 + (i0 < n_in - 1).long()
    l1 = s - i0.float()
    return i0.to(dev), i1.to(dev), (1 - l1).double().to(dev), l1.double().to(dev)


def _resize64(x, out_h, out_w):
    """bilinear resize of fp64 planes [k, H, W] with the reference's fp32 taps and weights, the blend in fp64"""
    i0, i1, a0, a1 = _taps(x.shape[1], out_h, x.device)
    j0, j1, b0, b1 = _taps(x.shape[2], out_w, x.device)
    top, bot = x[:, i0], x[:, i1]
    top = top[:, :, j0] * b0 + top[:, :, j1] * b1
    bot = bot[:, :, j0] * b0 + bot[:, :, j1] * b1
    return top * a0[:, None] + bot * a1[:, None]


def _composite64(mlog, max_shape, img, ori):
    """the reference's chain (sigmoid, resize to the padded size, crop, resize to the original size) in fp64 on its fp32 sample positions: the
    value the fp32 chains approximate up to the rounding of their blends"""
    a = _resize64(mlog.double().sigmoid(), *max_shape)[:, :img[0], :img[1]]
    return _resize64(a, *ori)


def _check_masks(got, mlog, max_shape, img, ori, what):
    """equal to the torch-CUDA chain except where the fp64 composite lies within NEAR of the threshold; returns the count of such pixels"""
    from oracle import sparseinst_infer_oracle as sio

    ref = sio.composite(mlog, max_shape, img, ori) > MASK_THRESHOLD
    diff = got.bool() != ref
    n = int(diff.sum())
    if n:
        c64 = torch.cat([_composite64(mlog[i:i + 8], max_shape, img, ori) for i in range(0, mlog.shape[0], 8)])
        far = diff & ((c64 - MASK_THRESHOLD).abs() >= NEAR)
        assert not far.any(), f"{what}: {int(far.sum())} of {n} differing pixels are not within {NEAR} of the threshold"
    return n


def test_paste_at_the_shipped_geometry(cuda):
    _, _, masks = _shipped_outputs(seed=5)
    B, N = masks.shape[:2]
    img, ori, hp, wp = (640, 853), (480, 640), 640, 864
    outs = _paste(masks, [img] * B, [N] * B, [ori] * B, hp, wp)
    near = sum(_check_masks(outs[b], masks[b], (hp, wp), img, ori, f"image {b}") for b in range(B))
    print(f"\npaste 16 x 100 at 480x640: {near} pixels within {NEAR} of the threshold differ from the torch chain")
    again = _paste(masks, [img] * B, [N] * B, [ori] * B, hp, wp)
    assert all(torch.equal(a, b) for a, b in zip(outs, again)), "two calls differ"


def test_paste_mixed_batch(cuda):
    g = torch.Generator().manual_seed(6)
    images = [(480, 640), (427, 320), (200, 611), (640, 480)]
    ori = [(480, 640), (854, 640), (100, 305), (1000, 750)]  # same, larger, smaller, larger
    hp, wp = 640, 640
    N = 12
    masks = (torch.randn(len(images), N, hp // 4, wp // 4, generator=g) * 2).cuda()
    counts = [5, 0, 12, 3]
    kept = torch.cat([torch.tensor([0, 2, 3, 7, 11]), torch.arange(12), torch.tensor([1, 4, 9])]).to(torch.int32).cuda()
    outs = _paste(masks, images, counts, ori, hp, wp, kept=kept)
    qs = [[0, 2, 3, 7, 11], [], list(range(12)), [1, 4, 9]]
    for b, q in enumerate(qs):
        assert outs[b].shape == (len(q), *ori[b])
        if q:
            _check_masks(outs[b], masks[b][q], (hp, wp), images[b], ori[b], f"image {b}")


# ------------------------------------------------------------------------------------------------------------------------------------
# D. the model
# ------------------------------------------------------------------------------------------------------------------------------------
def _register_backbone():
    from yolov7_d2_b200 import modeling

    from oracle import sparseinst_infer_oracle as sio

    if BACKBONE_NAME not in modeling.BACKBONE_REGISTRY:
        def build_sparseinst_standin_backbone(cfg, input_shape=None):
            return sio.StandInBackbone()

        modeling.BACKBONE_REGISTRY.register(build_sparseinst_standin_backbone)


def _cfg(decoder="GroupIAMDecoder", device="cuda", mask_format="bitmask"):
    from oracle.gen_golden_sparseinst_infer import cfg_of

    cfg = cfg_of()
    cfg.MODEL.DEVICE, cfg.INPUT.MASK_FORMAT = device, mask_format
    cfg.MODEL.YOLO.CONF_THRESHOLD = CLS_THRESHOLD
    cfg.MODEL.SPARSE_INST.DECODER.NAME = decoder
    return cfg


def _model(seed=20):
    from yolov7_d2_b200.sparseinst_model import SparseInst

    from oracle import sparseinst_encoder_oracle as seo
    from oracle import sparseinst_infer_oracle as sio
    from oracle import sparseinst_oracle as so

    _register_backbone()
    model = SparseInst(_cfg())
    parts = {"backbone": sio.standin_state_dict(seed), "encoder": seo.encoder_state_dict(seed + 1, (64, 128, 256), 256),
             "decoder": so.decoder_state_dict(seed + 2, groups=4)}
    model.load_state_dict({f"{p}.{k}": v.cuda() for p, sd in parts.items() for k, v in sd.items()}, strict=True)
    return model, parts


def test_state_dict_matches_the_reference(cuda):
    from test_sparseinst_infer_oracle_golden import gold

    model, _ = _model()
    g = gold()
    sd = model.state_dict()
    assert list(sd) == list(g["state_dict/keys"])
    assert [",".join(str(d) for d in v.shape) for v in sd.values()] == list(g["state_dict/shapes"])
    assert isinstance(model.pixel_mean, torch.Tensor) and model.pixel_mean.shape == (3, 1, 1)


def _batch(g, sizes, ori, instances=None):
    out = []
    for b, ((h, w), (h0, w0)) in enumerate(zip(sizes, ori)):
        x = {"image": torch.randint(0, 256, (3, h, w), generator=g, dtype=torch.uint8), "height": h0, "width": w0}
        if instances is not None:
            x["instances"] = instances[b]
        out.append(x)
    return out


def test_eval_matches_the_reference_inference(cuda):
    from oracle import sparseinst_infer_oracle as sio

    model, _ = _model()
    model.eval()
    g = torch.Generator().manual_seed(21)
    sizes, ori = [(320, 427), (288, 320), (192, 250)], [(480, 640), (250, 278), (384, 500)]
    batched = _batch(g, sizes, ori)
    cap = {}
    hook = model.decoder.register_forward_hook(lambda m, i, o: cap.update(o))
    try:
        with torch.no_grad():
            res = model(batched)
    finally:
        hook.remove()
    torch.cuda.synchronize()
    ref = sio.inference(cap["pred_logits"], cap["pred_scores"], cap["pred_masks"], (320, 448), sizes, ori, CLS_THRESHOLD, MASK_THRESHOLD)
    kept = 0
    for b, (r, e) in enumerate(zip(res, ref)):
        inst = r["instances"]
        assert tuple(inst.image_size) == ori[b]
        assert torch.equal(inst.pred_classes, e["labels"]) and inst.pred_classes.dtype == torch.int64
        torch.testing.assert_close(inst.scores, e["scores"], rtol=1e-5, atol=0)
        if e["masks"] is None:
            assert not hasattr(inst, "pred_masks")
            continue
        kept += len(e["labels"])
        assert inst.pred_masks.dtype == torch.bool and inst.pred_masks.shape == (len(e["labels"]), *ori[b])
        _check_masks(inst.pred_masks, cap["pred_masks"][b][e["keep"]], (320, 448), sizes[b], ori[b], f"image {b}")
    assert kept > 0
    model.cls_threshold = 1.0  # nothing kept: empty scores / pred_classes and no pred_masks attribute
    with torch.no_grad():
        res = model(batched)
    for r in res:
        inst = r["instances"]
        assert inst.scores.numel() == 0 and inst.pred_classes.numel() == 0 and inst.pred_classes.dtype == torch.int64
        assert "pred_masks" not in vars(inst) and not hasattr(inst, "pred_masks")


def _train_inputs(g, counts):
    from yolov7_d2_b200 import modeling
    from yolov7_d2_b200.sparseinst_model import BitMasks

    from test_sparseinst_criterion_gpu import _ellipses

    sizes = [(128, 160), (96, 128), (120, 100)][:len(counts)]
    insts, mask_list, labels = [], [], []
    for (h, w), n in zip(sizes, counts):
        m = _ellipses(g, n, h, w) if n else torch.zeros(0, h, w, dtype=torch.bool)
        lab = torch.randint(0, 80, (n,), generator=g)
        kw = {"gt_classes": lab}
        if n:
            kw["gt_masks"] = BitMasks(m)
        insts.append(modeling.Instances((h, w), **kw))
        mask_list.append(m)
        labels.append(lab)
    return _batch(g, sizes, sizes, insts), mask_list, torch.cat(labels), sizes


COEF = {"loss_ce": 0.7, "loss_objectness": 1.3, "loss_dice": 0.4, "loss_mask": 1.9}


def _step(model, batched):
    cap = {}
    hook = model.decoder.register_forward_hook(lambda m, i, o: cap.update({k: v.detach() for k, v in o.items()}))
    try:
        model.zero_grad(set_to_none=True)
        losses = model(batched)
        sum(COEF[k] * v for k, v in losses.items()).backward()
    finally:
        hook.remove()
    torch.cuda.synchronize()
    return {k: v.detach().clone() for k, v in losses.items()}, {k: p.grad.clone() for k, p in model.named_parameters()}, cap


def test_training_step_against_fp64(cuda):
    """losses and every parameter's gradient, backbone included, against the fp64 composition backbone -> encoder -> GroupIAMDecoder ->
    criterion on the engine's match; an image without instances is part of the batch; two steps give the same bits"""
    from yolov7_d2_b200.sparseinst_criterion import _Targets

    from oracle import sparseinst_criterion_oracle as sco
    from oracle import sparseinst_encoder_oracle as seo
    from oracle import sparseinst_infer_oracle as sio
    from oracle import sparseinst_oracle as so
    from oracle import sparseinst_storage_oracle as sso

    model, parts = _model(30)
    model.train()
    g = torch.Generator().manual_seed(31)
    counts = [3, 0, 4]
    batched, mask_list, labels, sizes = _train_inputs(g, counts)
    losses, grads, cap = _step(model, batched)
    assert set(losses) == {"loss_ce", "loss_objectness", "loss_dice", "loss_mask"} and all(torch.isfinite(v) for v in losses.values())
    assert all(torch.isfinite(v).all() and v.abs().sum() > 0 for v in grads.values()), "a parameter got no gradient"
    losses2, grads2, _ = _step(model, batched)
    assert all(torch.equal(losses[k], losses2[k]) for k in losses) and all(torch.equal(grads[k], grads2[k]) for k in grads), "two steps differ"
    hp, wp = 128, 160
    targets = model.prepare_targets([x["instances"] for x in batched])
    tg = _Targets(targets, (hp, wp), cap["pred_masks"].shape, cuda, "test")
    indices, _ = model.criterion.matcher.match(cap["pred_logits"].float().contiguous(), cap["pred_masks"].float().contiguous(), tg)
    wd = model.criterion.weight_dict
    images64, _ = sio.preprocess([x["image"].cuda() for x in batched], MEAN, STD, dtype=torch.float64)

    def oracle(storage):
        sds = {p: {k: v.double().cuda().requires_grad_(True) for k, v in sd.items()} for p, sd in parts.items()}
        bb = sio.StandInBackbone().double().cuda()
        feats = torch.func.functional_call(bb, sds["backbone"], (images64,))
        x = (seo.encoder_forward_storage if storage else seo.encoder_forward)(feats, sds["encoder"])
        o = (sso if storage else so).decoder_forward(x, sds["decoder"], groups=4)
        tm = sco.target_masks([m.cuda() for m in mask_list], (hp, wp), o["pred_masks"].shape[-2:], torch.float64)
        ref = sco.losses(o["pred_logits"], o["pred_masks"], o["pred_scores"], tm, counts, labels.cuda(), indices, wd, float(sum(counts)))
        sum(COEF[k] * v for k, v in ref.items()).backward()
        r = {f"{p}.{k}": v.grad for p, sd in sds.items() for k, v in sd.items()}
        r.update({f"loss/{k}": v.detach().reshape(1) for k, v in ref.items()})
        return r

    got = dict(grads)
    got.update({f"loss/{k}": v.double().reshape(1) for k, v in losses.items()})
    ref, emu = oracle(False), oracle(True)
    assert sorted(got) == sorted(ref)
    _judge(got, ref, emu, "SparseInst training step")


def test_errors_raise_before_any_kernel(cuda):
    from yolov7_d2_b200 import capi, modeling
    from yolov7_d2_b200.sparseinst_model import SparseInst

    from test_sparseinst_kernels_gpu import _Recorder

    _register_backbone()
    with pytest.raises(capi.Yb200Error, match="no CPU path"):
        SparseInst(_cfg(device="cpu"))
    with pytest.raises(capi.Yb200Error, match="not built"):
        SparseInst(_cfg(decoder="IAMDecoderX"))
    if modeling.HAVE_D2:
        return
    model = SparseInst(_cfg(mask_format="polygon"))
    model.train()
    recs = [_Recorder(m.L) for m in (model, model.encoder, model.decoder)]
    model.L, model.encoder.L, model.decoder.L = recs
    g = torch.Generator().manual_seed(40)
    inst = modeling.Instances((64, 64), gt_classes=torch.zeros(1, dtype=torch.int64), gt_masks=types.SimpleNamespace(polygons=[[[0.0, 0, 9, 0, 9, 9]]]))
    with pytest.raises(capi.Yb200Error, match="polygon"):
        model(_batch(g, [(64, 64)], [(64, 64)], [inst]))
    assert not any(r.log for r in recs), "kernels ran before the error"
