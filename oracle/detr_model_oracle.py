"""TEST INFRASTRUCTURE -- plain-torch restatement of the DETR meta-architecture's own arithmetic (yolov7/modeling/meta_arch/detr.py,
yolov7/modeling/backbone/detr_backbone.py): `preprocess_image` (:273-279), `MaskedBackboneTraceFriendly.mask_out_padding` (:389-403),
`PositionEmbeddingSine(normalize=True)` (:334-375), `prepare_targets` (:204-217), and `inference` (:219-265) followed by detectron2's
`detector_postprocess`; plus a small stand-in backbone for the meta-architecture's tests.

Device-agnostic and dtype-following: in fp32 the operations run in torch's order (the reference's arithmetic, bit for bit on the same device),
in fp64 they are the exact yardstick.  Pinned by tests/golden/detr_model.npz, produced by oracle/gen_golden_detr_model.py from the unmodified
reference; tests/test_detr_model_oracle_golden.py re-checks this file against it on every CPU run.  Only tests/ and tools/ may import it.
"""
import math
import types

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import sparseinst_infer_oracle as sio


def preprocess(images, mean, std, dtype=torch.float32):
    """(image - mean) / std per image, zero-padded to the batch maximum (ImageList.from_tensors, size_divisibility 0)"""
    return sio.preprocess(images, mean, std, dtype, divisibility=1)


def mask_out_padding(feature_shapes, strides, image_sizes, device=None):
    """per level bool [B, H, W]: False on the ceil(h / stride) x ceil(w / stride) top-left rectangle (float64 ceil), True elsewhere"""
    masks = []
    for shape, s in zip(feature_shapes, strides):
        n, _, h, w = shape
        m = torch.ones((n, h, w), dtype=torch.bool, device=device)
        for b, (ih, iw) in enumerate(image_sizes):
            m[b, :int(np.ceil(float(ih) / s)), :int(np.ceil(float(iw) / s))] = 0
        masks.append(m)
    return masks


def dim_t(num_pos_feats, temperature=10000, device=None, dtype=torch.float32):
    d = torch.arange(num_pos_feats, dtype=dtype, device=device)
    return temperature ** (2 * (d // 2) / num_pos_feats)


def position_sine(mask, num_pos_feats, temperature=10000, dtype=torch.float32):
    """PositionEmbeddingSine(num_pos_feats, temperature, normalize=True) of a padding mask [B, H, W]: [B, 2 num_pos_feats, H, W] in `dtype`"""
    not_mask = ~mask
    y_embed = not_mask.cumsum(1, dtype=dtype)
    x_embed = not_mask.cumsum(2, dtype=dtype)
    scale = 2 * math.pi
    y_embed = y_embed / (y_embed[:, -1:, :] + 1e-6) * scale
    x_embed = x_embed / (x_embed[:, :, -1:] + 1e-6) * scale
    dt = dim_t(num_pos_feats, temperature, mask.device, dtype)
    pos_x = x_embed[:, :, :, None] / dt
    pos_y = y_embed[:, :, :, None] / dt
    pos_x = torch.stack((pos_x[:, :, :, 0::2].sin(), pos_x[:, :, :, 1::2].cos()), dim=4).flatten(3)
    pos_y = torch.stack((pos_y[:, :, :, 0::2].sin(), pos_y[:, :, :, 1::2].cos()), dim=4).flatten(3)
    return torch.cat((pos_y, pos_x), dim=3).permute(0, 3, 1, 2)


def box_cxcywh_to_xyxy(x):
    x_c, y_c, w, h = x.unbind(-1)
    return torch.stack([(x_c - 0.5 * w), (y_c - 0.5 * h), (x_c + 0.5 * w), (y_c + 0.5 * h)], dim=-1)


def box_xyxy_to_cxcywh(x):
    x0, y0, x1, y1 = x.unbind(-1)
    return torch.stack([(x0 + x1) / 2, (y0 + y1) / 2, (x1 - x0), (y1 - y0)], dim=-1)


def prepare_targets(gt_boxes, gt_classes, image_sizes):
    """per image {"labels", "boxes"}: XYXY absolute boxes / [w, h, w, h], then cxcywh"""
    out = []
    for boxes, labels, (h, w) in zip(gt_boxes, gt_classes, image_sizes):
        size = torch.as_tensor([w, h, w, h], dtype=boxes.dtype, device=boxes.device)
        out.append({"labels": labels, "boxes": box_xyxy_to_cxcywh(boxes / size)})
    return out


def scores(box_cls):
    """softmax over all logits, max over the classes without no-object: (score [B, Q], label [B, Q], lowest index on ties)"""
    return F.softmax(box_cls, dim=-1)[:, :, :-1].max(-1)


def postprocess_boxes(box_pred, image_size, out_size):
    """the box chain of `inference` and detector_postprocess for one image's kept boxes [k, 4] (cxcywh): (xyxy clipped [k, 4], nonempty [k])"""
    h, w = image_size
    oh, ow = out_size
    b = box_cxcywh_to_xyxy(box_pred)
    b[:, 0::2] *= w  # Boxes.scale(scale_x=image_size[1], scale_y=image_size[0])
    b[:, 1::2] *= h
    b[:, 0::2] *= ow / w  # detector_postprocess: Boxes.scale(output / image), Boxes.clip, nonempty
    b[:, 1::2] *= oh / h
    assert torch.isfinite(b).all(), "Box tensor contains infinite or NaN!"
    b = torch.stack((b[:, 0].clamp(min=0, max=ow), b[:, 1].clamp(min=0, max=oh), b[:, 2].clamp(min=0, max=ow), b[:, 3].clamp(min=0, max=oh)), dim=-1)
    return b, ((b[:, 2] - b[:, 0]) > 0) & ((b[:, 3] - b[:, 1]) > 0)


def inference(box_cls, box_pred, image_sizes, out_sizes, ignore_thresh):
    """per image {"keep": query indices, "scores", "labels" int64, "boxes" xyxy [k, 4]} of the queries above the threshold with nonempty boxes"""
    s, lab = scores(box_cls)
    out = []
    for b in range(box_cls.shape[0]):
        idx = (s[b] > ignore_thresh).nonzero().flatten()
        boxes, ne = postprocess_boxes(box_pred[b][idx], image_sizes[b], out_sizes[b])
        out.append({"keep": idx[ne], "scores": s[b][idx][ne], "labels": lab[b][idx][ne], "boxes": boxes[ne]})
    return out


class StandInBackbone(nn.Module):
    """res4 / res5 at strides 16 / 32 from strided convolutions with ReLU: a cheap trainable backbone whose feature maps are floor(Hp / 16)
    rows, so that ceil(h / stride) reaches past them on some images"""

    def __init__(self, channels=(32, 64)):
        super().__init__()
        self.channels = tuple(channels)
        self.stem = nn.Conv2d(3, channels[0], 16, stride=16)
        self.res5 = nn.Conv2d(channels[0], channels[1], 2, stride=2)

    @property
    def size_divisibility(self):
        return 0

    def output_shape(self):
        return {k: types.SimpleNamespace(channels=c, stride=s, height=None, width=None) for k, c, s in zip(("res4", "res5"), self.channels, (16, 32))}

    def forward(self, x):
        r4 = F.relu(self.stem(x))
        return {"res4": r4, "res5": F.relu(self.res5(r4))}


def standin_state_dict(seed, channels=(32, 64)):
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for name, cin, cout, k in (("stem", 3, channels[0], 16), ("res5", channels[0], channels[1], 2)):
        sd[f"{name}.weight"] = torch.randn(cout, cin, k, k, generator=g) * (2.0 / (cin * k * k)) ** 0.5
        sd[f"{name}.bias"] = torch.randn(cout, generator=g) * 0.1
    return sd


def weight_dict(l1_weight, giou_weight, dec_layers, deep_supervision):
    """the reference's weight_dict (:102-108)"""
    wd = {"loss_ce": 1, "loss_bbox": l1_weight, "loss_giou": giou_weight}
    if deep_supervision:
        aux = {}
        for i in range(dec_layers - 1):
            aux.update({k + f"_{i}": v for k, v in wd.items()})
        wd.update(aux)
    return wd


def weighted(loss_dict, wd):
    """loss_dict[k] * wd[k] for the keys in wd, in the loss dict's order (:172-175)"""
    return {k: (v * wd[k] if k in wd else v) for k, v in loss_dict.items()}
