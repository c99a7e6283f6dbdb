"""TEST INFRASTRUCTURE -- plain-torch restatement of SparseInst's `preprocess_inputs` and `inference` (yolov7/modeling/meta_arch/sparseinst.py:96-100,
179-232), and a small stand-in backbone for the meta-architecture's tests.

Device-agnostic and dtype-following: in fp32 the operations run in torch's order (the reference's arithmetic, bit for bit on the same device),
in fp64 they are the exact yardstick.  Pinned by tests/golden/sparseinst_infer.npz, produced by oracle/gen_golden_sparseinst_infer.py from the
unmodified reference; tests/test_sparseinst_infer_oracle_golden.py re-checks this file against it on every CPU run.  Only tests/ and tools/
may import it.
"""
import types

import torch
import torch.nn as nn
import torch.nn.functional as F

SIZE_DIVISIBILITY = 32


def preprocess(images, mean, std, dtype=torch.float32, divisibility=SIZE_DIVISIBILITY):
    """(image - mean) / std per image ([3, h, w] uint8 or float), zero-padded to a multiple of `divisibility`: ([B, 3, Hp, Wp], [(h, w)])"""
    dev = images[0].device
    mean = torch.as_tensor(mean, dtype=dtype, device=dev).view(3, 1, 1)
    std = torch.as_tensor(std, dtype=dtype, device=dev).view(3, 1, 1)
    sizes = [(int(im.shape[1]), int(im.shape[2])) for im in images]
    hp = -(-max(h for h, _ in sizes) // divisibility) * divisibility
    wp = -(-max(w for _, w in sizes) // divisibility) * divisibility
    out = torch.zeros(len(images), 3, hp, wp, dtype=dtype, device=dev)
    for i, im in enumerate(images):
        out[i, :, :im.shape[1], :im.shape[2]] = (im - mean) / std
    return out, sizes


def scores(pred_logits, pred_scores):
    """sqrt(sigmoid(logits) * sigmoid(objectness)), then max over the classes: (score [B, N], label [B, N], lowest index on ties)"""
    s = torch.sqrt(pred_logits.sigmoid() * pred_scores.sigmoid())
    return s.max(dim=-1)


def composite(mask_logits, max_shape, img_shape, ori_shape):
    """sigmoid, bilinear to the padded size, crop to the image, bilinear to the original size (before the threshold): [k, H0, W0]"""
    h, w = img_shape
    m = F.interpolate(mask_logits.sigmoid().unsqueeze(1), size=tuple(max_shape), mode="bilinear", align_corners=False)[:, :, :h, :w]
    return F.interpolate(m, size=tuple(ori_shape), mode="bilinear", align_corners=False).squeeze(1)


def inference(pred_logits, pred_scores, pred_masks, max_shape, image_sizes, ori_shapes, cls_threshold, mask_threshold):
    """per image {"keep": query indices, "scores": rescored, "labels": int64, "masks": bool [k, H0, W0] or None when nothing is kept}"""
    score, label = scores(pred_logits, pred_scores)
    out = []
    for b in range(pred_logits.shape[0]):
        keep = score[b] > cls_threshold
        idx = keep.nonzero().flatten()
        s, lab = score[b][keep], label[b][keep]
        if s.numel() == 0:
            out.append({"keep": idx, "scores": s, "labels": lab, "masks": None})
            continue
        m = pred_masks[b][keep].sigmoid()
        p = (m > mask_threshold).to(m.dtype)
        s = s * ((m * p).sum([1, 2]) / (p.sum([1, 2]) + 1e-6))
        masks = composite(pred_masks[b][keep], max_shape, image_sizes[b], ori_shapes[b]) > mask_threshold
        out.append({"keep": idx, "scores": s, "labels": lab, "masks": masks})
    return out


class StandInBackbone(nn.Module):
    """res3 / res4 / res5 at strides 8 / 16 / 32 from strided convolutions with ReLU (channels multiples of 16): a cheap trainable backbone"""

    def __init__(self, channels=(64, 128, 256)):
        super().__init__()
        self.channels = tuple(channels)
        self.stem = nn.Conv2d(3, channels[0], 8, stride=8)
        self.res4 = nn.Conv2d(channels[0], channels[1], 2, stride=2)
        self.res5 = nn.Conv2d(channels[1], channels[2], 2, stride=2)

    @property
    def size_divisibility(self):
        return SIZE_DIVISIBILITY

    def output_shape(self):
        return {k: types.SimpleNamespace(channels=c, stride=s, height=None, width=None)
                for k, c, s in zip(("res3", "res4", "res5"), self.channels, (8, 16, 32))}

    def forward(self, x):
        r3 = F.relu(self.stem(x))
        r4 = F.relu(self.res4(r3))
        return {"res3": r3, "res4": r4, "res5": F.relu(self.res5(r4))}


def standin_state_dict(seed, channels=(64, 128, 256)):
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for name, cin, cout, k in (("stem", 3, channels[0], 8), ("res4", channels[0], channels[1], 2), ("res5", channels[1], channels[2], 2)):
        sd[f"{name}.weight"] = torch.randn(cout, cin, k, k, generator=g) * (2.0 / (cin * k * k)) ** 0.5
        sd[f"{name}.bias"] = torch.randn(cout, generator=g) * 0.1
    return sd
