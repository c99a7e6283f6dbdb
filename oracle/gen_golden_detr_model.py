"""TEST INFRASTRUCTURE -- generates tests/golden/detr_model.npz from the UNMODIFIED reference meta-architecture (yolov7/modeling/meta_arch/detr.py:
`Detr`, `MaskedBackboneTraceFriendly`) and backbone helpers (yolov7/modeling/backbone/detr_backbone.py: `Joiner`, `PositionEmbeddingSine`),
loaded as oracle/gen_golden_detr_criterion.load_reference() loads them.  detectron2 is not part of the reference tree, so its pieces are
stand-ins here: `build_backbone` (a stand-in backbone), `ImageList` (oracle/gen_golden_sparseinst_infer._ImageList), `Instances`, `Boxes`,
and a restatement of `detector_postprocess` (detectron2/modeling/postprocessing.py: Boxes.scale by output / image size, Boxes.clip with its
finiteness assertion, then nonempty()).  Cases (fp32 on the CPU):
  - u8_ragged: a ragged uint8 batch: the normalised batch, and the masks and sine positions of four levels (strides 4 / 8 with ceil-sized maps,
    16 / 32 with floor-sized ones, so that ceil(h / stride) reaches past the map on some images);
  - f32: an fp32 batch: the normalised batch and the masks;
  - infer: `inference` + detector_postprocess with original sizes larger and smaller than the input, an image with no kept query, exact logit
    ties, scores within 1e-7 of the threshold and boxes that clip to empty;
  - targets: `prepare_targets` with an image without targets;
  - state_dict: the keys and shapes of the reference `Detr(cfg)` at the torchvision DETR config's sizes on the stand-in backbone;
  - train: one reference `Detr` training forward (dropout 0, 256 wide, 8 heads, 2 + 2 layers, deep supervision) on the stand-in backbone: the
    weighted loss dict (keys, order, values) and the network outputs and targets it was computed from.
Run where the reference tree is available (YB200_REFERENCE):   python -m oracle.gen_golden_detr_model"""
import os
import types

import numpy as np
import torch

from . import detr_model_oracle as dmo
from .gen_golden_detr_criterion import load_reference
from .gen_golden_sparseinst_infer import _ImageList

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "detr_model.npz")
MEAN, STD = (123.675, 116.280, 103.530), (58.395, 57.120, 57.375)
THRESH = 0.3
NUM_POS_FEATS = 16
LEVELS = ((4, "ceil"), (8, "ceil"), (16, "floor"), (32, "floor"))
IMAGES = {"u8_ragged": ([(50, 70), (64, 45), (33, 81)], True), "f32": ([(40, 56), (47, 33)], False)}
INFER = dict(B=4, Q=30, K1=8, sizes=[(64, 81), (50, 70), (33, 45), (60, 60)], out=[(128, 160), (25, 35), (33, 45), (90, 40)])
TARGETS = dict(sizes=[(64, 81), (50, 70), (33, 45)], counts=[5, 0, 3])
TRAIN = dict(sizes=[(64, 96), (50, 70), (40, 90)], counts=[3, 0, 2], K=7, Q=10)


class _Instances:
    def __init__(self, image_size, **kw):
        self.image_size = image_size
        self.__dict__.update(kw)

    def to(self, device):
        return self


class _Boxes:
    def __init__(self, tensor):
        self.tensor = tensor

    def scale(self, scale_x, scale_y):
        self.tensor[:, 0::2] *= scale_x
        self.tensor[:, 1::2] *= scale_y


def detector_postprocess(results, output_height, output_width):
    """detectron2's detector_postprocess for boxes, restated"""
    scale_x, scale_y = output_width / results.image_size[1], output_height / results.image_size[0]
    boxes = results.pred_boxes
    boxes.scale(scale_x, scale_y)
    t = boxes.tensor
    assert torch.isfinite(t).all(), "Box tensor contains infinite or NaN!"
    t = torch.stack((t[:, 0].clamp(min=0, max=output_width), t[:, 1].clamp(min=0, max=output_height), t[:, 2].clamp(min=0, max=output_width),
                     t[:, 3].clamp(min=0, max=output_height)), dim=-1)
    keep = ((t[:, 2] - t[:, 0]) > 0) & ((t[:, 3] - t[:, 1]) > 0)
    return _Instances((output_height, output_width), pred_boxes=_Boxes(t[keep]), scores=results.scores[keep], pred_classes=results.pred_classes[keep])


class _ShapeBackbone(torch.nn.Module):
    """zero features at LEVELS' strides: ceil(Hp / s) or floor(Hp / s) rows and columns"""

    def __init__(self, channels=16):
        super().__init__()
        self.channels = channels

    def output_shape(self):
        return {f"p{s}": types.SimpleNamespace(channels=self.channels, stride=s) for s, _ in LEVELS}

    def forward(self, x):
        hp, wp = x.shape[-2:]
        r = lambda n, s, how: -(-n // s) if how == "ceil" else n // s
        return {f"p{s}": torch.zeros(x.shape[0], self.channels, r(hp, s, how), r(wp, s, how)) for s, how in LEVELS}


def image_case(name):
    sizes, u8 = IMAGES[name]
    g = torch.Generator().manual_seed(len(name))
    return [(torch.randint(0, 256, (3, h, w), generator=g, dtype=torch.uint8) if u8 else torch.rand(3, h, w, generator=g) * 255) for h, w in sizes]


def infer_case():
    B, Q, K1 = INFER["B"], INFER["Q"], INFER["K1"]
    g = torch.Generator().manual_seed(3)
    logits = torch.randn(B, Q, K1, generator=g) * 2
    boxes = torch.sigmoid(torch.randn(B, Q, 4, generator=g))
    logits[2, :, -1] += 30  # no-object dominates: nothing kept on image 2
    logits[:, :5, 1] = logits[:, :5, 3] = 6.0  # exact ties between classes 1 and 3: class 1 wins
    # image 3, queries 0..11: one logit a_q and zeros elsewhere, p_max = e^a / (e^a + K1 - 1) within 1e-7 of THRESH
    a = float(np.log((K1 - 1) * THRESH / (1 - THRESH)))
    logits[3, :12] = 0.0
    logits[3, :12, 2] = torch.tensor([np.float32(a) + k * 2.0 ** -22 for k in range(-6, 6)], dtype=torch.float32)
    # boxes that clip to empty on kept queries of images 0 and 1: entirely left of / below / right of the image
    for b in (0, 1):
        logits[b, 10:13, 0] = 12.0
        boxes[b, 10] = torch.tensor([-0.3, 0.5, 0.2, 0.2])
        boxes[b, 11] = torch.tensor([0.5, 1.4, 0.3, 0.2])
        boxes[b, 12] = torch.tensor([1.0, 0.5, 0.0, 0.3])  # zero width at the right edge
    return logits, boxes


def targets_case():
    g = torch.Generator().manual_seed(4)
    boxes, classes = [], []
    for (h, w), n in zip(TARGETS["sizes"], TARGETS["counts"]):
        xy = torch.rand(n, 2, generator=g) * torch.tensor([w * 0.7, h * 0.7])
        wh = torch.rand(n, 2, generator=g) * torch.tensor([w * 0.3, h * 0.3]) + 0.5
        boxes.append(torch.cat([xy, xy + wh], 1))
        classes.append(torch.randint(0, 80, (n,), generator=g))
    return boxes, classes


def cfg_of(hidden=256, nheads=8, enc=6, dec=6, ffn=2048, queries=100, classes=80, dropout=0.1, device="cpu", backbone="build_detr_standin_backbone"):
    """the torchvision DETR config's MODEL keys (configs/coco/detr/detr_256_6_6_torchvision.yaml) with the stand-in backbone"""
    ns = types.SimpleNamespace
    detr = ns(NUM_CLASSES=classes, HIDDEN_DIM=hidden, NUM_OBJECT_QUERIES=queries, NHEADS=nheads, DROPOUT=dropout, DIM_FEEDFORWARD=ffn, ENC_LAYERS=enc,
              DEC_LAYERS=dec, PRE_NORM=False, GIOU_WEIGHT=2.0, L1_WEIGHT=5.0, DEEP_SUPERVISION=True, NO_OBJECT_WEIGHT=0.1, FROZEN_WEIGHTS="")
    return ns(MODEL=ns(DEVICE=device, PIXEL_MEAN=list(MEAN), PIXEL_STD=list(STD), MASK_ON=False, BACKBONE=ns(NAME=backbone, FREEZE_AT=0),
                       YOLO=ns(CONF_THRESHOLD=THRESH), DETR=detr))


def train_case():
    g = torch.Generator().manual_seed(5)
    batched, boxes, classes = [], [], []
    for (h, w), n in zip(TRAIN["sizes"], TRAIN["counts"]):
        img = torch.randint(0, 256, (3, h, w), generator=g, dtype=torch.uint8)
        xy = torch.rand(n, 2, generator=g) * torch.tensor([w * 0.6, h * 0.6])
        wh = torch.rand(n, 2, generator=g) * torch.tensor([w * 0.35, h * 0.35]) + 2.0
        bx, cl = torch.cat([xy, xy + wh], 1), torch.randint(0, TRAIN["K"], (n,), generator=g)
        boxes.append(bx)
        classes.append(cl)
        batched.append({"image": img, "height": h, "width": w, "instances": _Instances((h, w), gt_boxes=_Boxes(bx), gt_classes=cl)})
    return batched, boxes, classes


def load_meta_arch():
    detr, misc = load_reference()
    detr.ImageList, detr.Instances, detr.Boxes, detr.detector_postprocess = _ImageList, _Instances, _Boxes, detector_postprocess
    return detr, misc


def main():
    detr, _ = load_meta_arch()
    res = {}
    stub = types.SimpleNamespace(device=torch.device("cpu"), ignore_thresh=THRESH, mask_on=False)
    mean, std = torch.Tensor(MEAN).view(3, 1, 1), torch.Tensor(STD).view(3, 1, 1)
    stub.normalizer = lambda x: (x - mean) / std
    detr.build_backbone = lambda cfg: _ShapeBackbone()
    cfg = cfg_of()
    for name in IMAGES:
        il = detr.Detr.preprocess_image(stub, [{"image": im} for im in image_case(name)])
        res[f"{name}/images"] = il.tensor.numpy()
        joiner = detr.Joiner(detr.MaskedBackboneTraceFriendly(cfg), detr.PositionEmbeddingSine(NUM_POS_FEATS, normalize=True))
        feats, pos = joiner(il)
        for l, (f, p) in enumerate(zip(feats, pos)):
            res[f"{name}/mask{l}"] = f.mask.numpy()
            if name == "u8_ragged":
                res[f"{name}/pos{l}"] = p.numpy()
    logits, boxes = infer_case()
    sizes = [tuple(s) for s in INFER["sizes"]]
    results = detr.Detr.inference(stub, logits, boxes.clone(), None, sizes)
    for b, (r, (oh, ow)) in enumerate(zip(results, INFER["out"])):
        r = detector_postprocess(r, oh, ow)
        res[f"infer/{b}/scores"], res[f"infer/{b}/labels"], res[f"infer/{b}/boxes"] = r.scores.numpy(), r.pred_classes.numpy(), r.pred_boxes.tensor.numpy()
    tb, tc = targets_case()
    insts = [_Instances(s, gt_boxes=_Boxes(b), gt_classes=c) for s, b, c in zip(TARGETS["sizes"], tb, tc)]
    for b, t in enumerate(detr.Detr.prepare_targets(stub, insts)):
        res[f"targets/{b}/labels"], res[f"targets/{b}/boxes"] = t["labels"].numpy(), t["boxes"].numpy()
    # state_dict of the reference model at the torchvision config's sizes
    detr.build_backbone = lambda cfg: dmo.StandInBackbone()
    sd = detr.Detr(cfg).state_dict()
    res["state_dict/keys"] = np.array(list(sd.keys()))
    res["state_dict/shapes"] = np.array([",".join(str(d) for d in v.shape) for v in sd.values()])
    # one training forward
    torch.manual_seed(6)
    model = detr.Detr(cfg_of(enc=2, dec=2, ffn=64, queries=TRAIN["Q"], classes=TRAIN["K"], dropout=0.0))
    model.detr.backbone[0].backbone.load_state_dict(dmo.standin_state_dict(7))
    model.train()
    cap = {}
    model.detr.register_forward_hook(lambda m, i, o: cap.update(o))
    batched, _, _ = train_case()
    losses = model(batched)
    layers = list(cap["aux_outputs"]) + [cap]
    res["train/logits"] = np.stack([o["pred_logits"].detach().numpy() for o in layers])
    res["train/boxes"] = np.stack([o["pred_boxes"].detach().numpy() for o in layers])
    res["train/keys"] = np.array(list(losses.keys()))
    res["train/values"] = np.array([float(v.detach()) for v in losses.values()], dtype=np.float32)
    res["train/weight_keys"] = np.array(list(model.criterion.weight_dict.keys()))
    res["train/weight_values"] = np.array(list(model.criterion.weight_dict.values()), dtype=np.float64)
    np.savez_compressed(OUT, **res)
    print("wrote", OUT, "%.1f KB" % (os.path.getsize(OUT) / 1e3))


if __name__ == "__main__":
    main()
