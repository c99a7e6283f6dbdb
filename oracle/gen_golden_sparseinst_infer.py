"""TEST INFRASTRUCTURE -- generates tests/golden/sparseinst_infer.npz from the UNMODIFIED reference meta-architecture
(yolov7/modeling/meta_arch/sparseinst.py), loaded as oracle/gen_golden_sparseinst_encoder.py and oracle/gen_golden_sparseinst_criterion.py load
the transcoders and the loss, with stand-ins for detectron2's structures (ImageList, Instances, BitMasks) and build_backbone, and for alfred.
`SparseInst.preprocess_inputs` and `SparseInst.inference` are called on a stub `self` carrying the device, the pixel statistics and the two
thresholds.  Cases (fp32 on the CPU):
  - a_mixed: three images of different sizes in one padded batch; original sizes larger than one image and smaller than another;
  - b_empty: an image with no kept query next to one with kept queries;
  - c_ties: duplicated class logits (pins the lowest-index tie of max(dim));
  - d_near: mask logits whose sigmoid lies close to MASK_THRESHOLD.
The fixture also stores the reference meta-architecture's state_dict keys and shapes, built on oracle.sparseinst_infer_oracle.StandInBackbone.
Run where the reference tree is available (YB200_REFERENCE):   python -m oracle.gen_golden_sparseinst_infer"""
import importlib
import os
import sys
import types

import numpy as np
import torch
import torch.nn.functional as F

from . import ref_shim
from . import sparseinst_infer_oracle as sio
from .gen_golden_sparseinst_criterion import load_reference as load_loss
from .gen_golden_sparseinst_encoder import load_encoder_module

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "sparseinst_infer.npz")
MEAN, STD = (123.675, 116.280, 103.530), (58.395, 57.120, 57.375)
CLS_THRESHOLD, MASK_THRESHOLD = 0.01, 0.45
# name: (seed, N, K, per-image (h, w), per-image original (H0, W0), uint8 images)
CASES = {
    "a_mixed": (1, 12, 6, [(64, 96), (50, 70), (33, 41)], [(80, 120), (40, 56), (66, 82)], True),
    "b_empty": (2, 10, 5, [(64, 64), (40, 60)], [(64, 64), (30, 45)], False),
    "c_ties": (3, 16, 8, [(32, 64), (30, 50)], [(48, 96), (15, 25)], True),
    "d_near": (4, 8, 4, [(64, 64), (60, 48)], [(96, 96), (45, 36)], True),
}


class _ImageList:
    """detectron2.structures.ImageList.from_tensors: pad to the batch maximum rounded up to size_divisibility with 0"""

    def __init__(self, tensor, image_sizes):
        self.tensor, self.image_sizes = tensor, image_sizes

    @staticmethod
    def from_tensors(tensors, size_divisibility=0, pad_value=0.0):
        sizes = [tuple(t.shape[-2:]) for t in tensors]
        h, w = max(s[0] for s in sizes), max(s[1] for s in sizes)
        if size_divisibility > 1:
            h, w = -(-h // size_divisibility) * size_divisibility, -(-w // size_divisibility) * size_divisibility
        out = tensors[0].new_full((len(tensors), tensors[0].shape[0], h, w), pad_value)
        for i, t in enumerate(tensors):
            out[i, :, :t.shape[-2], :t.shape[-1]].copy_(t)
        return _ImageList(out, sizes)


class _Instances:
    def __init__(self, image_size, **kw):
        self.image_size = image_size
        self.__dict__.update(kw)


class _BitMasks:
    def __init__(self, tensor):
        self.tensor = tensor


def load_meta_arch():
    load_encoder_module()
    load_loss()
    d2m = sys.modules["detectron2.modeling"]
    d2m.build_backbone = lambda cfg: sio.StandInBackbone(cfg.STANDIN_CHANNELS)
    ref_shim._mod("detectron2.structures", ImageList=_ImageList, Instances=_Instances, BitMasks=_BitMasks)
    sys.modules["alfred"].print_shape = lambda *a, **k: None
    ref_shim._pkg("yolov7.modeling.meta_arch", os.path.join(ref_shim.REF, "yolov7", "modeling", "meta_arch"))
    return importlib.import_module("yolov7.modeling.meta_arch.sparseinst")


def cfg_of(channels=(64, 128, 256), decoder="GroupIAMDecoder"):
    ns = types.SimpleNamespace
    dec = ns(NAME=decoder, SCALE_FACTOR=2.0, OUTPUT_IAM=False, NUM_MASKS=100, KERNEL_DIM=128, NUM_CLASSES=80, GROUPS=4, INST=ns(DIM=256, CONVS=4),
             MASK=ns(DIM=256, CONVS=4))
    loss = ns(NAME="SparseInstCriterion", ITEMS=("labels", "masks"), CLASS_WEIGHT=2.0, MASK_PIXEL_WEIGHT=5.0, MASK_DICE_WEIGHT=2.0,
              OBJECTNESS_WEIGHT=1.0)
    sp = ns(ENCODER=ns(NAME="InstanceContextEncoder", NUM_CHANNELS=256, IN_FEATURES=["res3", "res4", "res5"], NORM=""), DECODER=dec, LOSS=loss,
            MATCHER=ns(NAME="SparseInstMatcher", ALPHA=0.8, BETA=0.2), MASK_THRESHOLD=MASK_THRESHOLD, MAX_DETECTIONS=100, CLS_THRESHOLD=0.005)
    return ns(MODEL=ns(DEVICE="cpu", PIXEL_MEAN=list(MEAN), PIXEL_STD=list(STD), BACKBONE=ns(NAME="build_sparseinst_standin_backbone", FREEZE_AT=0),
                       SPARSE_INST=sp, YOLO=ns(CONF_THRESHOLD=CLS_THRESHOLD)),
              INPUT=ns(MASK_FORMAT="bitmask"), STANDIN_CHANNELS=tuple(channels))


def case_inputs(name):
    """images, decoder outputs (pred_logits [B, N, K], pred_scores [B, N, 1], pred_masks [B, N, Hp/4, Wp/4]) and batched_inputs"""
    seed, N, K, sizes, ori, u8 = CASES[name]
    g = torch.Generator().manual_seed(seed)
    images = [(torch.randint(0, 256, (3, h, w), generator=g, dtype=torch.uint8) if u8 else torch.rand(3, h, w, generator=g) * 255) for h, w in sizes]
    hp, wp = (-(-max(s[i] for s in sizes) // 32) * 32 for i in (0, 1))
    B = len(sizes)
    logits = torch.randn(B, N, K, generator=g) * 2 - 1
    obj = torch.randn(B, N, 1, generator=g) * 2
    masks = torch.randn(B, N, hp // 4, wp // 4, generator=g) * 3
    if name == "b_empty":
        logits[1] -= 30  # sqrt(sigmoid(-31) ...) << CLS_THRESHOLD
    if name == "c_ties":
        logits[:, :, 5] = logits[:, :, 2]
        logits[:, :, 2] += 5  # the largest class appears twice: at 2 and 5
        logits[:, :, 5] = logits[:, :, 2]
    if name == "d_near":
        t = float(np.log(MASK_THRESHOLD / (1 - MASK_THRESHOLD)))
        masks = t + (masks - masks.mean()) * 1e-3
    batched = [{"image": im, "height": h0, "width": w0} for im, (h0, w0) in zip(images, ori)]
    return images, logits, obj, masks, batched


def main():
    mod = load_meta_arch()
    res = {}
    stub = types.SimpleNamespace(device=torch.device("cpu"), pixel_mean=torch.Tensor(MEAN).view(3, 1, 1), pixel_std=torch.Tensor(STD).view(3, 1, 1),
                                 cls_threshold=CLS_THRESHOLD, mask_threshold=MASK_THRESHOLD)
    stub.normalizer = lambda x: mod.SparseInst.normalizer(stub, x)
    for name in CASES:
        images, logits, obj, masks, batched = case_inputs(name)
        il = mod.SparseInst.preprocess_inputs(stub, batched)
        res[f"{name}/images"] = il.tensor.numpy()
        out = {"pred_logits": logits, "pred_scores": obj, "pred_masks": masks}
        results = mod.SparseInst.inference(stub, out, batched, il.tensor.shape[2:], il.image_sizes)
        for b, r in enumerate(results):
            key = f"{name}/{b}"
            res[f"{key}/scores"] = r.scores.numpy()
            res[f"{key}/labels"] = r.pred_classes.numpy()
            res[f"{key}/has_masks"] = np.array(hasattr(r, "pred_masks"))
            if hasattr(r, "pred_masks"):
                res[f"{key}/masks"] = np.packbits(r.pred_masks.numpy(), axis=-1)
                res[f"{key}/mask_shape"] = np.array(r.pred_masks.shape)
    model = mod.SparseInst(cfg_of())
    sd = model.state_dict()
    res["state_dict/keys"] = np.array(list(sd.keys()))
    res["state_dict/shapes"] = np.array([",".join(str(d) for d in v.shape) for v in sd.values()])
    np.savez_compressed(OUT, **res)
    print("wrote", OUT, "%.1f KB" % (os.path.getsize(OUT) / 1e3))


if __name__ == "__main__":
    main()
