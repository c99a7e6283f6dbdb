"""TEST INFRASTRUCTURE -- generates tests/golden/sparseinst_criterion.npz from the UNMODIFIED reference SparseInstMatcher and SparseInstCriterion
(yolov7/modeling/loss/sparseinst_loss.py and yolov7/utils/misc.py imported through oracle/ref_shim.py).  fvcore is not installed: its
`sigmoid_focal_loss_jit` is stubbed with fvcore's formula evaluated in the inputs' dtype, and detectron2's Registry with ref_shim's.
Run where the reference tree is available (YB200_REFERENCE):   python -m oracle.gen_golden_sparseinst_criterion

Everything runs in fp64.  Per case: the inputs, the per-image cost blocks, the assignment, the weighted loss dict and the autograd gradients of
Σ coef[k] · loss[k] with respect to pred_logits, pred_masks and pred_scores.  To keep the fixture small:
  - mask logits are int8 codes × 2^-4 (exact in fp32); no code lies within 2^-8 of logit(0.4), so σ(m) >= 0.4 is decided alike in fp32 and fp64;
  - ground-truth masks are stored with np.packbits;
  - d pred_masks is kept on matched rows only (the others are zero), d pred_logits on matched rows plus UNMATCHED_ROWS unmatched rows per image.
Every resized target value is either exactly 0.5 in fp32 and fp64 or at least 1e-5 away from it, so t > 0.5 is decided alike too."""
import importlib
import math
import os
import sys
import types

import numpy as np
import torch
import torch.nn.functional as F

from . import ref_shim
from . import sparseinst_criterion_oracle as sco

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "sparseinst_criterion.npz")
LOGIT_STEP = 2.0 ** -4
UNMATCHED_ROWS = 3
DEFAULT_W = (2.0, 5.0, 2.0, 1.0)  # CLASS, MASK_PIXEL, MASK_DICE, OBJECTNESS weights of config_sparseinst.py

# name: (B, N, K, (H, W), input_shape, per-image (h, w), targets per image, (alpha, beta), weights (class, mask, dice, objectness), items)
CASES = {
    "a_pad": (2, 100, 80, (40, 40), (160, 160), [(150, 140), (120, 160)], [3, 5], (0.8, 0.2), DEFAULT_W, ("labels", "masks")),
    "b_empty_image": (2, 20, 10, (20, 20), (80, 80), [(70, 80), (80, 60)], [0, 4], (0.8, 0.2), DEFAULT_W, ("labels", "masks")),
    "c_ragged": (2, 16, 12, (24, 22), (100, 90), [(100, 90), (87, 71)], [4, 2], (0.8, 0.2), DEFAULT_W, ("labels", "masks")),
    "d_weights": (1, 30, 20, (32, 32), (128, 128), [(128, 120)], [6], (0.5, 0.7), (3.0, 4.0, 1.5, 0.7), ("labels", "masks", "loss_objectness")),
    "e_g_eq_n": (2, 12, 8, (16, 16), (64, 64), [(64, 64), (50, 60)], [12, 3], (0.8, 0.2), DEFAULT_W, ("labels", "masks")),
}


def _cfg(N, K, alpha, beta, weights, items):
    ns = types.SimpleNamespace
    return ns(MODEL=ns(SPARSE_INST=ns(LOSS=ns(NAME="SparseInstCriterion", ITEMS=items, CLASS_WEIGHT=weights[0], MASK_PIXEL_WEIGHT=weights[1],
                                              MASK_DICE_WEIGHT=weights[2], OBJECTNESS_WEIGHT=weights[3]),
                                      MATCHER=ns(NAME="SparseInstMatcher", ALPHA=alpha, BETA=beta), DECODER=ns(NUM_CLASSES=K, NUM_MASKS=N))))


def load_reference():
    ref_shim.install()
    fv = types.ModuleType("fvcore")
    fv.__path__ = []
    fvnn = types.ModuleType("fvcore.nn")

    def sigmoid_focal_loss_jit(inputs, targets, alpha: float = -1, gamma: float = 2, reduction: str = "none"):
        p = torch.sigmoid(inputs)
        ce_loss = F.binary_cross_entropy_with_logits(inputs, targets, reduction="none")
        p_t = p * targets + (1 - p) * (1 - targets)
        loss = ce_loss * ((1 - p_t) ** gamma)
        if alpha >= 0:
            alpha_t = alpha * targets + (1 - alpha) * (1 - targets)
            loss = alpha_t * loss
        if reduction == "mean":
            loss = loss.mean()
        elif reduction == "sum":
            loss = loss.sum()
        return loss

    fvnn.sigmoid_focal_loss_jit = sigmoid_focal_loss_jit
    sys.modules["fvcore"], sys.modules["fvcore.nn"] = fv, fvnn
    u = sys.modules.get("detectron2.utils") or types.ModuleType("detectron2.utils")
    u.__path__ = []
    reg = types.ModuleType("detectron2.utils.registry")
    reg.Registry = lambda name: ref_shim._Registry()
    sys.modules["detectron2.utils"], sys.modules["detectron2.utils.registry"] = u, reg
    ref_shim._pkg("yolov7.modeling.loss", os.path.join(ref_shim.REF, "yolov7", "modeling", "loss"))
    return importlib.import_module("yolov7.modeling.loss.sparseinst_loss")


def ellipses(g, n, h, w):
    """n random filled ellipses inside an h x w image (bool [n, h, w])"""
    yy, xx = torch.meshgrid(torch.arange(h, dtype=torch.float64), torch.arange(w, dtype=torch.float64), indexing="ij")
    out = torch.zeros(n, h, w, dtype=torch.bool)
    for k in range(n):
        cy, cx = float(torch.rand(1, generator=g)) * h, float(torch.rand(1, generator=g)) * w
        ry, rx = 4 + float(torch.rand(1, generator=g)) * h / 3, 4 + float(torch.rand(1, generator=g)) * w / 3
        out[k] = ((yy - cy) / ry) ** 2 + ((xx - cx) / rx) ** 2 <= 1
    return out


def check_threshold_margin(mask_list, input_shape, size):
    t64 = sco.target_masks(mask_list, input_shape, size, torch.float64)
    t32 = sco.target_masks(mask_list, input_shape, size, torch.float32).double()
    near = ((t64 - 0.5).abs() < 1e-5) & ~((t64 == 0.5) & (t32 == 0.5))
    assert not near.any(), "a resized target value lies within 1e-5 of 0.5"


def avoid_band(codes):
    """move codes within 2^-8 of logit(0.4) one step away (none exist at a 2^-4 step; kept for other steps)"""
    thr = math.log(0.4 / 0.6)
    bad = ((codes.double() * LOGIT_STEP) - thr).abs() < 2.0 ** -8
    codes[bad] -= 1
    return codes


def make_case(g, B, N, K, size, input_shape, hw, sizes):
    mask_list = [ellipses(g, n, h, w) for n, (h, w) in zip(sizes, hw)]
    check_threshold_margin(mask_list, input_shape, size)
    tm = sco.target_masks(mask_list, input_shape, size, torch.float64)
    noise = torch.randn(B, N, *size, generator=g, dtype=torch.float64) * 2.5
    off = 0
    for b, n in enumerate(sizes):  # some queries resemble a target, so that dice and IoU are not all near zero
        perm = torch.randperm(N, generator=g)[:n]
        for j in range(n):
            noise[b, perm[j]] += 8.0 * (tm[off + j] - 0.5)
        off += n
    codes = avoid_band(torch.clamp(torch.round(noise / LOGIT_STEP), -127, 127).to(torch.int8))
    cls = (torch.randn(B, N, K, generator=g) * 2.0 - 2.0).float().double()
    scores = torch.randn(B, N, 1, generator=g).float().double()
    labels = torch.randint(0, K, (sum(sizes),), generator=g)
    return mask_list, codes, cls, scores, labels


def grad_rows(B, N, indices):
    rows = []
    for b in range(B):
        matched = set(indices[b][0].tolist())
        unmatched = [q for q in range(N) if q not in matched][:UNMATCHED_ROWS]
        rows += [b * N + q for q in sorted(matched) + unmatched]
    return np.array(sorted(rows), dtype=np.int64)


def main():
    mod = load_reference()
    out = {}
    g = torch.Generator().manual_seed(23)
    for name, (B, N, K, size, input_shape, hw, sizes, (alpha, beta), weights, items) in CASES.items():
        mask_list, codes, cls, scores, labels = make_case(g, B, N, K, size, input_shape, hw, sizes)
        cfg = _cfg(N, K, alpha, beta, weights, items)
        crit = mod.build_sparse_inst_criterion(cfg)
        lg = cls.clone().requires_grad_(True)
        mk = (codes.double() * LOGIT_STEP).requires_grad_(True)
        sc = scores.clone().requires_grad_(True)
        off = np.concatenate([[0], np.cumsum(sizes)])
        targets = [{"labels": labels[off[b]:off[b + 1]], "masks": sco.BitMasks(mask_list[b])} for b in range(B)]
        outputs = {"pred_logits": lg, "pred_masks": mk, "pred_scores": sc}
        losses = crit(outputs, targets, input_shape)
        coef = {k: float(c) for k, c in zip(sco.LOSS_KEYS, torch.rand(4, generator=g) * 2.0 + 0.25)}
        total = sum(coef[k] * v for k, v in losses.items())
        dl, dm, ds = torch.autograd.grad(total, (lg, mk, sc))
        indices = crit.matcher(outputs, targets, input_shape)
        # the reference matcher's cost, restricted to the per-image blocks (the same arithmetic as :320-340)
        with torch.no_grad():
            tm = sco.target_masks(mask_list, input_shape, size, torch.float64)
            dice = mod.dice_score(mk.detach().view(B * N, -1), tm.flatten(1))
            C = (dice ** alpha * lg.detach().sigmoid().view(B * N, -1)[:, labels] ** beta).view(B, N, -1)
            blocks = [blk[b].flatten() for b, blk in enumerate(C.split(sizes, -1))]
        rows = grad_rows(B, N, indices)
        mrows = np.array([b * N + int(q) for b, (i, _) in enumerate(indices) for q in i.tolist()], dtype=np.int64)
        p = name + "/"
        out.update({p + "dims": np.array([B, N, K, *size, *input_shape]), p + "sizes": np.array(sizes, dtype=np.int64),
                    p + "image_hw": np.array(hw, dtype=np.int64).reshape(B, 2),
                    p + "mask_bits": np.packbits(torch.cat([m.flatten() for m in mask_list]).numpy()) if sum(sizes) else np.zeros(0, np.uint8),
                    p + "logit_codes": codes.numpy(), p + "logit_step": np.float64(LOGIT_STEP),
                    p + "pred_logits": cls.float().numpy(), p + "pred_scores": scores.float().numpy(), p + "labels": labels.numpy(),
                    p + "alpha_beta": np.array([alpha, beta]), p + "weights": np.array(weights), p + "items": np.array(items),
                    p + "coef": np.array([coef[k] for k in sco.LOSS_KEYS]),
                    p + "cost": torch.cat(blocks).numpy() if blocks else np.zeros(0),
                    p + "idx_i": torch.cat([i for i, _ in indices]).numpy(), p + "idx_j": torch.cat([j for _, j in indices]).numpy(),
                    p + "keys": np.array(list(losses.keys())), p + "losses": np.array([float(v.detach()) for v in losses.values()]),
                    p + "grad_rows": rows, p + "dlogits": dl.reshape(B * N, K)[rows].numpy(),
                    p + "mask_rows": mrows, p + "dmasks": dm.reshape(B * N, -1)[mrows].numpy(), p + "dscores": ds.numpy()})
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, "%.1f KB" % (os.path.getsize(OUT) / 1e3))


if __name__ == "__main__":
    main()
