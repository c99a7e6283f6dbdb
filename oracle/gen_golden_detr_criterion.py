"""TEST INFRASTRUCTURE -- generates tests/golden/detr_criterion.npz from the UNMODIFIED reference HungarianMatcher, SetCriterion, MLP and DETR
(yolov7/utils/detr_utils.py, yolov7/modeling/meta_arch/detr.py) imported through oracle/ref_shim.py plus the stubs detr.py's imports need.
Run where the reference tree is available (YB200_REFERENCE):   python -m oracle.gen_golden_detr_criterion

Per case: the inputs, the packed cost blocks (yb200_detr_match_cost's layout), the assignment, the loss values and the autograd gradients of
Σ w[l, k] · loss[l, k] with respect to every layer's logits and boxes.  Plus the DETR tail (input_proj, class_embed, bbox_embed, sigmoid) on a
small feature map.  To keep the fixture small, the logits are multiples of 2^-10 stored as int16 codes (exact in fp32), and the logit gradient is
kept on a sample of query rows: every matched row and the first UNMATCHED_ROWS unmatched rows of each (layer, image).  The box gradient is kept whole."""
import importlib
import os
import sys
import types

import numpy as np
import torch
import torch.nn as nn

from . import gen_golden_detr, ref_shim

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "detr_criterion.npz")

# name: (L, B, Q, K1, target counts per image, eos_coef, (cost_class, cost_bbox, cost_giou))
# (K1 = 21 is Pascal VOC's 20 classes + no-object; 81 and 92 are the cfg default and the original DETR's 91 + 1)
CASES = {
    "l6": (6, 1, 16, 81, [9], 0.1, (1.0, 5.0, 2.0)),
    "q100": (1, 1, 100, 81, [9], 0.1, (1.0, 5.0, 2.0)),
    "q300": (1, 1, 300, 21, [1], 0.1, (1.0, 5.0, 2.0)),
    "g_over_q": (2, 3, 8, 92, [12, 0, 8], 0.3, (2.0, 5.0, 2.0)),
    "empty": (2, 2, 10, 81, [0, 0], 0.1, (1.0, 5.0, 2.0)),
}
LOGIT_SCALE = 2.0 ** -10
UNMATCHED_ROWS = 3
LOSSES = ["labels", "boxes", "cardinality"]


def load_reference():
    gen_golden_detr.load_reference()  # ref_shim + detectron2.utils.comm
    for name, attrs in (("fvcore", {}), ("fvcore.nn", {"giou_loss": None, "smooth_l1_loss": None}),
                        ("detectron2.structures", {n: object for n in ("Boxes", "ImageList", "Instances", "BitMasks", "PolygonMasks")}),
                        ("detectron2.utils.logger", {"log_first_n": lambda *a, **k: None}),
                        ("alfred.utils", {}), ("alfred.utils.log", {"logger": sys.modules["alfred"].logger})):
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        m.__path__ = []
        sys.modules[name] = m
    sys.modules["detectron2.modeling"].build_backbone = None
    sys.modules["detectron2.modeling"].detector_postprocess = None
    ref_shim._pkg("yolov7.modeling.meta_arch", os.path.join(ref_shim.REF, "yolov7", "modeling", "meta_arch"))
    return importlib.import_module("yolov7.modeling.meta_arch.detr"), importlib.import_module("yolov7.utils.misc")


def _np(t):
    return t.detach().cpu().numpy()


def make_case(g, L, B, Q, K1, sizes):
    codes = torch.clamp(torch.round(torch.randn(L, B, Q, K1, generator=g) * 2.0 / LOGIT_SCALE), -32767, 32767).to(torch.int16)
    flat = codes.view(-1, K1)
    while True:  # a unique maximum per row, so that argmax / topk (cardinality_error, class_error) are not decided by tie-breaking
        tied = ((flat == flat.max(1, keepdim=True).values).sum(1) > 1).nonzero().flatten()
        if not len(tied):
            break
        flat[tied, flat[tied].argmax(1)] += 1
    logits = codes.float() * LOGIT_SCALE
    boxes = torch.sigmoid(torch.randn(L, B, Q, 4, generator=g))
    targets = []
    for n in sizes:
        cxcy = torch.rand(n, 2, generator=g) * 0.8 + 0.1
        wh = torch.rand(n, 2, generator=g) * 0.45 + 0.05
        targets.append({"labels": torch.randint(0, K1 - 1, (n,), generator=g), "boxes": torch.cat([cxcy, wh], 1)})
    return codes, logits, boxes, targets


def grad_rows(L, B, Q, indices):
    """flat [L*B*Q] indices of the query rows whose logit gradient the fixture keeps"""
    rows = []
    for l in range(L):
        for b in range(B):
            matched = set(indices[l][b][0].tolist())
            unmatched = [q for q in range(Q) if q not in matched][:UNMATCHED_ROWS]
            rows += [(l * B + b) * Q + q for q in sorted(matched) + unmatched]
    return np.array(sorted(rows), dtype=np.int64)

def loss_weights(g, L):
    """arbitrary non-unit weights [L, 3] of (loss_ce, loss_bbox, loss_giou) per layer (the last row is the model's output)"""
    return torch.rand(L, 3, generator=g) * 2.0 + 0.25


def main():
    detr, misc = load_reference()
    out = {}
    g = torch.Generator().manual_seed(11)
    for name, (L, B, Q, K1, sizes, eos, costs) in CASES.items():
        codes, logits, boxes, targets = make_case(g, L, B, Q, K1, sizes)
        w = loss_weights(g, L)
        matcher = detr.HungarianMatcher(cost_class=costs[0], cost_bbox=costs[1], cost_giou=costs[2])
        crit = detr.SetCriterion(K1 - 1, matcher=matcher, weight_dict={}, eos_coef=eos, losses=LOSSES)
        lg = [logits[l].clone().requires_grad_(True) for l in range(L)]
        bx = [boxes[l].clone().requires_grad_(True) for l in range(L)]
        outputs = {"pred_logits": lg[-1], "pred_boxes": bx[-1]}
        if L > 1:
            outputs["aux_outputs"] = [{"pred_logits": lg[l], "pred_boxes": bx[l]} for l in range(L - 1)]
        losses = crit(outputs, targets)
        total = 0
        vals = np.full((L, 5), np.nan, dtype=np.float32)
        for l in range(L):
            sfx = "" if l == L - 1 else f"_{l}"
            for k, key in enumerate(("loss_ce", "loss_bbox", "loss_giou")):
                total = total + w[l, k] * losses[key + sfx]
                vals[l, k] = float(losses[key + sfx].detach())
            vals[l, 3] = float(losses["cardinality_error" + sfx])
        vals[L - 1, 4] = float(losses["class_error"])
        total.backward()
        # the cost blocks and assignments of every layer, as the reference's matcher computes them (packed like yb200_detr_match_cost)
        blocks, ii, jj, idx = [], [], [], []
        for l in range(L):
            o = {"pred_logits": logits[l], "pred_boxes": boxes[l]}
            with torch.no_grad():
                bs, nq = o["pred_logits"].shape[:2]
                prob = o["pred_logits"].flatten(0, 1).softmax(-1)
                ob = o["pred_boxes"].flatten(0, 1)
                ids = torch.cat([t["labels"] for t in targets])
                tb = torch.cat([t["boxes"] for t in targets])
                c = matcher.cost_bbox * torch.cdist(ob, tb, p=1) + matcher.cost_class * -prob[:, ids] + \
                    matcher.cost_giou * -detr.generalized_box_iou(detr.box_cxcywh_to_xyxy(ob), detr.box_cxcywh_to_xyxy(tb))
                c = c.view(bs, nq, -1)
                for b, blk in enumerate(c.split(sizes, -1)):
                    blocks.append(blk[b].flatten())
            idx.append(matcher(o, targets))
            for i, j in idx[-1]:
                ii.append(i)
                jj.append(j)
        rows = grad_rows(L, B, Q, idx)
        p = name + "/"
        out.update({p + "dims": np.array([L, B, Q, K1]), p + "sizes": np.array(sizes), p + "eos_coef": np.float32(eos), p + "costs": np.array(costs),
                    p + "logit_codes": _np(codes), p + "logit_scale": np.float32(LOGIT_SCALE), p + "boxes": _np(boxes), p + "weights": _np(w), p + "losses": vals,
                    p + "labels": _np(torch.cat([t["labels"] for t in targets])), p + "tboxes": _np(torch.cat([t["boxes"] for t in targets]).reshape(-1, 4)),
                    p + "cost": _np(torch.cat(blocks)) if blocks else np.zeros(0, np.float32),
                    p + "idx_i": _np(torch.cat(ii)), p + "idx_j": _np(torch.cat(jj)),
                    p + "keys": np.array(list(losses.keys())),
                    p + "grad_rows": rows, p + "dlogits": np.stack([_np(t.grad) for t in lg]).reshape(-1, K1)[rows], p + "dboxes": np.stack([_np(t.grad) for t in bx])})

    # the DETR tail: stand-in backbone and transformer, so that input_proj, the heads and the sigmoid are what is pinned
    hidden, ch, nq, k1, L, B, H, W = 32, 48, 8, 81, 2, 2, 4, 5
    src = torch.randn(B, ch, H, W, generator=g)
    mask = torch.zeros(B, H, W, dtype=torch.bool)
    mask[1, :, 3:] = True
    pos = torch.randn(B, hidden, H, W, generator=g)
    hs = torch.randn(L, B, nq, hidden, generator=g)

    class Backbone(nn.Module):
        num_channels = ch

        def forward(self, samples):
            return [misc.NestedTensor(src, mask)], [pos]

    class Transformer(nn.Module):
        d_model = hidden

        def forward(self, x, m, query, p):
            self.seen = x.detach().clone()
            return hs, None

    torch.manual_seed(5)
    tr = Transformer()
    model = detr.DETR(Backbone(), tr, num_classes=k1 - 1, num_queries=nq, aux_loss=True)
    res = model(misc.NestedTensor(torch.zeros(B, 3, 8, 8), torch.zeros(B, 8, 8, dtype=torch.bool)))
    out.update({"heads/src": _np(src), "heads/mask": _np(mask), "heads/pos": _np(pos), "heads/hs": _np(hs), "heads/proj": _np(tr.seen),
                "heads/pred_logits": _np(res["pred_logits"]), "heads/pred_boxes": _np(res["pred_boxes"]),
                "heads/aux_logits": np.stack([_np(a["pred_logits"]) for a in res["aux_outputs"]]),
                "heads/aux_boxes": np.stack([_np(a["pred_boxes"]) for a in res["aux_outputs"]])})
    for k, v in model.state_dict().items():
        out["heads/sd/" + k] = _np(v)
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, "%.1f KB" % (os.path.getsize(OUT) / 1e3))


if __name__ == "__main__":
    main()
