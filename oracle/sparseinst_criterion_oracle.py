"""TEST INFRASTRUCTURE -- plain-torch restatement of SparseInst's matcher and criterion (yolov7/modeling/loss/sparseinst_loss.py:19-354).

Device-agnostic and dtype-following (the tests run it in fp64 on the CPU).  Pinned by tests/golden/sparseinst_criterion.npz, produced by
oracle/gen_golden_sparseinst_criterion.py from the unmodified reference; tests/test_sparseinst_criterion_oracle_golden.py re-checks this file
against those vectors on every CPU run.  Only tests/ and tools/ may import it.
"""
import torch
import torch.nn.functional as F
from scipy.optimize import linear_sum_assignment

LOSS_KEYS = ("loss_ce", "loss_objectness", "loss_dice", "loss_mask")


class BitMasks:
    """the part of detectron2's BitMasks the criterion reads: .tensor [g, h, w] and len()"""

    def __init__(self, tensor):
        self.tensor = tensor

    def __len__(self):
        return self.tensor.shape[0]


def target_masks(masks, input_shape, size, dtype):
    """nested_masks_from_list(masks, input_shape) then F.interpolate(bilinear, align_corners=False) to `size` (:320-331): [G, H, W] in dtype"""
    G = sum(m.shape[0] for m in masks)
    pad = torch.zeros(G, *input_shape, dtype=dtype, device=masks[0].device if masks else None)
    i = 0
    for m in masks:
        pad[i:i + m.shape[0], :m.shape[1], :m.shape[2]] = m.to(dtype)
        i += m.shape[0]
    if G == 0:
        return pad.new_zeros(0, *size)
    return F.interpolate(pad[:, None], size=tuple(size), mode="bilinear", align_corners=False)[:, 0]


def match_cost(logits, masks, tmasks, sizes, labels, alpha, beta):
    """SparseInstMatcher's cost (:333-340) for the per-image blocks only: [N, g_b] = dice(σ(m), t)^α · σ(logit[label])^β"""
    blocks, off = [], 0
    for b, g in enumerate(sizes):
        s = masks[b].flatten(1).sigmoid()
        t = tmasks[off:off + g].flatten(1)
        dice = 2 * (s @ t.T) / ((s * s).sum(-1)[:, None] + (t * t).sum(-1) + 1e-4)
        prob = logits[b].sigmoid()[:, labels[off:off + g].long()]
        blocks.append(dice ** alpha * prob ** beta)
        off += g
    return blocks


def assign(blocks):
    """linear_sum_assignment(maximize=True) per image, as int64 tensors"""
    out = []
    for c in blocks:
        i, j = linear_sum_assignment(c.detach().cpu().numpy(), maximize=True)
        out.append((torch.as_tensor(i, dtype=torch.int64), torch.as_tensor(j, dtype=torch.int64)))
    return out


def sigmoid_focal_loss(x, t, alpha=0.25, gamma=2.0):
    """fvcore's sigmoid_focal_loss, reduction="sum", in the inputs' dtype"""
    p = torch.sigmoid(x)
    ce = F.binary_cross_entropy_with_logits(x, t, reduction="none")
    p_t = p * t + (1 - p) * (1 - t)
    return (alpha * t + (1 - alpha) * (1 - t)) * ce * ((1 - p_t) ** gamma)


def losses(logits, masks, scores, tmasks, sizes, labels, indices, weight_dict, num_instances, items=("labels", "masks")):
    """SparseInstCriterion.forward (:197-231) given the assignment: the weighted loss dict in the reference's key order.  Differentiable w.r.t.
    logits [B, N, K], masks [B, N, H, W] and scores [B, N, 1].  An empty batch gives loss_ce over all-background labels and 0 · sum mask losses."""
    B, N, K = logits.shape
    off = [0]
    for g in sizes:
        off.append(off[-1] + g)
    b_idx = torch.cat([torch.full_like(i, b) for b, (i, _) in enumerate(indices)])
    q_idx = torch.cat([i for i, _ in indices])
    t_idx = torch.cat([j + off[b] for b, (_, j) in enumerate(indices)])
    out = {}
    for item in items:
        if item == "labels":
            onehot = torch.zeros_like(logits)
            onehot[b_idx, q_idx, labels[t_idx].long()] = 1
            out["loss_ce"] = sigmoid_focal_loss(logits, onehot).sum() / num_instances
        elif item == "masks":
            if off[-1] == 0:
                out.update(loss_dice=masks.sum() * 0.0, loss_mask=masks.sum() * 0.0, loss_objectness=scores.sum() * 0.0)
                continue
            src = masks[b_idx, q_idx].flatten(1)
            tgt = tmasks[t_idx].flatten(1)
            with torch.no_grad():
                bp, bt = (src.sigmoid() >= 0.4).to(src.dtype), (tgt > 0.5).to(src.dtype)
                inter = (bp * bt).sum(-1)
                iou = inter / (bt.sum(-1) + bp.sum(-1) - inter + 1e-6)
            s = src.sigmoid()
            dice = 1 - 2 * (s * tgt).sum(1) / ((s * s).sum(-1) + (tgt * tgt).sum(-1) + 1e-4)
            out["loss_objectness"] = F.binary_cross_entropy_with_logits(scores[b_idx, q_idx].flatten(), iou)
            out["loss_dice"] = dice.sum() / num_instances
            out["loss_mask"] = F.binary_cross_entropy_with_logits(src, tgt)
    return {k: v * weight_dict[k] for k, v in out.items()}


def criterion(logits, masks, scores, mask_list, labels, input_shape, alpha, beta, weight_dict, items=("labels", "masks"), indices=None):
    """matcher + losses; mask_list: per-image [g, h, w] ground-truth masks.  Returns (loss dict, indices, cost blocks)."""
    sizes = [m.shape[0] for m in mask_list]
    tm = target_masks(mask_list, input_shape, masks.shape[-2:], masks.dtype)
    blocks = match_cost(logits.detach(), masks.detach(), tm, sizes, labels, alpha, beta)
    if indices is None:
        indices = assign(blocks)
    num_instances = float(max(sum(sizes), 1))
    return losses(logits, masks, scores, tm, sizes, labels, indices, weight_dict, num_instances, items), indices, blocks


def loss_gradients(logits, masks, scores, loss_dict, coef):
    """d (Σ coef[k] · loss[k]) / d (logits, masks, scores) through autograd; coef maps loss keys to floats"""
    total = sum(coef[k] * v for k, v in loss_dict.items())
    return torch.autograd.grad(total, (logits, masks, scores), allow_unused=True)


def assignment_cost(block, ij):
    """total cost of an assignment (i, j) on one [N, g] block"""
    i, j = ij
    return float(block[i.long(), j.long()].double().sum()) if len(i) else 0.0
