"""TEST INFRASTRUCTURE -- plain-torch restatement of DETR's matching cost, SetCriterion and the DETR tail (class_embed, bbox_embed, input_proj).

References: yolov7/utils/detr_utils.py:12-91 (HungarianMatcher), yolov7/modeling/meta_arch/detr.py:282-294 (MLP), :406-472 (DETR), :475-647
(SetCriterion), yolov7/utils/boxes.py:28-31, 85-122 (box_cxcywh_to_xyxy, box_iou, generalized_box_iou).  Pinned by tests/golden/detr_criterion.npz,
produced by oracle/gen_golden_detr_criterion.py from the unmodified reference classes; tests/test_detr_criterion_oracle_golden.py re-checks this
file against those vectors on every CPU run.  Every function follows the dtype of its inputs (fp32 or fp64).  Only tests/ and tools/ may import it.
"""
import torch
import torch.nn.functional as F
from scipy.optimize import linear_sum_assignment

def box_cxcywh_to_xyxy(x):
    x_c, y_c, w, h = x.unbind(-1)
    return torch.stack([(x_c - 0.5 * w), (y_c - 0.5 * h), (x_c + 0.5 * w), (y_c + 0.5 * h)], dim=-1)


def generalized_box_iou(boxes1, boxes2):
    """[N, M] GIoU of xyxy boxes (without the reference's degenerate-box assert)"""
    area1 = (boxes1[:, 2] - boxes1[:, 0]) * (boxes1[:, 3] - boxes1[:, 1])
    area2 = (boxes2[:, 2] - boxes2[:, 0]) * (boxes2[:, 3] - boxes2[:, 1])
    lt = torch.max(boxes1[:, None, :2], boxes2[:, :2])
    rb = torch.min(boxes1[:, None, 2:], boxes2[:, 2:])
    wh = (rb - lt).clamp(min=0)
    inter = wh[:, :, 0] * wh[:, :, 1]
    union = area1[:, None] + area2 - inter
    iou = inter / union
    lt = torch.min(boxes1[:, None, :2], boxes2[:, :2])
    rb = torch.max(boxes1[:, None, 2:], boxes2[:, 2:])
    wh = (rb - lt).clamp(min=0)
    area = wh[:, :, 0] * wh[:, :, 1]
    return iou - (area - union) / area


def match_cost(logits, boxes, targets, cost_class=1.0, cost_bbox=1.0, cost_giou=1.0):
    """detr_utils.py:65-86 for one layer: logits [B, Q, K1], boxes [B, Q, 4] -> the per-image blocks [Q, G_b] of the cost matrix"""
    bs, nq = logits.shape[:2]
    prob = logits.flatten(0, 1).softmax(-1)
    out_bbox = boxes.flatten(0, 1)
    tgt_ids = torch.cat([t["labels"] for t in targets]).long()
    tgt_bbox = torch.cat([t["boxes"] for t in targets]).to(out_bbox.dtype)
    c = cost_bbox * torch.cdist(out_bbox, tgt_bbox, p=1) + cost_class * -prob[:, tgt_ids] + \
        cost_giou * -generalized_box_iou(box_cxcywh_to_xyxy(out_bbox), box_cxcywh_to_xyxy(tgt_bbox))
    c = c.view(bs, nq, -1)
    sizes = [len(t["boxes"]) for t in targets]
    return [blk[b] for b, blk in enumerate(c.split(sizes, -1))]


def assign(blocks):
    """scipy's linear_sum_assignment per image, as the reference returns it"""
    out = []
    for c in blocks:
        i, j = linear_sum_assignment(c.detach().cpu().numpy())
        out.append((torch.as_tensor(i, dtype=torch.int64), torch.as_tensor(j, dtype=torch.int64)))
    return out


def set_losses(logits, boxes, targets, indices, num_classes, eos_coef, num_boxes, losses=("labels", "boxes", "cardinality"), log=True):
    """loss_labels / loss_boxes / loss_cardinality (detr.py:495-570) of one layer, differentiable w.r.t. logits and boxes"""
    out = {}
    batch_idx = torch.cat([torch.full_like(src, i) for i, (src, _) in enumerate(indices)]).to(logits.device)
    src_idx = torch.cat([src for (src, _) in indices]).to(logits.device)
    for loss in losses:
        if loss == "labels":
            empty_weight = torch.ones(num_classes + 1, dtype=logits.dtype, device=logits.device)
            empty_weight[-1] = eos_coef
            tco = torch.cat([t["labels"][j.to(t["labels"].device)] for t, (_, j) in zip(targets, indices)]).long().to(logits.device)
            tc = torch.full(logits.shape[:2], num_classes, dtype=torch.int64, device=logits.device)
            tc[batch_idx, src_idx] = tco
            out["loss_ce"] = F.cross_entropy(logits.transpose(1, 2), tc, empty_weight)
            if log:
                if tco.numel() == 0:
                    acc = torch.zeros([], dtype=logits.dtype, device=logits.device)
                else:
                    acc = (logits.detach()[batch_idx, src_idx].argmax(-1) == tco).to(logits.dtype).sum() * (100.0 / tco.numel())
                out["class_error"] = 100 - acc
        elif loss == "boxes":
            src = boxes[batch_idx, src_idx]
            tgt = torch.cat([t["boxes"][j.to(t["boxes"].device)] for t, (_, j) in zip(targets, indices)], dim=0).to(boxes)
            out["loss_bbox"] = F.l1_loss(src, tgt, reduction="none").sum() / num_boxes
            out["loss_giou"] = (1 - torch.diag(generalized_box_iou(box_cxcywh_to_xyxy(src), box_cxcywh_to_xyxy(tgt)))).sum() / num_boxes
        elif loss == "cardinality":
            with torch.no_grad():
                lengths = torch.as_tensor([len(t["labels"]) for t in targets], dtype=logits.dtype, device=logits.device)
                card = (logits.argmax(-1) != logits.shape[-1] - 1).sum(1)
                out["cardinality_error"] = F.l1_loss(card.to(logits.dtype), lengths)
    return out


def criterion(layers, targets, num_classes, eos_coef, costs=(1.0, 1.0, 1.0), losses=("labels", "boxes", "cardinality"), indices=None):
    """SetCriterion.forward (detr.py:608-647) for `layers` = [(logits [B, Q, K1], boxes [B, Q, 4])] with the last layer the model's output and
    the others its aux_outputs in order.  costs = (cost_class, cost_bbox, cost_giou).  indices (per layer, per image) replace the matcher when
    given.  Returns (loss dict in the reference's key order, indices per layer)."""
    if indices is None:
        indices = [assign(match_cost(lg.detach(), bx.detach(), targets, *costs)) for lg, bx in layers]
    num_boxes = float(max(sum(len(t["labels"]) for t in targets), 1))
    last = len(layers) - 1
    out = dict(set_losses(*layers[last], targets, indices[last], num_classes, eos_coef, num_boxes, losses))
    for i in range(last):
        d = set_losses(*layers[i], targets, indices[i], num_classes, eos_coef, num_boxes, losses, log=False)
        out.update({k + f"_{i}": v for k, v in d.items()})
    return out, indices


def assignment_cost(block, ij):
    """total cost of an assignment (i, j) on one [Q, G] block"""
    i, j = ij
    return float(block[i.long(), j.long()].double().sum()) if len(i) else 0.0


# ---- the DETR tail: input_proj (1x1 conv), class_embed, bbox_embed (MLP), sigmoid ------------------------------------------------------------------
def input_proj(src, sd, storage=None):
    """nn.Conv2d(num_channels, hidden_dim, 1) of detr.py:426"""
    q = storage or (lambda t: t)
    return F.conv2d(q(src), q(sd["input_proj.weight"]), sd["input_proj.bias"])


def heads(hs, sd, storage=None):
    """class_embed and sigmoid(bbox_embed) over hs [L, B, Q, C] (detr.py:464-466); storage rounds what the kernels store in 16 bits"""
    q = storage or (lambda t: t)
    logits = F.linear(q(hs), q(sd["class_embed.weight"]), sd["class_embed.bias"])
    x = q(hs)
    for i in range(3):
        x = F.linear(x, q(sd[f"bbox_embed.layers.{i}.weight"]), sd[f"bbox_embed.layers.{i}.bias"])
        x = q(F.relu(x)) if i < 2 else x
    return logits, torch.sigmoid(x)


def bf16(t):
    return t.to(torch.bfloat16).to(t.dtype)
