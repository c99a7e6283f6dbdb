"""DETR's HungarianMatcher and SetCriterion on the sm_90a kernels (csrc/detr_criterion.cu).

Reference: yolov7/utils/detr_utils.py:12-91 (`HungarianMatcher`) and yolov7/modeling/meta_arch/detr.py:475-647 (`SetCriterion`).  Same
constructor arguments, attributes, buffers and return values.  The device computes the matching cost of every decoder layer in one launch (only
the per-image blocks the assignment reads) together with a status word that validates the targets; one pinned device-to-host copy and one
synchronisation bring all of it to the host, where `scipy.optimize.linear_sum_assignment` solves each (layer, image) problem exactly as the
reference does.  The match table returns to the device with one non-blocking copy, and one autograd node computes the losses of every layer
and their gradients (csrc/detr_criterion.cu).  There is no CPU implementation.
"""
import numpy as np
import torch
import torch.distributed as dist
import torch.nn as nn
from scipy.optimize import linear_sum_assignment

from . import capi

STATUS_BAD_LABEL, STATUS_BAD_BOX = 1, 2  # bits of the status word written by yb200_detr_match_cost


def num_per_rank(total, device):
    """the target count normalising the losses, averaged over the ranks and clamped to >= 1 (detr.py:620-624, sparseinst_loss.py:204-212);
    without a process group it is known on the host and costs no synchronisation"""
    if dist.is_available() and dist.is_initialized():
        nb = torch.as_tensor([total], dtype=torch.float, device=device)
        dist.all_reduce(nb)
        return torch.clamp(nb / dist.get_world_size(), min=1).item()
    return float(max(total, 1))


class _Targets:
    """the batch's targets packed for the kernels: labels int32 [G], boxes fp32 [G, 4], offsets int32 [B + 1] (device), sizes (host)"""

    def __init__(self, targets, device):
        self.sizes = [int(t["labels"].shape[0]) for t in targets]
        self.offsets_host = np.concatenate([[0], np.cumsum(self.sizes)]).astype(np.int64)
        self.total = int(self.offsets_host[-1])
        if self.total:
            self.labels = torch.cat([t["labels"] for t in targets]).to(device=device, dtype=torch.int32).contiguous()
            self.boxes = torch.cat([t["boxes"] for t in targets]).to(device=device, dtype=torch.float32).contiguous()
        else:  # the kernels take non-null target pointers; nothing reads them
            self.labels = torch.zeros(1, dtype=torch.int32, device=device)
            self.boxes = torch.zeros(1, 4, device=device)
        off = torch.from_numpy(self.offsets_host.astype(np.int32)).pin_memory()
        self.offsets = off.to(device, non_blocking=True)


def _check_outputs(logits, boxes):
    if not (logits.is_cuda and boxes.is_cuda):
        raise capi.Yb200Error("DETR criterion: pred_logits / pred_boxes must be CUDA tensors (no CPU path)")
    if logits.dim() != 4 or boxes.shape != logits.shape[:3] + (4,):
        raise capi.Yb200Error(f"DETR criterion: pred_logits {tuple(logits.shape[1:])} and pred_boxes {tuple(boxes.shape[1:])} do not match")


class HungarianMatcher(nn.Module):
    """detr_utils.py:12-91: forward(outputs, targets) -> [(int64 index_i, int64 index_j)] per image"""

    def __init__(self, cost_class: float = 1, cost_bbox: float = 1, cost_giou: float = 1):
        super().__init__()
        self.cost_class = cost_class
        self.cost_bbox = cost_bbox
        self.cost_giou = cost_giou
        assert cost_class != 0 or cost_bbox != 0 or cost_giou != 0, "all costs cant be 0"

    @torch.no_grad()
    def forward(self, outputs, targets):
        logits, boxes = outputs["pred_logits"].unsqueeze(0), outputs["pred_boxes"].unsqueeze(0)
        indices, _ = self.match_layers(logits, boxes, _Targets(targets, logits.device))
        return indices[0]

    @torch.no_grad()
    def match_layers(self, logits, boxes, tg):
        """all L layers of [L, B, Q, K1] logits and [L, B, Q, 4] boxes in one cost launch and one host synchronisation.
        Returns (indices[l][b] = (int64 i, int64 j), match table int32 [L, B, Q] in pinned host memory: target index within the image or -1)."""
        _check_outputs(logits, boxes)
        L, B, Q, K1 = logits.shape
        if len(tg.sizes) != B:
            raise capi.Yb200Error(f"HungarianMatcher: {len(tg.sizes)} targets for a batch of {B} images")
        logits = logits.detach().float().contiguous()
        boxes = boxes.detach().float().contiguous()
        G = tg.total
        cost = torch.empty(L * Q * G + 1, device=logits.device)
        capi.detr_match_cost(logits, boxes, tg.labels, tg.boxes, tg.offsets, G, self.cost_class, self.cost_bbox, self.cost_giou, cost)
        host = torch.empty(cost.shape, dtype=torch.float32, pin_memory=True)
        host.copy_(cost, non_blocking=True)
        done = torch.cuda.Event()
        done.record()
        done.synchronize()
        status = int(host[-1:].view(torch.int32)[0])
        if status & STATUS_BAD_LABEL:
            raise capi.Yb200Error(f"HungarianMatcher: a target label lies outside [0, {K1 - 1}]")
        if status & STATUS_BAD_BOX:
            raise capi.Yb200Error("HungarianMatcher: a target box has a negative width or height (generalized_box_iou needs x1 >= x0, y1 >= y0)")
        c = host.numpy()
        match = torch.full((L, B, Q), -1, dtype=torch.int32, pin_memory=True)
        mt = match.numpy()
        indices = []
        for l in range(L):
            per_image = []
            for b, gb in enumerate(tg.sizes):
                start = l * Q * G + Q * int(tg.offsets_host[b])
                i, j = linear_sum_assignment(c[start:start + Q * gb].reshape(Q, gb))
                mt[l, b, i] = j
                per_image.append((torch.as_tensor(i, dtype=torch.int64), torch.as_tensor(j, dtype=torch.int64)))
            indices.append(per_image)
        return indices, match


class _SetLossFn(torch.autograd.Function):
    """the losses of every layer and their gradients w.r.t. each layer's pred_logits / pred_boxes (yb200_detr_set_loss / _bwd).
    args: (stacked logits [L, B, Q, K1], stacked boxes, device match table, targets, eos_coef, num_boxes), then the L logits and L boxes
    tensors the caller passed (the gradients are routed back to them)"""

    @staticmethod
    def forward(ctx, args, *inputs):
        logits, boxes, match, tg, eos_coef, num_boxes = args
        out = torch.empty(logits.shape[0], 5, device=logits.device)
        capi.detr_set_loss(logits, boxes, match, tg.labels, tg.boxes, tg.offsets, eos_coef, num_boxes, out)
        ctx.args = args
        return out

    @staticmethod
    def backward(ctx, g_out):
        logits, boxes, match, tg, eos_coef, num_boxes = ctx.args
        L = logits.shape[0]
        dlogits, dboxes = torch.empty_like(logits), torch.empty_like(boxes)
        capi.detr_set_loss_bwd(logits, boxes, match, tg.labels, tg.boxes, tg.offsets, eos_coef, num_boxes, g_out[:, :3].float().contiguous(), dlogits,
                               dboxes)
        return (None,) + tuple(dlogits[l] for l in range(L)) + tuple(dboxes[l] for l in range(L))


class SetCriterion(nn.Module):
    """detr.py:475-647 for the "labels", "boxes" and "cardinality" losses.  forward(outputs, targets) returns the reference's dict:
    loss_ce, class_error, loss_bbox, loss_giou, cardinality_error (in the order of `losses`), then the same keys suffixed _i for every
    auxiliary layer i (without class_error).  The values are unweighted; `weight_dict` is kept for the caller, as in the reference."""

    def __init__(self, num_classes, matcher, weight_dict, eos_coef, losses):
        super().__init__()
        self.num_classes = num_classes
        self.matcher = matcher
        self.weight_dict = weight_dict
        self.eos_coef = eos_coef
        self.losses = losses
        empty_weight = torch.ones(self.num_classes + 1)
        empty_weight[-1] = self.eos_coef
        self.register_buffer("empty_weight", empty_weight)

    def forward(self, outputs, targets):
        for loss in self.losses:
            if loss == "masks":
                raise capi.Yb200Error("SetCriterion: the mask losses are not implemented")
            if loss not in ("labels", "boxes", "cardinality"):
                raise capi.Yb200Error(f"SetCriterion: unknown loss {loss!r}")
        layers = list(outputs.get("aux_outputs", [])) + [outputs]
        logits_in = [o["pred_logits"] for o in layers]
        boxes_in = [o["pred_boxes"] for o in layers]
        for lg, bx in zip(logits_in, boxes_in):
            _check_outputs(lg.unsqueeze(0), bx.unsqueeze(0))
            if lg.shape != logits_in[-1].shape:
                raise capi.Yb200Error("SetCriterion: every decoder layer must have the same [B, Q, K1] logits")
        if logits_in[-1].shape[-1] != self.num_classes + 1:
            raise capi.Yb200Error(f"SetCriterion: {logits_in[-1].shape[-1]} logits per query for num_classes={self.num_classes}")
        device = logits_in[-1].device
        with torch.no_grad():
            logits = torch.stack([t.detach() for t in logits_in]).float().contiguous()
            boxes = torch.stack([t.detach() for t in boxes_in]).float().contiguous()
        tg = _Targets(targets, device)
        _, match_host = self.matcher.match_layers(logits, boxes, tg)
        match = match_host.to(device, non_blocking=True)
        num_boxes = num_per_rank(tg.total, device)
        out = _SetLossFn.apply((logits, boxes, match, tg, float(self.eos_coef), num_boxes), *logits_in, *boxes_in)
        stats = out.detach()
        L = len(layers)
        losses = {}
        for l in [L - 1] + list(range(L - 1)):
            sfx = "" if l == L - 1 else f"_{l}"
            for loss in self.losses:
                if loss == "labels":
                    losses["loss_ce" + sfx] = out[l, 0]
                    if l == L - 1:
                        losses["class_error"] = stats[l, 4]
                elif loss == "boxes":
                    losses["loss_bbox" + sfx] = out[l, 1]
                    losses["loss_giou" + sfx] = out[l, 2]
                else:
                    losses["cardinality_error" + sfx] = stats[l, 3]
        return losses
