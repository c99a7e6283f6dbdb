"""SparseInst's SparseInstMatcher and SparseInstCriterion on the sm_90a kernels (csrc/sparseinst_criterion.cu).

Reference: yolov7/modeling/loss/sparseinst_loss.py -- `SparseInstCriterion` :49-231, `SparseInstMatcher` :297-354 and the two builders :357-365.
Same constructors (`cfg.MODEL.SPARSE_INST.{LOSS,MATCHER}.*` and `DECODER.NUM_CLASSES`), attributes and return values.  One call:
  1. the targets are packed (labels, per-image offsets, the uint8 masks in one buffer with an (offset, h, w) table);
  2. one kernel resizes every ground-truth mask to the prediction size (the zero padding to `input_shape` is never materialised) and sums Σt²;
     the matcher and the losses share the result;
  3. one kernel computes the matching cost of the per-image blocks only, with a status word that validates the targets;
  4. one pinned device-to-host copy and one event synchronisation bring it to the host, where `scipy.optimize.linear_sum_assignment(maximize=True)`
     solves each image as the reference does;
  5. the match table returns to the device with one non-blocking copy, and one autograd node runs the loss kernels forward and the gradient
     kernel backward.
Defined where the reference is not (DESIGN.md §7): an image with more targets than queries raises `Yb200Error` before any kernel runs; a batch
without any instance gives loss_ce over all-background labels with num_instances = 1 and zero mask losses.  There is no CPU implementation.
"""
import numpy as np
import torch
import torch.nn as nn
from scipy.optimize import linear_sum_assignment

from . import capi
from .detr_criterion import num_per_rank

STATUS_BAD_LABEL, STATUS_TOO_MANY = 1, 2  # bits of the status word written by yb200_sparseinst_match_cost
LOSS_KEYS = ("loss_ce", "loss_objectness", "loss_dice", "loss_mask")  # the order of yb200_sparseinst_set_loss's outputs


def _to_device(arr, device):
    """a host array to the device through pinned memory, without a synchronisation"""
    return torch.from_numpy(np.ascontiguousarray(arr)).pin_memory().to(device, non_blocking=True)


def _predictions(outputs, who):
    """(pred_logits [B, N, K], pred_masks [B, N, H, W], pred_scores [B, N, 1]) as given, after checking devices and shapes"""
    logits, masks, scores = outputs["pred_logits"], outputs["pred_masks"], outputs["pred_scores"]
    if not (logits.is_cuda and masks.is_cuda and scores.is_cuda):
        raise capi.Yb200Error(f"{who}: pred_logits / pred_masks / pred_scores must be CUDA tensors (no CPU path)")
    if logits.dim() != 3 or masks.dim() != 4 or masks.shape[:2] != logits.shape[:2] or scores.numel() != logits.shape[0] * logits.shape[1]:
        raise capi.Yb200Error(f"{who}: pred_logits {tuple(logits.shape)}, pred_masks {tuple(masks.shape)} and pred_scores {tuple(scores.shape)} "
                              "do not match")
    return logits, masks, scores


class _Targets:
    """the batch's targets on the device: labels int32 [G], offsets int32 [B + 1], the masks resized to the prediction size fp32 [G, H, W] and
    their Σt² [G]; sizes per image (host)"""

    def __init__(self, targets, input_shape, masks_shape, device, who):
        B, N, H, W = masks_shape
        in_h, in_w = (int(v) for v in input_shape)
        if len(targets) != B:
            raise capi.Yb200Error(f"{who}: {len(targets)} targets for a batch of {B} images")
        self.sizes, table, bufs, off = [], [], [], 0
        for b, t in enumerate(targets):
            labels, m = t["labels"], t["masks"].tensor
            g = int(labels.shape[0])
            if not (labels.is_cuda and m.is_cuda):
                raise capi.Yb200Error(f"{who}: the labels and masks of image {b} must be CUDA tensors (no CPU path)")
            if m.dim() != 3 or m.shape[0] != g or m.dtype not in (torch.bool, torch.uint8):
                raise capi.Yb200Error(f"{who}: image {b} has {g} labels and masks {tuple(m.shape)} of {m.dtype} (expected [{g}, h, w] bool / uint8)")
            h, w = int(m.shape[1]), int(m.shape[2])
            if g and (h > in_h or w > in_w):
                raise capi.Yb200Error(f"{who}: the {h}x{w} masks of image {b} are larger than input_shape {in_h}x{in_w}")
            if g > N:
                raise capi.Yb200Error(f"{who}: image {b} has {g} targets for {N} queries (the reference's mix_tgt_idx needs every target matched)")
            self.sizes.append(g)
            table += [(off + j * h * w, h, w) for j in range(g)]
            if g:
                bufs.append((m.view(torch.uint8) if m.dtype == torch.bool else m).reshape(-1))
            off += g * h * w
        self.offsets_host = np.concatenate([[0], np.cumsum(self.sizes)]).astype(np.int64)
        self.total = G = int(self.offsets_host[-1])
        self.offsets = _to_device(self.offsets_host.astype(np.int32), device)
        if G:
            self.labels = torch.cat([t["labels"] for t in targets]).to(device=device, dtype=torch.int32).contiguous()
            self.masks = torch.empty(G, H, W, device=device)
            self.tsq = torch.empty(G, device=device)
            capi.sparseinst_target_masks(torch.cat(bufs), _to_device(np.array(table, dtype=np.int64), device), G, (in_h, in_w), (H, W), self.masks,
                                         self.tsq)
        else:  # the kernels take non-null target pointers; nothing reads them
            self.labels = torch.zeros(1, dtype=torch.int32, device=device)
            self.masks = torch.zeros(1, device=device)
            self.tsq = torch.zeros(1, device=device)


class SparseInstMatcher(nn.Module):
    """sparseinst_loss.py:297-354: forward(outputs, targets, input_shape) -> [(int64 index_i, int64 index_j)] per image"""

    def __init__(self, cfg):
        super().__init__()
        self.alpha = cfg.MODEL.SPARSE_INST.MATCHER.ALPHA
        self.beta = cfg.MODEL.SPARSE_INST.MATCHER.BETA

    def forward(self, outputs, targets, input_shape):
        logits, masks, _ = _predictions(outputs, "SparseInstMatcher")
        logits, masks = logits.detach().float().contiguous(), masks.detach().float().contiguous()
        indices, _ = self.match(logits, masks, _Targets(targets, input_shape, masks.shape, logits.device, "SparseInstMatcher"))
        return indices

    @torch.no_grad()
    def match(self, logits, masks, tg):
        """fp32 contiguous logits [B, N, K] and masks [B, N, H, W] against packed targets, in one cost launch and one host synchronisation.
        Returns (indices[b] = (int64 i, int64 j), match table int32 [B, N] in pinned host memory: target index within the image or -1)."""
        B, N, K = logits.shape
        G = tg.total
        cost = torch.empty(N * G + 1, device=logits.device)
        capi.sparseinst_match_cost(logits, masks, tg.labels, tg.offsets, tg.masks, tg.tsq, G, self.alpha, self.beta, cost)
        host = torch.empty(cost.shape, dtype=torch.float32, pin_memory=True)
        host.copy_(cost, non_blocking=True)
        done = torch.cuda.Event()
        done.record()
        done.synchronize()
        status = int(host[-1:].view(torch.int32)[0])
        if status & STATUS_BAD_LABEL:
            raise capi.Yb200Error(f"SparseInstMatcher: a target label lies outside [0, {K - 1}]")
        if status & STATUS_TOO_MANY:
            raise capi.Yb200Error(f"SparseInstMatcher: an image has more targets than its {N} queries")
        c = host.numpy()
        match = torch.full((B, N), -1, dtype=torch.int32, pin_memory=True)
        mt = match.numpy()
        indices = []
        for b, gb in enumerate(tg.sizes):
            start = N * int(tg.offsets_host[b])
            if gb:
                i, j = linear_sum_assignment(c[start:start + N * gb].reshape(N, gb), maximize=True)
                mt[b, i] = j
            else:
                i, j = np.zeros(0, np.int64), np.zeros(0, np.int64)
            indices.append((torch.as_tensor(i, dtype=torch.int64), torch.as_tensor(j, dtype=torch.int64)))
        return indices, match


class _SetLossFn(torch.autograd.Function):
    """the four weighted losses and their gradients w.r.t. pred_logits / pred_masks / pred_scores (yb200_sparseinst_set_loss / _bwd).
    args: (fp32 contiguous logits, masks, scores [B, N], device match table, targets, number of matched pairs, the four weights,
    num_instances), then the three tensors the caller passed (the gradients are routed back to them)"""

    @staticmethod
    def forward(ctx, args, logits_in, masks_in, scores_in):
        logits, masks, scores, match, tg, num_pairs, weights, num_inst = args
        B, N, _ = logits.shape
        out = torch.empty(4, device=logits.device)
        save = torch.empty(B, N, 8, device=logits.device)
        capi.sparseinst_set_loss(logits, masks, scores, match, tg.labels, tg.offsets, tg.masks, tg.tsq, num_pairs, weights, num_inst, save, out)
        ctx.args, ctx.save = args, save
        ctx.shapes = (masks_in.shape, scores_in.shape)
        return out

    @staticmethod
    def backward(ctx, g_out):
        logits, masks, scores, match, tg, num_pairs, weights, num_inst = ctx.args
        dlogits, dmasks, dscores = torch.empty_like(logits), torch.empty_like(masks), torch.empty_like(scores)
        capi.sparseinst_set_loss_bwd(logits, masks, scores, match, tg.labels, tg.offsets, tg.masks, tg.tsq, ctx.save, num_pairs, weights, num_inst,
                                     g_out.float().contiguous(), dlogits, dmasks, dscores)
        return None, dlogits, dmasks.view(ctx.shapes[0]), dscores.view(ctx.shapes[1])


class SparseInstCriterion(nn.Module):
    """sparseinst_loss.py:49-231.  forward(outputs, targets, input_shape) returns the reference's dict: loss_ce for "labels", then
    loss_objectness, loss_dice, loss_mask for "masks" (in the order of LOSS.ITEMS), each multiplied by its weight_dict entry."""

    def __init__(self, cfg, matcher):
        super().__init__()
        self.matcher = matcher
        self.losses = cfg.MODEL.SPARSE_INST.LOSS.ITEMS
        self.weight_dict = self.get_weight_dict(cfg)
        self.num_classes = cfg.MODEL.SPARSE_INST.DECODER.NUM_CLASSES

    def get_weight_dict(self, cfg):
        loss = cfg.MODEL.SPARSE_INST.LOSS
        return dict(zip(("loss_ce", "loss_mask", "loss_dice", "loss_objectness"),
                        (loss.CLASS_WEIGHT, loss.MASK_PIXEL_WEIGHT, loss.MASK_DICE_WEIGHT, loss.OBJECTNESS_WEIGHT)))

    def forward(self, outputs, targets, input_shape):
        for item in self.losses:
            if item not in ("labels", "masks", "loss_objectness"):
                raise capi.Yb200Error(f"SparseInstCriterion: unknown loss {item!r}")
        if not isinstance(self.matcher, SparseInstMatcher):
            raise capi.Yb200Error(f"SparseInstCriterion: the matcher must be this package's SparseInstMatcher, not {type(self.matcher).__name__}")
        logits_in, masks_in, scores_in = _predictions(outputs, "SparseInstCriterion")
        if logits_in.shape[-1] != self.num_classes:
            raise capi.Yb200Error(f"SparseInstCriterion: {logits_in.shape[-1]} logits per query for num_classes={self.num_classes}")
        device = logits_in.device
        with torch.no_grad():
            logits = logits_in.detach().float().contiguous()
            masks = masks_in.detach().float().contiguous()
            scores = scores_in.detach().float().reshape(logits.shape[:2]).contiguous()
        tg = _Targets(targets, input_shape, masks.shape, device, "SparseInstCriterion")
        indices, match_host = self.matcher.match(logits, masks, tg)
        match = match_host.to(device, non_blocking=True)
        num_inst = num_per_rank(tg.total, device)
        num_pairs = sum(len(i) for i, _ in indices)
        weights = tuple(float(self.weight_dict[k]) for k in LOSS_KEYS)
        out = _SetLossFn.apply((logits, masks, scores, match, tg, num_pairs, weights, num_inst), logits_in, masks_in, scores_in)
        losses = {}
        for item in self.losses:
            if item == "labels":
                losses["loss_ce"] = out[0]
            elif item == "masks" and tg.total:
                losses.update(loss_objectness=out[1], loss_dice=out[2], loss_mask=out[3])
            elif item == "masks":  # the reference's key order for a batch without instances (:140-146)
                losses.update(loss_dice=out[2], loss_mask=out[3], loss_objectness=out[1])
        return losses


def build_sparse_inst_matcher(cfg):
    name = cfg.MODEL.SPARSE_INST.MATCHER.NAME
    if name != "SparseInstMatcher":
        raise capi.Yb200Error(f"build_sparse_inst_matcher: {name!r} is not built (only SparseInstMatcher)")
    return SparseInstMatcher(cfg)


def build_sparse_inst_criterion(cfg):
    matcher = build_sparse_inst_matcher(cfg)
    name = cfg.MODEL.SPARSE_INST.LOSS.NAME
    if name != "SparseInstCriterion":
        raise capi.Yb200Error(f"build_sparse_inst_criterion: {name!r} is not built (only SparseInstCriterion)")
    return SparseInstCriterion(cfg, matcher)


def _register():
    try:
        from detectron2.utils.registry import Registry  # noqa: F401  # pragma: no cover
    except Exception:  # noqa: BLE001
        return
    try:  # pragma: no cover
        from yolov7.modeling.loss.sparseinst_loss import SPARSE_INST_CRITERION_REGISTRY, SPARSE_INST_MATCHER_REGISTRY
        SPARSE_INST_MATCHER_REGISTRY._obj_map["SparseInstMatcher"] = SparseInstMatcher
        SPARSE_INST_CRITERION_REGISTRY._obj_map["SparseInstCriterion"] = SparseInstCriterion
    except Exception:  # noqa: BLE001
        pass


_register()
