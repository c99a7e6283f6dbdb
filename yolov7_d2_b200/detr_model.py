"""DETR meta-architecture on the sm_90a kernels: `@META_ARCH_REGISTRY.register() class Detr(nn.Module)`.

Reference: yolov7/modeling/meta_arch/detr.py -- `Detr` :33-279, `MaskedBackboneTraceFriendly` :340-403; yolov7/modeling/backbone/detr_backbone.py
-- `Joiner` :496-512, `PositionEmbeddingSine` :309-375.  Same constructor (`cfg.MODEL.{DEVICE, PIXEL_MEAN, PIXEL_STD, MASK_ON, BACKBONE.NAME}`,
`cfg.MODEL.YOLO.CONF_THRESHOLD` as `ignore_thresh`, `cfg.MODEL.DETR.*`), attributes, state_dict keys and return values.  The backbone stays the
caller's (detectron2's `build_backbone(cfg)`, or the bundled registry without detectron2); the transformer, heads and criterion are this
package's (detr.py, detr_criterion.py).

  * Input (`preprocess_image` :273-279): one copy per image into one staging buffer, then one `yb200_normalize_pad` launch writes the normalised
    batch zero-padded to the batch maximum (ImageList.from_tensors without size divisibility), bit-identical to the reference's torch arithmetic.
  * Backbone (`Joiner`): the caller's backbone on the padded batch, then one `yb200_detr_mask_pos` launch writes the padding mask and the sine
    position embedding of every level.
  * Training (:167-177): `yb200_detr_pack_targets` normalises every target box of the batch in one launch; the criterion's loss dict is weighted
    by `weight_dict` as in the reference; gradients reach the backbone through input_proj.
  * Eval (`inference` :219-265 with detectron2's `detector_postprocess`): `yb200_detr_infer` scores, thresholds, scales, clips and compacts every
    query of the batch; ONE device-to-host copy of the B counts (and a status word) and one event synchronisation per batch.
There is no CPU path, no DETRsegm (MASK_ON), no pre-norm transformer and no ONNX path: all raise Yb200Error before any kernel runs.
"""
import ctypes
import math

import numpy as np
import torch
import torch.nn as nn

from . import capi
from .batch_input import normalize_pad, pinned_to
from .detr import DETR, Transformer
from .detr_criterion import HungarianMatcher, SetCriterion
from .modeling import BACKBONE_REGISTRY, HAVE_D2, META_ARCH_REGISTRY, Boxes, Instances, ShapeSpec

SIZE_DIVISIBILITY = 0  # ImageList.from_tensors(images) (:278)
STATUS_NONFINITE_BOX = 1  # bit of yb200_detr_infer's status word
MAX_LEVELS = 8  # YB200_DETR_MAX_LEVELS

if HAVE_D2:  # pragma: no cover - detectron2 is not installed in the build container
    from detectron2.modeling import build_backbone
    from detectron2.structures import ImageList
else:
    build_backbone = None

    class ImageList:
        """the part of detectron2's ImageList the backbone wrapper reads: the padded batch `.tensor` and the images' `.image_sizes`"""

        def __init__(self, tensor, image_sizes):
            self.tensor, self.image_sizes = tensor, image_sizes


class NestedTensor:
    """yolov7/utils/misc.py NestedTensor: a level's features and its padding mask"""

    def __init__(self, tensors, mask):
        self.tensors, self.mask = tensors, mask

    def decompose(self):
        return self.tensors, self.mask


class DetrLevel(ctypes.Structure):
    """mirror of `yb200_detr_level` (include/yb200.h)"""

    _fields_ = [("mask", ctypes.c_void_p), ("pos", ctypes.c_void_p), ("h", ctypes.c_int32), ("w", ctypes.c_int32)]


class MaskedBackbone(nn.Module):
    """MaskedBackboneTraceFriendly (:340-403) around the caller's backbone: `feature_strides` and `num_channels` (of the last level) come from
    output_shape() in key order; forward returns the backbone's feature dict.  The masks are written with the positions (Joiner)."""

    def __init__(self, backbone):
        super().__init__()
        self.backbone = backbone
        shape = backbone.output_shape()
        self.feature_strides = [shape[f].stride for f in shape.keys()]
        self.num_channels = shape[list(shape.keys())[-1]].channels
        self.onnx_export = False

    def forward(self, images):
        return self.backbone(images.tensor)


class PositionEmbeddingSine(nn.Module):
    """detr_backbone.py:309-375 with normalize=True (the only form DETR builds): forward(feature shapes, strides, image sizes) -> (masks bool
    [B, h, w], positions fp32 [B, 2 num_pos_feats, h, w]) for every level in one `yb200_detr_mask_pos` launch.  Parameter-free.  dim_t is
    computed once per device with the reference's torch expression, so every sin / cos argument has the reference's bits."""

    def __init__(self, num_pos_feats=64, temperature=10000, normalize=False, scale=None):
        super().__init__()
        if not normalize or scale is not None:
            raise capi.Yb200Error("PositionEmbeddingSine: only normalize=True with the default scale 2 pi is built")
        if num_pos_feats <= 0 or num_pos_feats % 2:
            raise capi.Yb200Error(f"PositionEmbeddingSine: num_pos_feats {num_pos_feats} (positive and even)")
        self.num_pos_feats, self.temperature, self.normalize, self.scale = num_pos_feats, temperature, normalize, 2 * math.pi
        self._dim_t = {}
        self.L = capi.lib()

    def dim_t(self, device):
        if device not in self._dim_t:
            d = torch.arange(self.num_pos_feats, dtype=torch.float32, device=device)
            self._dim_t[device] = self.temperature ** (2 * (d // 2) / self.num_pos_feats)
        return self._dim_t[device]

    def forward(self, feature_shapes, strides, image_sizes, device):
        if len(feature_shapes) != len(strides) or not 0 < len(strides) <= MAX_LEVELS:
            raise capi.Yb200Error(f"Joiner: {len(feature_shapes)} feature levels for {len(strides)} strides (1 to {MAX_LEVELS})")
        B = len(image_sizes)
        valid = np.zeros((len(strides), B, 2), dtype=np.int32)
        masks, pos = [], []
        table = (DetrLevel * len(strides))()
        for l, (shape, s) in enumerate(zip(feature_shapes, strides)):
            n, _, h, w = shape
            if n != B:
                raise capi.Yb200Error(f"Joiner: level {l} has {n} images for a batch of {B}")
            for b, (ih, iw) in enumerate(image_sizes):  # :396-401, in float64
                valid[l, b] = (min(int(np.ceil(float(ih) / s)), h), min(int(np.ceil(float(iw) / s)), w))
            masks.append(torch.empty(B, h, w, dtype=torch.bool, device=device))
            pos.append(torch.empty(B, 2 * self.num_pos_feats, h, w, device=device))
            table[l] = DetrLevel(masks[-1].data_ptr(), pos[-1].data_ptr(), h, w)
        valid_d = pinned_to(valid, device)
        capi.check(self.L.yb200_detr_mask_pos(table, len(strides), B, capi.ptr(valid_d), capi.ptr(self.dim_t(device)), self.num_pos_feats,
                                              capi.stream_ptr()), "detr_mask_pos")
        return masks, pos


class Joiner(nn.Sequential):
    """detr_backbone.py:496-512: [0] the masked backbone, [1] the position embedding; forward(ImageList) -> (per level NestedTensor(features,
    mask), per level positions in the features' dtype)"""

    def __init__(self, backbone, position_embedding):
        super().__init__(backbone, position_embedding)

    def forward(self, images):
        feats = list(self[0](images).values())
        masks, pos = self[1]([f.shape for f in feats], self[0].feature_strides, images.image_sizes, feats[0].device)
        return [NestedTensor(f, m) for f, m in zip(feats, masks)], [p.to(f.dtype) for f, p in zip(feats, pos)]


def _gather(ts, device, dtype):
    """one device tensor from per-image tensors: host tensors are concatenated on the host and copied once"""
    if all(t.device.type == "cpu" for t in ts):
        return torch.cat(ts).to(dtype).pin_memory().to(device, non_blocking=True)
    return torch.cat([t.to(device, dtype) for t in ts])


@META_ARCH_REGISTRY.register()
class Detr(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        self.device = torch.device(cfg.MODEL.DEVICE)
        if self.device.type != "cuda":
            raise capi.Yb200Error(f"Detr: MODEL.DEVICE {cfg.MODEL.DEVICE!r} (the kernels run on CUDA only; there is no CPU path)")
        self.ignore_thresh = cfg.MODEL.YOLO.CONF_THRESHOLD
        self.num_classes = cfg.MODEL.DETR.NUM_CLASSES
        self.mask_on = cfg.MODEL.MASK_ON
        if self.mask_on:
            raise capi.Yb200Error("Detr: MODEL.MASK_ON (DETRsegm and the mask losses) is not built")
        d = cfg.MODEL.DETR
        if d.PRE_NORM:
            raise capi.Yb200Error("Detr: MODEL.DETR.PRE_NORM (normalize_before=True) is not built")
        hidden_dim = d.HIDDEN_DIM
        if HAVE_D2:  # pragma: no cover
            bb = build_backbone(cfg)
        else:
            bb = BACKBONE_REGISTRY.get(cfg.MODEL.BACKBONE.NAME)(cfg, ShapeSpec(channels=len(cfg.MODEL.PIXEL_MEAN)))
        d2_backbone = MaskedBackbone(bb)
        if d2_backbone.num_channels % 16:
            raise capi.Yb200Error(f"Detr: the backbone's last level has {d2_backbone.num_channels} channels (input_proj's GEMM needs a multiple of 16)")
        backbone = Joiner(d2_backbone, PositionEmbeddingSine(hidden_dim // 2, normalize=True))
        backbone.num_channels = d2_backbone.num_channels
        transformer = Transformer(d_model=hidden_dim, dropout=d.DROPOUT, nhead=d.NHEADS, dim_feedforward=d.DIM_FEEDFORWARD,
                                  num_encoder_layers=d.ENC_LAYERS, num_decoder_layers=d.DEC_LAYERS, normalize_before=d.PRE_NORM,
                                  return_intermediate_dec=d.DEEP_SUPERVISION, device=self.device)
        self.detr = DETR(backbone, transformer, num_classes=self.num_classes, num_queries=d.NUM_OBJECT_QUERIES, aux_loss=d.DEEP_SUPERVISION)
        self.detr.to(self.device)
        matcher = HungarianMatcher(cost_class=1, cost_bbox=d.L1_WEIGHT, cost_giou=d.GIOU_WEIGHT)
        weight_dict = {"loss_ce": 1, "loss_bbox": d.L1_WEIGHT}
        weight_dict["loss_giou"] = d.GIOU_WEIGHT
        if d.DEEP_SUPERVISION:
            aux_weight_dict = {}
            for i in range(d.DEC_LAYERS - 1):
                aux_weight_dict.update({k + f"_{i}": v for k, v in weight_dict.items()})
            weight_dict.update(aux_weight_dict)
        self.criterion = SetCriterion(self.num_classes, matcher=matcher, weight_dict=weight_dict, eos_coef=d.NO_OBJECT_WEIGHT,
                                      losses=["labels", "boxes", "cardinality"])
        self.criterion.to(self.device)
        # plain tensors, not buffers (:117-119): they are not in the state_dict
        self.pixel_mean = torch.Tensor(cfg.MODEL.PIXEL_MEAN).to(self.device).view(3, 1, 1)
        self.pixel_std = torch.Tensor(cfg.MODEL.PIXEL_STD).to(self.device).view(3, 1, 1)
        self.to(self.device)
        self.onnx_export = False
        self.L = capi.lib()

    def update_iter(self, i):
        self.iter = i

    # ---- input -------------------------------------------------------------------------------------------------------------------
    def preprocess_image(self, batched_inputs):
        """:273-279: an ImageList of the normalised batch, zero-padded to the batch maximum"""
        out, sizes = normalize_pad(self.L, [x["image"] for x in batched_inputs], self.pixel_mean, self.pixel_std, SIZE_DIVISIBILITY, "Detr")
        return ImageList(out, sizes)

    def prepare_targets(self, targets):
        """:204-217: per image {"labels": int64, "boxes": normalised cxcywh fp32 [n, 4]}, views into one tensor each; the boxes of the whole
        batch are written by one yb200_detr_pack_targets launch"""
        dev = self.device
        boxes, classes, table = [], [], []
        first = 0
        for t in targets:
            h, w = t.image_size
            gb = getattr(t, "gt_boxes", None)
            gb = torch.zeros(0, 4) if gb is None else gb.tensor.reshape(-1, 4)
            gc = getattr(t, "gt_classes", None)
            gc = torch.zeros(0, dtype=torch.int64) if gc is None else gc.reshape(-1)
            if gc.shape[0] != gb.shape[0]:
                raise capi.Yb200Error(f"Detr: an image has {gb.shape[0]} gt_boxes and {gc.shape[0]} gt_classes")
            boxes.append(gb)
            classes.append(gc)
            table.append((first, gb.shape[0], int(h), int(w)))
            first += gb.shape[0]
        if not table:
            raise capi.Yb200Error("Detr: empty batch")
        G = first
        packed = torch.empty(max(G, 1), 4, device=dev)
        labels = _gather(classes, dev, torch.int64)
        if G:
            src = _gather(boxes, dev, torch.float32)
            table_d = pinned_to(np.array(table, dtype=np.int32), dev)
            capi.check(self.L.yb200_detr_pack_targets(capi.ptr(src), capi.ptr(table_d), len(table), G, capi.ptr(packed), capi.stream_ptr()),
                       "detr_pack_targets")
        return [{"labels": labels[f:f + n], "boxes": packed[f:f + n]} for f, n, _, _ in table]

    # ---- forward -----------------------------------------------------------------------------------------------------------------
    def forward(self, batched_inputs):
        if self.onnx_export or torch.onnx.is_in_onnx_export():
            raise capi.Yb200Error("Detr: ONNX export is not supported")
        images = self.preprocess_image(batched_inputs)
        output = self.detr(images)
        if self.training:
            targets = self.prepare_targets([x["instances"] for x in batched_inputs])
            loss_dict = self.criterion(output, targets)
            weight_dict = self.criterion.weight_dict
            for k in loss_dict.keys():
                if k in weight_dict:
                    loss_dict[k] = loss_dict[k] * weight_dict[k]
            return loss_dict
        out_sizes = [(int(x.get("height", s[0])), int(x.get("width", s[1]))) for x, s in zip(batched_inputs, images.image_sizes)]
        results = self.inference(output["pred_logits"], output["pred_boxes"], images.image_sizes, out_sizes)
        return [{"instances": r} for r in results]

    @torch.no_grad()
    def inference(self, box_cls, box_pred, image_sizes, out_sizes):
        """:219-265 followed by detector_postprocess at `out_sizes`, for the whole batch: per image an Instances at (height, width) with
        pred_boxes (XYXY, scaled and clipped), scores fp32 and pred_classes int64 of the queries with score > ignore_thresh and a nonempty
        box, in ascending query order"""
        L, sp, dev = self.L, capi.stream_ptr(), self.device
        logits = box_cls.detach().float().contiguous()
        boxes = box_pred.detach().float().contiguous()
        B, Q, K1 = logits.shape
        if len(image_sizes) != B or len(out_sizes) != B:
            raise capi.Yb200Error(f"Detr: {len(image_sizes)} image sizes for a batch of {B}")
        sizes = np.array([(w, h, np.float32(ow / w), np.float32(oh / h), ow, oh) for (h, w), (oh, ow) in zip(image_sizes, out_sizes)],
                         dtype=np.float32)  # the ratios in double, then fp32: detector_postprocess's Boxes.scale
        sizes_d = pinned_to(sizes, dev)
        score, kept_score = torch.empty(B * Q, device=dev), torch.empty(B * Q, device=dev)
        label, kept_query = torch.empty(B * Q, dtype=torch.int32, device=dev), torch.empty(B * Q, dtype=torch.int32, device=dev)
        keep = torch.empty(B * Q, dtype=torch.uint8, device=dev)
        box, kept_box = torch.empty(B * Q, 4, device=dev), torch.empty(B * Q, 4, device=dev)
        counts, offsets = torch.empty(B + 1, dtype=torch.int32, device=dev), torch.empty(B + 1, dtype=torch.int32, device=dev)
        kept_label = torch.empty(B * Q, dtype=torch.int64, device=dev)
        capi.check(L.yb200_detr_infer(capi.ptr(logits), capi.ptr(boxes), B, Q, K1, capi.ptr(sizes_d), ctypes.c_float(self.ignore_thresh), capi.ptr(score),
                                      capi.ptr(label), capi.ptr(keep), capi.ptr(box), capi.ptr(counts), capi.ptr(offsets), capi.ptr(kept_query),
                                      capi.ptr(kept_score), capi.ptr(kept_label), capi.ptr(kept_box), capi.ptr(counts[B:]), sp), "detr_infer")
        host = torch.empty(B + 1, dtype=torch.int32, pin_memory=True)
        host.copy_(counts, non_blocking=True)  # the B counts and the status word
        done = torch.cuda.Event()
        done.record()
        done.synchronize()
        cnt = host.tolist()
        if cnt[B] & STATUS_NONFINITE_BOX:
            raise capi.Yb200Error("Detr: a predicted box above the score threshold is not finite (Boxes.clip requires finite boxes)")
        first = np.concatenate([[0], np.cumsum(cnt[:B])]).astype(np.int64)
        results = []
        for b in range(B):
            lo, hi = int(first[b]), int(first[b + 1])
            result = Instances(out_sizes[b])
            result.pred_boxes = Boxes(kept_box[lo:hi])
            result.scores = kept_score[lo:hi]
            result.pred_classes = kept_label[lo:hi]
            results.append(result)
        return results
