"""SparseInst meta-architecture on the sm_90a kernels: `@META_ARCH_REGISTRY.register() class SparseInst(nn.Module)`.

Reference: yolov7/modeling/meta_arch/sparseinst.py -- `SparseInst` :55-241.  Same constructor (`cfg.MODEL.{DEVICE, PIXEL_MEAN, PIXEL_STD,
BACKBONE.NAME}`, `cfg.MODEL.SPARSE_INST.*`, `cfg.MODEL.YOLO.CONF_THRESHOLD` as the class threshold, `cfg.INPUT.MASK_FORMAT`), attributes,
state_dict keys and return values.  The backbone stays the caller's (detectron2's `build_backbone(cfg)`, or the bundled registry without
detectron2); the encoder, decoders and criterion are this package's.

  * Input (`preprocess_inputs` :96-100): one non-blocking copy per image into one staging buffer, then one `yb200_normalize_pad` launch writes
    the normalised batch zero-padded to a multiple of 32, bit-identical to the reference's torch arithmetic.
  * Training: the criterion's loss dict, with gradients through decoder, encoder and backbone.
  * Eval (`inference` :179-232): `yb200_sparseinst_infer_scores` scores, thresholds, rescores and compacts every query of the batch; ONE
    device-to-host copy of the B keep counts and one event synchronisation; then `yb200_sparseinst_paste_masks` resizes every kept mask to its
    image's original size and thresholds it in one launch (per 64 images), without a full-resolution intermediate in global memory.
There is no CPU path and no ONNX path (`inference_onnx`): both raise Yb200Error.
"""
import ctypes

import numpy as np
import torch
import torch.nn as nn

from . import capi
from .batch_input import normalize_pad
from .modeling import BACKBONE_REGISTRY, HAVE_D2, META_ARCH_REGISTRY, Instances, ShapeSpec
from .sparseinst import BaseIAMDecoder, GroupIAMDecoder
from .sparseinst_criterion import build_sparse_inst_criterion
from .sparseinst_encoder import InstanceContextEncoder

SIZE_DIVISIBILITY = 32  # ImageList.from_tensors(images, 32) (:99)
DECODERS = {"BaseIAMDecoder": BaseIAMDecoder, "GroupIAMDecoder": GroupIAMDecoder}

if HAVE_D2:  # pragma: no cover - detectron2 is not installed in the build container
    from detectron2.modeling import build_backbone
    from detectron2.structures import BitMasks
else:
    build_backbone = None

    class BitMasks:
        """the part of detectron2's BitMasks the targets need: a bool `.tensor` [g, h, w], `.to(device)` and len()"""

        def __init__(self, tensor):
            self.tensor = torch.as_tensor(tensor).to(torch.bool)

        def to(self, device):
            return BitMasks(self.tensor.to(device))

        def __len__(self):
            return self.tensor.shape[0]


class PasteImage(ctypes.Structure):
    """mirror of `yb200_paste_image` (include/yb200.h)"""

    _fields_ = [("h", ctypes.c_int32), ("w", ctypes.c_int32), ("out_h", ctypes.c_int32), ("out_w", ctypes.c_int32), ("first", ctypes.c_int32),
                ("count", ctypes.c_int32), ("out_off", ctypes.c_int64)]


PASTE_MAX_IMAGES = 64  # YB200_PASTE_MAX_IMAGES


@META_ARCH_REGISTRY.register()
class SparseInst(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        name = cfg.MODEL.SPARSE_INST.DECODER.NAME
        if name not in DECODERS:
            raise capi.Yb200Error(f"SparseInst: decoder {name!r} is not built (only {sorted(DECODERS)})")
        self.device = torch.device(cfg.MODEL.DEVICE)
        if self.device.type != "cuda":
            raise capi.Yb200Error(f"SparseInst: MODEL.DEVICE {cfg.MODEL.DEVICE!r} (the kernels run on CUDA only; there is no CPU path)")
        if HAVE_D2:  # pragma: no cover
            self.backbone = build_backbone(cfg)
        else:
            self.backbone = BACKBONE_REGISTRY.get(cfg.MODEL.BACKBONE.NAME)(cfg, ShapeSpec(channels=len(cfg.MODEL.PIXEL_MEAN)))
        self.backbone.to(self.device)
        self.size_divisibility = self.backbone.size_divisibility
        output_shape = self.backbone.output_shape()
        self.encoder = InstanceContextEncoder(cfg, output_shape, device=self.device)
        self.decoder = DECODERS[name](cfg, device=self.device)
        self.criterion = build_sparse_inst_criterion(cfg)
        self.mask_format = cfg.INPUT.MASK_FORMAT
        # plain tensors, not buffers (:78-81): they are not in the state_dict
        self.pixel_mean = torch.Tensor(cfg.MODEL.PIXEL_MEAN).to(self.device).view(3, 1, 1)
        self.pixel_std = torch.Tensor(cfg.MODEL.PIXEL_STD).to(self.device).view(3, 1, 1)
        self.cls_threshold = cfg.MODEL.YOLO.CONF_THRESHOLD
        self.mask_threshold = cfg.MODEL.SPARSE_INST.MASK_THRESHOLD
        self.max_detections = cfg.MODEL.SPARSE_INST.MAX_DETECTIONS  # unused, as in the reference's inference
        self.L = capi.lib()

    # ---- input -------------------------------------------------------------------------------------------------------------------
    def preprocess_inputs(self, batched_inputs):
        """fp32 [B, 3, Hp, Wp] normalised and zero-padded to a multiple of 32, and the images' (h, w)"""
        return normalize_pad(self.L, [x["image"] for x in batched_inputs], self.pixel_mean, self.pixel_std, SIZE_DIVISIBILITY, "SparseInst")

    def prepare_targets(self, targets):
        """:102-120: per image {"labels": int64 on the device, "masks": BitMasks on the device}"""
        new_targets = []
        for t in targets:
            h, w = t.image_size
            gt_masks = getattr(t, "gt_masks", None) if not hasattr(t, "has") else (t.gt_masks if t.has("gt_masks") else None)
            if gt_masks is None:
                gt_masks = BitMasks(torch.empty(0, h, w, dtype=torch.bool))
            elif self.mask_format == "polygon":
                if not HAVE_D2:
                    raise capi.Yb200Error("SparseInst: MASK_FORMAT 'polygon' needs detectron2's BitMasks.from_polygon_masks (not installed); "
                                          "use MASK_FORMAT 'bitmask'")
                if len(gt_masks.polygons) == 0:  # pragma: no cover
                    gt_masks = BitMasks(torch.empty(0, h, w, dtype=torch.bool))
                else:  # pragma: no cover
                    gt_masks = BitMasks.from_polygon_masks(gt_masks.polygons, h, w)
            new_targets.append({"labels": t.gt_classes.to(self.device), "masks": gt_masks.to(self.device)})
        return new_targets

    # ---- forward -----------------------------------------------------------------------------------------------------------------
    def forward(self, batched_inputs):
        if torch.onnx.is_in_onnx_export():
            raise capi.Yb200Error("SparseInst: ONNX export (inference_onnx) is not supported")
        targets = self.prepare_targets([x["instances"] for x in batched_inputs]) if self.training else None
        images, image_sizes = self.preprocess_inputs(batched_inputs)
        max_shape = images.shape[2:]
        features = self.backbone(images)
        features = self.encoder(features)
        output = self.decoder(features)
        if self.training:
            return self.criterion(output, targets, max_shape)
        results = self.inference(output, batched_inputs, max_shape, image_sizes)
        return [{"instances": r} for r in results]

    @torch.no_grad()
    def inference(self, output, batched_inputs, max_shape, image_sizes):
        """:179-232 for the whole batch: per image an Instances at ("height", "width") with pred_masks bool [k, height, width], scores (the
        rescored fp32 values) and pred_classes int64, kept queries in ascending order; an image without kept queries has no pred_masks"""
        L, sp, dev = self.L, capi.stream_ptr(), self.device
        logits = output["pred_logits"].float().contiguous()
        masks = output["pred_masks"].float().contiguous()
        obj = output["pred_scores"].float().contiguous()
        B, N, K = logits.shape
        hm, wm = int(masks.shape[-2]), int(masks.shape[-1])
        hp, wp = int(max_shape[0]), int(max_shape[1])
        ori = [(int(x["height"]), int(x["width"])) for x in batched_inputs]
        score, rescored, kept_score = (torch.empty(B * N, device=dev) for _ in range(3))
        label, kept_query = torch.empty(B * N, dtype=torch.int32, device=dev), torch.empty(B * N, dtype=torch.int32, device=dev)
        keep = torch.empty(B * N, dtype=torch.uint8, device=dev)
        counts, offsets = torch.empty(B, dtype=torch.int32, device=dev), torch.empty(B + 1, dtype=torch.int32, device=dev)
        kept_label = torch.empty(B * N, dtype=torch.int64, device=dev)
        capi.check(L.yb200_sparseinst_infer_scores(capi.ptr(logits), capi.ptr(obj), capi.ptr(masks), B, N, K, hm * wm, ctypes.c_float(self.cls_threshold),
                                                   ctypes.c_float(self.mask_threshold), capi.ptr(score), capi.ptr(label), capi.ptr(keep),
                                                   capi.ptr(rescored), capi.ptr(counts), capi.ptr(offsets), capi.ptr(kept_query), capi.ptr(kept_score),
                                                   capi.ptr(kept_label), sp), "sparseinst_infer_scores")
        host = torch.empty(B, dtype=torch.int32, pin_memory=True)
        host.copy_(counts, non_blocking=True)
        done = torch.cuda.Event()
        done.record()
        done.synchronize()
        cnt = host.tolist()
        first = np.concatenate([[0], np.cumsum(cnt)]).astype(np.int64)
        nbytes = [c * h * w for c, (h, w) in zip(cnt, ori)]
        out_off = np.concatenate([[0], np.cumsum(nbytes)]).astype(np.int64)
        pasted = torch.empty(max(int(out_off[-1]), 1), dtype=torch.uint8, device=dev)
        plane = hm * wm
        for b0 in range(0, B, PASTE_MAX_IMAGES):
            b1 = min(B, b0 + PASTE_MAX_IMAGES)
            if first[b1] == first[b0]:
                continue
            table = (PasteImage * (b1 - b0))()
            for i, b in enumerate(range(b0, b1)):
                table[i] = PasteImage(image_sizes[b][0], image_sizes[b][1], ori[b][0], ori[b][1], int(first[b] - first[b0]), cnt[b],
                                      int(out_off[b] - out_off[b0]))
            capi.check(L.yb200_sparseinst_paste_masks(ctypes.c_void_p(masks.data_ptr() + 4 * b0 * N * plane), N, hm, wm,
                                                      ctypes.c_void_p(kept_query.data_ptr() + 4 * int(first[b0])), table, b1 - b0, hp, wp,
                                                      ctypes.c_float(self.mask_threshold), ctypes.c_void_p(pasted.data_ptr() + int(out_off[b0])), sp),
                       "sparseinst_paste_masks")
        results = []
        for b in range(B):
            result = Instances(ori[b])
            lo, hi = int(first[b]), int(first[b + 1])
            if hi > lo:  # no pred_masks on an image without kept queries (:198-202)
                h, w = ori[b]
                result.pred_masks = pasted[int(out_off[b]):int(out_off[b + 1])].view(hi - lo, h, w).view(torch.bool)
            result.scores = kept_score[lo:hi]
            result.pred_classes = kept_label[lo:hi]
            results.append(result)
        return results
