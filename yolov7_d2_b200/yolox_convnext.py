"""YOLOX on a ConvNeXt-T backbone (BASELINE.json configs[2], `configs/coco/yolox/yolox_convnext.yaml`): execution plan.

The shipped config is not runnable upstream: `build_convnext_backbone` returns stages 0,1,2 = 96/192/384 channels at strides 4/8/16
(convnext.py:209-230) while `YOLOX` builds `YOLOPAFPN(width=0.5)` with in_channels [256,512,1024]*0.5 and head strides [8,16,32]
(yolox.py:60-70, yolo_pafpn.py:18-21, yolox_head.py:29) -- SURVEY.md par.0.2.  The corrected wiring used here (a documented deviation):

    ConvNeXt-T stages 1, 2, 3 (192 / 384 / 768 channels at strides 8 / 16 / 32, each through its output LayerNorm norm{i})
      -> YOLOPAFPN(depth 0.33, width 0.75)   (in_channels = [256, 512, 1024] * 0.75 = [192, 384, 768])
      -> YOLOXHead(num_classes, width 0.75)  (hidden 192), SimOTA + IoU / BCE losses

Two plans share the work: `ConvNeXtEngine` (csrc/convnext.cu kernels + the wgmma GEMM) and the neck + head range of a width-0.75
`YoloxEngine` (whose own CSPDarknet range never runs).  The object mirrors the YoloxEngine interface that modeling.YOLOX, bench.py and
optim.py use (params / grads / buffers under the reference's `backbone.` / `neck.` / `head.` names, train_step, eval_forward, ...), with
TWO flat parameter buffers (`flat_buffers()`): one optimizer launch and one all-reduce each.
"""
import torch

from . import capi
from .convnext import ConvNeXtEngine
from .engine import YoloxEngine

WIDTH, DEPTH = 0.75, 0.33
STAGES = (1, 2, 3)
FEATS = ("dark3", "dark4", "dark5")


class YoloxConvNeXtEngine:
    def __init__(self, batch, height, width, num_classes=80, max_gt=100, device="cuda", share_params_of=None, layer_scale_init_value=1e-6):
        s = share_params_of
        self.dev = torch.device(device)
        self.n, self.h, self.w, self.nc = batch, height, width, num_classes
        self.cn = ConvNeXtEngine(batch, height, width, out_indices=STAGES, layer_scale_init_value=layer_scale_init_value, device=device,
                                 share_params_of=s.cn if s is not None else None)
        self.yx = YoloxEngine(batch, height, width, num_classes, WIDTH, DEPTH, max_gt, device, share_params_of=s.yx if s is not None else None, strict=False)
        self.range = (self.yx.ranges["neck"][0], len(self.yx.ops))
        self.pad_value = 114.0
        self.device_pad = False  # ConvNeXt's patchify reads images_u8 as is: the host side fills the padding (modeling._stage_batch)
        # reference-named views
        self.params = {"backbone." + n: t for n, t in self.cn.params.items()}
        self.grads = {"backbone." + n: t for n, t in self.cn.grads.items()}
        for n in self.yx.param_names:
            if not n.startswith("backbone."):
                self.params[n], self.grads[n] = self.yx.params[n], self.yx.grads[n]
        self.buffers = {n: t for n, t in self.yx.buffers.items() if not n.startswith("backbone.")}
        self.param_names = ["backbone." + n for n in self.cn.param_names] + [n for n in self.yx.param_names if not n.startswith("backbone.")]
        self.levels, self.num_anchors = self.yx.levels, self.yx.num_anchors
        self.overlap_wgrad = True

    # --- state shared with the YOLOX plan (same objects, so modeling / bench code works on either engine) ---
    images_u8 = property(lambda self: self.cn.images_u8, lambda self, v: setattr(self.cn, "images_u8", v))
    labels = property(lambda self: self.yx.labels, lambda self, v: setattr(self.yx, "labels", v))
    hw_valid = property(lambda self: self.yx.hw_valid, lambda self, v: setattr(self.yx, "hw_valid", v))
    outputs = property(lambda self: self.yx.outputs)
    losses = property(lambda self: self.yx.losses)
    loss_weights = property(lambda self: self.yx.loss_weights)
    fg_mask = property(lambda self: self.yx.fg_mask)
    matched_gt = property(lambda self: self.yx.matched_gt)
    matched_iou = property(lambda self: self.yx.matched_iou)
    matched_cls = property(lambda self: self.yx.matched_cls)
    totals = property(lambda self: self.yx.totals)
    kernel_launches = property(lambda self: self.cn.kernel_launches + self.yx.kernel_launches)

    def flat_buffers(self):
        """[(flat_param, flat_grad, param_layout, norm_param_names)]: one entry per flat buffer (optim.build_optimizers, gradient all-reduce)"""
        yx_norm = {n for n in self.yx.param_names if ".bn." in n}
        cn_layout = [("backbone." + n, off, cnt) for n, off, cnt in self.cn.param_layout]
        return [(self.cn.flat_param, self.cn.flat_grad, cn_layout, set()),  # ConvNeXt's LayerNorm is a custom module: not a torch norm
                (self.yx.flat_param, self.yx.flat_grad, self.yx.param_layout, yx_norm)]

    def init_weights(self, seed=0):
        self.cn.init_weights(seed)
        self.yx.init_weights(seed + 1)

    def load_state_dict(self, sd):
        self.cn.load_state_dict(sd, prefix="backbone.")
        missing = []
        for name, dst in list(self.yx.params.items()) + list(self.yx.buffers.items()):
            if name.startswith("backbone."):
                continue
            if name not in sd:
                missing.append(name)
                continue
            dst.copy_(sd[name].to(self.dev).reshape(dst.shape))
        if missing:
            raise KeyError(f"state_dict lacks {len(missing)} tensors, e.g. {missing[:3]}")

    def state_dict(self):
        out = {k: v.detach().clone() for k, v in self.params.items()}
        out.update({k: v.detach().clone() for k, v in self.buffers.items()})
        return out

    # --- execution ---
    def pack_weights(self):
        self.cn.pack_weights()
        self.yx.pack_weights()

    def preprocess(self):
        pass  # the ConvNeXt stem reads the uint8 image directly (patchify4)

    def forward_features(self, training=True):
        feats = self.cn.forward_features()
        for k, t in zip(FEATS, feats):  # ConvNeXt stage outputs -> the slots where the PAFPN expects dark3 / dark4 / dark5
            self.yx.features[k].tensor().copy_(t)
        self.yx.forward_features(training, self.range)

    def assign_and_loss(self, with_grad=True):
        self.yx.assign_and_loss(with_grad)

    def loss_grad_only(self):
        self.yx.loss_grad_only()

    def backward(self, accumulate=False):
        self.yx.overlap_wgrad = self.cn.overlap_wgrad = self.overlap_wgrad
        self.yx.backward(accumulate, self.range)
        for i, k in zip(STAGES, FEATS):
            self.cn.stage[i].gout.t.copy_(self.yx.features[k].grad_tensor())
        self.cn.backward(accumulate)

    def train_step(self, accumulate=False):
        self.pack_weights()
        self.forward_features(True)
        self.assign_and_loss(True)
        self.backward(accumulate)
        return self.losses

    def eval_forward(self):
        self.pack_weights()
        self.forward_features(False)
        return self.outputs


def check_backbone_name(name):
    if name != "build_convnext_backbone":
        raise capi.Yb200Error(f"YoloxConvNeXtEngine serves MODEL.BACKBONE.NAME = build_convnext_backbone, not {name!r}")
