"""Drop-in surface: the reference's registry / module contracts for the YOLOX path, backed by the H100 engine.

Mirrors (same names, constructor arguments, attributes, state_dict keys and return types):
  * `@META_ARCH_REGISTRY.register() class YOLOX(nn.Module)`            yolov7/modeling/meta_arch/yolox.py:35-252
  * `@BACKBONE_REGISTRY.register() build_cspdarknetx_backbone(cfg, _)`   yolov7/modeling/backbone/darknetx.py:194-213
  * `CSPDarknet`, `YOLOPAFPN`, `YOLOXHead`                               darknetx.py:103, yolo_pafpn.py:13, yolox_head.py:24
  * `postprocess(prediction, num_classes, conf_thre, nms_thre)`          yolov7/utils/boxes.py:171-210
When detectron2 is importable the classes register into ITS registries (so train_det.py / configs/*.yaml drive them);
otherwise a bundled registry with the same interface is used.  All arithmetic happens in libyb200.so: the modules only
own parameters (views into the engine's flat fp32 buffers) and marshal tensors.
"""
import ctypes
import math

import os

import torch
import torch.nn as nn

from . import capi
from .engine import YoloxEngine

try:  # pragma: no cover - detectron2 is not installed in the build container
    from detectron2.modeling import META_ARCH_REGISTRY
    from detectron2.modeling.backbone import BACKBONE_REGISTRY, Backbone
    from detectron2.layers import ShapeSpec
    from detectron2.structures import Boxes, ImageList, Instances
    from detectron2.modeling.postprocessing import detector_postprocess
    HAVE_D2 = True
except Exception:  # noqa: BLE001
    HAVE_D2 = False

    class _Registry(dict):
        """detectron2.utils.registry.Registry look-alike"""

        def __init__(self, name):
            super().__init__()
            self._name = name

        def register(self, obj=None):
            if obj is None:
                return lambda o: self.register(o)
            assert obj.__name__ not in self, f"{obj.__name__} already registered in {self._name}"
            self[obj.__name__] = obj
            return obj

        def get(self, name):
            if name not in self:
                raise KeyError(f"No object named '{name}' found in '{self._name}' registry!")
            return self[name]

    META_ARCH_REGISTRY = _Registry("META_ARCH")
    BACKBONE_REGISTRY = _Registry("BACKBONE")

    class Backbone(nn.Module):
        @property
        def size_divisibility(self):
            return 0

    class ShapeSpec:
        def __init__(self, channels=None, height=None, width=None, stride=None):
            self.channels, self.height, self.width, self.stride = channels, height, width, stride

    class Boxes:
        def __init__(self, tensor):
            self.tensor = tensor

    class Instances:
        def __init__(self, image_size, **kw):
            self.image_size = image_size
            self.__dict__.update(kw)

    def detector_postprocess(results, output_height, output_width):
        sx, sy = output_width / results.image_size[1], output_height / results.image_size[0]
        b = results.pred_boxes.tensor.clone()
        b[:, 0::2] = (b[:, 0::2] * sx).clamp(0, output_width)
        b[:, 1::2] = (b[:, 1::2] * sy).clamp(0, output_height)
        keep = ((b[:, 2] - b[:, 0]) > 0) & ((b[:, 3] - b[:, 1]) > 0)
        out = Instances((output_height, output_width))
        out.pred_boxes, out.scores, out.pred_classes = Boxes(b[keep]), results.scores[keep], results.pred_classes[keep]
        return out


# ------------------------------------------------------------------------------------------------
# postprocess
# ------------------------------------------------------------------------------------------------
_nms_ws = {}


def postprocess(prediction, num_classes, conf_thre=0.7, nms_thre=0.45, tie_order="stable"):
    """boxes.py:171-210: returns a list with one [n_i, 7] tensor (x1,y1,x2,y2,obj,cls_conf,cls) or None per image and, like
    the reference, rewrites prediction[:, :, :4] to corner format in place.
    tie_order: order of detections with bit-identical scores.  "stable" (default) = lower anchor first, the order of torchvision's `nms`
    (the reference on CUDA, and on the CPU for <= 1000 candidates).  "torch_cpu_sort" re-applies, for images that contain ties, the
    permutation of the UNSTABLE `scores[keep].sort(descending=True)` that ends torchvision's CPU `_batched_nms_vanilla` (the reference on
    the CPU with > 1000 candidates) -- by issuing that very call on the kept scores; images without ties never leave the device path."""
    if not (prediction.is_cuda and prediction.dtype == torch.float32 and prediction.dim() == 3):
        raise capi.Yb200Error("postprocess: expects a CUDA fp32 [B, A, 5+C] tensor (no CPU fallback)")
    if tie_order not in ("stable", "torch_cpu_sort"):
        raise ValueError(f"postprocess: unknown tie_order {tie_order!r}")
    pred = prediction if prediction.is_contiguous() else prediction.contiguous()
    b, a, ch = pred.shape
    if ch != 5 + num_classes:
        raise IndexError(f"prediction has {ch} channels, expected {5 + num_classes}")
    L = capi.lib()
    key = (pred.device.index, b, a)
    if key not in _nms_ws:
        _nms_ws[key] = (torch.empty(L.yb200_nms_workspace(b, a), dtype=torch.uint8, device=pred.device),
                        torch.empty(b, a, 7, device=pred.device), torch.empty(2, b, dtype=torch.int32, device=pred.device),
                        torch.empty(b, a, dtype=torch.int32, device=pred.device))
    ws, det, cnt, anchor = _nms_ws[key]
    want_ties = tie_order == "torch_cpu_sort"
    capi.check(L.yb200_postprocess_nms_indexed(capi.ptr(pred), b, a, num_classes, ctypes.c_float(conf_thre), ctypes.c_float(nms_thre), 1, capi.ptr(ws),
                                               capi.ptr(det), capi.ptr(cnt[0]), capi.ptr(anchor) if want_ties else None,
                                               capi.ptr(cnt[1]) if want_ties else None, capi.stream_ptr()), "postprocess_nms")
    if pred is not prediction:
        prediction.copy_(pred)
    counts, ties = cnt.tolist()  # the one host synchronisation: the output is a ragged Python list
    out = []
    for i, n in enumerate(counts):
        if n == 0:
            out.append(None)
            continue
        d = det[i, :n].clone()
        if want_ties and ties[i] > 0:
            d = d[anchor[i, :n].argsort()]                       # ascending anchor = the order of `torch.where(keep_mask)`
            perm = (d[:, 4] * d[:, 5]).cpu().sort(descending=True)[1]  # boxes.py:199-203 scores; torchvision/ops/boxes.py `_batched_nms_vanilla` last line
            d = d[perm.to(d.device)]
        out.append(d)
    return out


# ------------------------------------------------------------------------------------------------
# modules
# ------------------------------------------------------------------------------------------------
class _ParamTree(nn.Module):
    """nn.Module tree whose Parameters / buffers are views of an engine's flat storage, under the reference's names"""

    def __init__(self):
        super().__init__()

    def _adopt(self, engine, prefix):
        for name, t in engine.params.items():
            if name.startswith(prefix):
                self._place(name[len(prefix):], nn.Parameter(t, requires_grad=True), False)
        for name, t in engine.buffers.items():
            if name.startswith(prefix):
                self._place(name[len(prefix):], t, True)

    def _place(self, dotted, value, is_buffer):
        mod = self
        parts = dotted.split(".")
        for p in parts[:-1]:
            if p not in mod._modules:
                mod.add_module(p, nn.Module())
            mod = mod._modules[p]
        if is_buffer:
            mod.register_buffer(parts[-1], value)
        else:
            mod.register_parameter(parts[-1], value)


_ADOPTING = [False]  # True while YOLOX.__init__ builds its sub-modules: they adopt YOLOX's parameter storage instead of creating their own


class _PartFn(torch.autograd.Function):
    """One of the three parts of the plan (backbone / neck / head-train) executed on its own: forward = the engine ops of that range,
    backward = the same range of the engine backward, seeded with the gradients autograd delivers for the part's outputs."""

    @staticmethod
    def forward(ctx, eng, part, training, in_views, out_views, n_in, *tensors):
        inputs = tensors[:n_in]
        eng.pack_weights()
        for v, t in zip(in_views, inputs):
            v.tensor().copy_(t.detach().permute(0, 2, 3, 1))
        eng.forward_features(training, eng.ranges[part])
        ctx.eng, ctx.part, ctx.in_views, ctx.out_views, ctx.n_in = eng, part, in_views, out_views, n_in
        ctx.need_in = [t.requires_grad for t in inputs]
        return tuple(v.tensor().permute(0, 3, 1, 2).float().contiguous() for v in out_views)

    @staticmethod
    def backward(ctx, *grads):
        eng = ctx.eng
        for v, g in zip(ctx.out_views, grads):
            gt = v.grad_tensor()
            if g is None:
                gt.zero_()
            else:
                gt.copy_(g.permute(0, 2, 3, 1))
        eng.backward(False, eng.ranges[ctx.part], seeded=ctx.out_views)
        gin = [v.grad_tensor().permute(0, 3, 1, 2).float().contiguous() if need else None for v, need in zip(ctx.in_views, ctx.need_in)]
        prefix = ctx.part + "."
        gpar = [eng.grads[n].clone() for n in eng.param_names if n.startswith(prefix)]
        return (None,) * 6 + tuple(gin) + tuple(gpar)


class _Part(_ParamTree):
    """shared machinery of the standalone modules: own parameter storage (a root plan) unless adopted by YOLOX, one plan per input shape"""

    _part = None

    def _init_storage(self, num_classes, width, depth, device=None):
        self._root, self._plans = None, {}
        self._cfg = (num_classes, width, depth)
        if not _ADOPTING[0]:
            dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
            self._root = YoloxEngine(1, 32, 32, num_classes, width, depth, 100, dev)
            self._root.init_weights(0)
            self._adopt(self._root, self._part + ".")

    def _adopt_root(self, root):
        self._root, self._plans = root, {}
        self._adopt(root, self._part + ".")

    def _plan(self, batch, h, w):
        if self._root is None:
            raise capi.Yb200Error(f"{type(self).__name__} has no parameter storage (constructed inside YOLOX but never adopted)")
        key = (batch, h, w)
        if key not in self._plans:
            nc, wm, dm = self._cfg
            self._plans[key] = YoloxEngine(batch, h, w, nc, wm, dm, 100, self._root.dev, share_params_of=self._root)
        return self._plans[key]

    def _params_of_part(self, eng):
        by_name = dict(self.named_parameters())
        pre = self._part + "."
        return [by_name[n[len(pre):]] for n in eng.param_names if n.startswith(pre)]

    def _run(self, eng, in_views, out_views, inputs):
        for t in inputs:
            if not (t.is_cuda and t.dim() == 4):
                raise capi.Yb200Error(f"{type(self).__name__}.forward expects CUDA NCHW tensors (no CPU fallback)")
        if torch.is_grad_enabled() and self.training:
            return _PartFn.apply(eng, self._part, True, in_views, out_views, len(inputs), *inputs, *self._params_of_part(eng))
        with torch.no_grad():
            return _PartFn.apply(eng, self._part, self.training, in_views, out_views, len(inputs), *inputs)


class CSPDarknet(Backbone, _Part):
    """YOLOX CSPDarknet (darknetx.py:103-191).  Inside YOLOX the parameters live in the model's engine and execution is fused into
    YOLOX.forward; used on its own (the YOLOV5 / YOLOV7P / YOLOMask architectures build it through BACKBONE_REGISTRY and call
    `backbone(x)`), `forward(x)` runs the backbone range of the plan and returns the reference's dict of NCHW fp32 features."""

    _part = "backbone"

    def __init__(self, dep_mul, wid_mul, out_features=("dark3", "dark4", "dark5"), depthwise=False, act="silu"):
        Backbone.__init__(self)
        if depthwise:
            raise capi.Yb200Error("depthwise CSPDarknet is not implemented by this path")
        if act != "silu":
            raise AttributeError("Unsupported act type: {}".format(act))
        assert out_features, "please provide output features of Darknet"
        self.dep_mul, self.wid_mul, self.out_features = dep_mul, wid_mul, out_features
        bc = int(wid_mul * 64)
        self.output_shape_dict = {f"dark{i + 2}": ShapeSpec(channels=bc * 2 ** (i + 1)) for i in range(4)}
        self._init_storage(80, wid_mul, dep_mul)

    def output_shape(self):
        return self.output_shape_dict

    @property
    def size_divisibility(self):
        return 32

    def forward(self, x):
        """x: [B, 3, H, W] float (H, W multiples of 32) -> {name: [B, C, H/s, W/s] fp32 for name in out_features}   (darknetx.py:165-177).
        The Focus slice (wrappers.py:210-220) is laid out by torch indexing; everything after it runs in libyb200.so.  Activations are
        stored in bf16 (the input image too), as in YOLOX.forward."""
        b, c, h, w = x.shape
        if c != 3 or h % 32 or w % 32:
            raise capi.Yb200Error(f"CSPDarknet.forward: input {tuple(x.shape)} must be [B, 3, H, W] with H, W multiples of 32")
        eng = self._plan(b, h, w)
        focus = torch.cat((x[..., ::2, ::2], x[..., 1::2, ::2], x[..., ::2, 1::2], x[..., 1::2, 1::2]), 1)  # [B, 12, H/2, W/2]
        eng.focus.t[..., :12].copy_(focus.detach().permute(0, 2, 3, 1))
        names = [k for k in ("dark2", "dark3", "dark4", "dark5") if k in self.out_features]
        outs = self._run(eng, (), tuple(eng.features[k] for k in names), ())
        return dict(zip(names, outs))


class YOLOPAFPN(_Part):
    """yolo_pafpn.py:13-114: forward(dict of backbone features) -> (pan_out2, pan_out1, pan_out0), NCHW fp32"""

    _part = "neck"

    def __init__(self, depth=1.0, width=1.0, in_features=("dark3", "dark4", "dark5"), in_channels=[256, 512, 1024], depthwise=False, act="silu"):
        super().__init__()
        if depthwise:
            raise capi.Yb200Error("depthwise YOLOPAFPN is not implemented by this path")
        self.in_features, self.in_channels = in_features, in_channels
        self._init_storage(80, width, depth)

    def forward(self, out_features):
        feats = [out_features[f] for f in self.in_features]
        b, _, h8, w8 = feats[0].shape
        eng = self._plan(b, 8 * h8, 8 * w8)
        in_views = tuple(eng.features[k] for k in ("dark3", "dark4", "dark5"))
        for v, t in zip(in_views, feats):
            if tuple(t.shape) != (v.shape[0], v.shape[3], v.shape[1], v.shape[2]):
                raise capi.Yb200Error(f"YOLOPAFPN.forward: feature {tuple(t.shape)} does not match the plan {v.shape}")
        return self._run(eng, in_views, eng.pan, tuple(feats))


class YOLOXHead(_Part):
    """yolox_head.py:24-272.  Evaluation: forward(xin) -> [B, A, 5+C] decoded predictions (sigmoid applied).  Training with labels runs
    inside YOLOX.forward (one fused autograd node); the standalone module covers the inference call of the other architectures."""

    _part = "head"

    def __init__(self, num_classes, width=1.0, strides=[8, 16, 32], in_channels=[256, 512, 1024], act="silu", depthwise=False):
        super().__init__()
        if depthwise:
            raise capi.Yb200Error("depthwise YOLOXHead is not implemented by this path")
        self.n_anchors, self.num_classes = 1, num_classes
        self.decode_in_inference = True
        self.use_l1 = False
        self.strides = strides
        self.onnx_export = False
        self.hw = None
        self._init_storage(num_classes, width, 0.33)

    def initialize_biases(self, prior_prob):
        """yolox_head.py:140-149"""
        v = -math.log((1 - prior_prob) / prior_prob)
        with torch.no_grad():
            for name, p in self.named_parameters():
                if name.endswith(".bias") and (name.startswith("cls_preds") or name.startswith("obj_preds")):
                    p.fill_(v)

    def forward(self, xin, labels=None, imgs=None):
        if self.training or labels is not None:
            raise capi.Yb200Error("YOLOXHead training (SimOTA + losses) runs fused inside YOLOX.forward; the standalone head is the "
                                  "inference path: call .eval() and forward(xin)")
        feats = list(xin)
        b, _, h8, w8 = feats[0].shape
        eng = self._plan(b, 8 * h8, 8 * w8)
        self.hw = [tuple(f.shape[-2:]) for f in feats]
        with torch.no_grad():
            eng.pack_weights()
            for v, t in zip(eng.pan, feats):
                v.tensor().copy_(t.permute(0, 2, 3, 1))
            eng.forward_features(False, eng.ranges["head"])
            return eng.outputs.clone()


@BACKBONE_REGISTRY.register()
def build_cspdarknetx_backbone(cfg, input_shape=None):
    """darknetx.py:194-213"""
    return CSPDarknet(dep_mul=cfg.MODEL.YOLO.DEPTH_MUL, wid_mul=cfg.MODEL.YOLO.WIDTH_MUL, depthwise=cfg.MODEL.DARKNET.DEPTH_WISE,
                      out_features=cfg.MODEL.DARKNET.OUT_FEATURES, act="silu")


def _run_graphed(eng, key, fn):
    """Run `fn` (a fixed sequence of launches on the plan's static buffers) -- eagerly for the first call (lazy allocations),
    then captured once into a CUDA graph and replayed: the public API then costs one graph launch per pass instead of ~250 kernel launches."""
    if not getattr(eng, "use_graphs", False):
        return fn()
    st = eng.__dict__.setdefault("_api_graphs", {})
    ent = st.setdefault(key, {"calls": 0, "graph": None})
    if ent["graph"] is None:
        ent["calls"] += 1
        if ent["calls"] <= 1:
            return fn()
        try:
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, capture_error_mode="thread_local"):
                fn()
            ent["graph"] = g
        except Exception as e:  # noqa: BLE001  (capture unsupported in this context: stay eager, loudly)
            import warnings
            warnings.warn(f"yolov7_d2_b200: CUDA graph capture of the {key} pass failed ({e}); continuing with eager launches")
            eng.use_graphs = False
            torch.cuda.synchronize()
            return fn()
    ent["graph"].replay()


class _TrainStep(torch.autograd.Function):
    """forward = engine forward + SimOTA + losses; backward = the whole engine backward.  Inputs are the model's
    parameters so that autograd / DDP / optimizers see ordinary per-parameter gradients."""

    @staticmethod
    def forward(ctx, engine, flat_grads, *params):
        ctx.flat_grads = flat_grads

        def fwd():
            engine.pack_weights()
            engine.preprocess()
            engine.forward_features(True)
            engine.assign_and_loss(with_grad=False)

        l1 = bool(getattr(getattr(engine, "yx", engine), "use_l1", False))  # the captured graphs differ (decode keeps the raw outputs, the loss has a fourth term)
        ctx.graph_tag = "+l1" if l1 else ""
        _run_graphed(engine, "forward" + ctx.graph_tag, fwd)
        ctx.engine = engine
        l = engine.losses
        return l[0].clone(), l[1].clone(), l[2].clone(), l[3].clone(), l[4].clone()

    @staticmethod
    def backward(ctx, g_total, g_iou, g_obj, g_cls, g_l1):
        eng = ctx.engine
        # outputs: total = 5*iou + obj + cls [+ l1], iou_loss = 5*iou, conf_loss = obj, cls_loss = cls, l1_loss = l1   (yolox.py:201-208)
        eng.loss_weights.copy_(torch.stack([5.0 * (g_total + g_iou), g_total + g_obj, g_total + g_cls, g_total + g_l1]).float())
        if ctx.flat_grads:
            # every parameter's .grad already is its slice of the flat gradient buffer (YOLOX.attach_flat_grads): accumulate in place
            gb = getattr(eng, "_grad_buckets", None)
            if gb is not None:  # data parallel: backward range by range, each bucket's all-reduce overlapping the next range (dist.py)
                eng.loss_grad_only()
                gb.step_backward(accumulate=True)
                gb.wait()
            else:
                def bwd():
                    eng.loss_grad_only()
                    eng.backward(accumulate=True)

                _run_graphed(eng, "backward" + ctx.graph_tag, bwd)
            return (None, None) + (None,) * len(eng.param_names)
        eng.loss_grad_only()
        eng.backward()
        return (None, None) + tuple(eng.grads[n].clone() for n in eng.param_names)


@META_ARCH_REGISTRY.register()
class YOLOX(nn.Module):
    """yolox.py:35-252.  `forward(batched_inputs)` -> loss dict (training) or list of {"instances": Instances} (eval)."""

    def __init__(self, cfg):
        super().__init__()
        self.device = torch.device(cfg.MODEL.DEVICE)
        if self.device.type != "cuda":
            raise capi.Yb200Error("the YOLOX path of this package needs MODEL.DEVICE = cuda")
        self.conf_threshold = cfg.MODEL.YOLO.CONF_THRESHOLD
        self.nms_threshold = cfg.MODEL.YOLO.NMS_THRESHOLD
        self.nms_type = cfg.MODEL.NMS_TYPE
        self.loss_type = cfg.MODEL.YOLO.LOSS_TYPE
        self.use_l1 = False
        self.depth_mul, self.width_mul = cfg.MODEL.YOLO.DEPTH_MUL, cfg.MODEL.YOLO.WIDTH_MUL
        self.iter = 0
        self.max_iter = cfg.SOLVER.MAX_ITER
        self.enable_l1_loss_at = cfg.INPUT.MOSAIC_AND_MIXUP.DISABLE_AT_ITER
        self.num_classes = cfg.MODEL.YOLO.CLASSES
        self.max_boxes_num = cfg.MODEL.YOLO.MAX_BOXES_NUM
        self.in_features = cfg.MODEL.YOLO.IN_FEATURES
        self.padded_value = cfg.MODEL.PADDED_VALUE
        self.size_divisibility = 32
        self.onnx_export = False

        # parameter storage lives in a tiny "root" plan; execution plans per (batch, H, W) share it
        self._convnext = cfg.MODEL.BACKBONE.NAME == "build_convnext_backbone"
        self._plans = {}
        if self._convnext:
            # configs/coco/yolox/yolox_convnext.yaml with the corrected wiring of yolox_convnext.py (the shipped one does not run: SURVEY.md par.0.2):
            # ConvNeXt-T stages 1-3 -> PAFPN / head of width 0.75
            from .yolox_convnext import DEPTH, WIDTH, YoloxConvNeXtEngine
            self.width_mul, self.depth_mul = WIDTH, DEPTH
            self._root = YoloxConvNeXtEngine(1, 32, 32, self.num_classes, self.max_boxes_num, self.device)
            self._root.init_weights(0)
            _ADOPTING[0] = True
            try:
                self.backbone = _Part()
                self.neck = YOLOPAFPN(depth=DEPTH, width=WIDTH, in_features=self.in_features)
                self.head = YOLOXHead(self.num_classes, width=WIDTH)
            finally:
                _ADOPTING[0] = False
            self.backbone._adopt(self._root, "backbone.")
            for part in (self.neck, self.head):
                part._cfg = (self.num_classes, WIDTH, DEPTH)
                part._adopt_root(self._root.yx)
        else:
            self._root = YoloxEngine(1, 32, 32, self.num_classes, self.width_mul, self.depth_mul, self.max_boxes_num, self.device)
            self._root.init_weights(0)
            _ADOPTING[0] = True  # the sub-modules share this model's parameter storage instead of allocating their own
            try:
                self.backbone = BACKBONE_REGISTRY.get(cfg.MODEL.BACKBONE.NAME)(cfg, None)
                self.neck = YOLOPAFPN(depth=self.depth_mul, width=self.width_mul, in_features=self.in_features)
                self.head = YOLOXHead(self.num_classes, width=self.width_mul)
            finally:
                _ADOPTING[0] = False
            for part in (self.backbone, self.neck, self.head):
                part._cfg = (self.num_classes, self.width_mul, self.depth_mul)
                part._adopt_root(self._root)
        self.head.initialize_biases(1e-2)
        self._param_list = None
        self._flat_grads = False
        self._copy_stream = None
        self._prefetched = None
        # training passes replay CUDA graphs captured on the plan's static buffers after two eager warm-up calls (YB200_API_GRAPHS=0: eager)
        import os
        self.use_cuda_graphs = os.environ.get("YB200_API_GRAPHS", "1") == "1"

    @property
    def engine(self):
        """the plan that owns the flat parameter / gradient buffers (yolov7_d2_b200.optim builds its optimizers on them)"""
        return self._root

    def attach_flat_grads(self):
        """Make every parameter's .grad a view into the flat gradient buffer, so that backward writes gradients where the flat
        optimizer and the single all-reduce read them (no per-parameter copies).  Needs zero_grad(set_to_none=False)."""
        for name, p in zip(self._root.param_names, self._params_in_engine_order()):
            p.grad = self._root.grads[name]
        self._flat_grads = True

    def _ensure_flat_grads(self):
        """zero_grad(set_to_none=True) (torch's default) drops the views: re-attach them, zeroed, which is what "none" means to autograd"""
        for name, p in zip(self._root.param_names, self._params_in_engine_order()):
            view = self._root.grads[name]
            if p.grad is None or p.grad.data_ptr() != view.data_ptr():
                view.zero_()
                p.grad = view

    def enable_overlapped_allreduce(self, group=None):
        """Data-parallel training on the flat buffers without DistributedDataParallel: after attach_flat_grads(), every backward reduces the
        gradient in three buckets (head / neck / backbone + BatchNorm) over `group`, each NCCL all-reduce overlapping the backward of the next
        range (yolov7_d2_b200.dist.GradientBuckets).  The SUM is left in the buffer; set optimizer.grad_scale = 1 / world_size for DDP's mean."""
        if self._convnext:
            raise capi.Yb200Error("enable_overlapped_allreduce: only the CSPDarknet plan is bucketed; all-reduce engine.flat_buffers() for ConvNeXt")
        self._dp_group = (group,)
        for eng in self._plans.values():
            self._attach_buckets(eng)

    def _attach_buckets(self, eng):
        from .dist import GradientBuckets
        eng._grad_buckets = GradientBuckets(eng, self._dp_group[0])

    def update_iter(self, i):
        self.iter = i

    def _maybe_enable_l1(self):
        """yolox.py:105-121: past `INPUT.MOSAIC_AND_MIXUP.DISABLE_AT_ITER` (the last, augmentation-free iterations) the head adds the L1 term.  The
        reference broadcasts rank 0's decision; every rank evaluates the same `iter > enable_l1_loss_at`, so the flag is set locally."""
        if self.training and not self.use_l1 and self.iter > self.enable_l1_loss_at:
            self.use_l1 = True
            self.head.use_l1 = True

    # -- helpers ---------------------------------------------------------------------------------
    def _plan(self, batch, h, w):
        key = (batch, h, w)
        if key not in self._plans and self._convnext:
            from .yolox_convnext import YoloxConvNeXtEngine
            self._plans[key] = YoloxConvNeXtEngine(batch, h, w, self.num_classes, self.max_boxes_num, self.device, share_params_of=self._root)
        if key not in self._plans:
            self._plans[key] = YoloxEngine(batch, h, w, self.num_classes, self.width_mul, self.depth_mul, self.max_boxes_num, self.device,
                                           share_params_of=self._root)
            self._plans[key].pad_value = float(self.padded_value)  # cfg.MODEL.PADDED_VALUE (yolox.py:55, ImageList.from_tensors pad_value)
            self._plans[key].use_graphs = self.use_cuda_graphs
            if getattr(self, "_dp_group", None) is not None:
                self._attach_buckets(self._plans[key])
        return self._plans[key]

    def _params_in_engine_order(self):
        if self._param_list is None:
            by_name = dict(self.named_parameters())
            self._param_list = [by_name[n] for n in self._root.param_names]
        return self._param_list

    def _plan_for(self, batched_inputs):
        imgs = [x["image"] for x in batched_inputs]
        hmax = max(i.shape[-2] for i in imgs)
        wmax = max(i.shape[-1] for i in imgs)
        hp, wp = (hmax + 31) // 32 * 32, (wmax + 31) // 32 * 32
        return self._plan(len(imgs), hp, wp), imgs, hp, wp

    def _stage_batch(self, batched_inputs, training, eng, imgs, hp, wp, images_dst, labels_dst, hw_dst):
        """copies of one batch into device buffers on the CURRENT stream (yolox.py:95-162: uint8 CHW images padded bottom/right to a
        multiple of 32 -- pad pixels become PADDED_VALUE on the device --, labels [B, max_boxes, 5] = (cls, cx, cy, w, h) from XYXY boxes)"""
        same = all(i.shape[-2:] == (hp, wp) and i.dtype == torch.uint8 for i in imgs)
        if same and all(i.is_cuda for i in imgs):
            images_dst.copy_(torch.stack(imgs))
        elif same:
            # host images: one H2D copy of the whole batch if the images are consecutive slices of one pinned tensor (a collated batch)
            nbytes = imgs[0].numel()
            base = imgs[0]
            contiguous_run = base.is_pinned() and all(i.is_contiguous() and i.data_ptr() == base.data_ptr() + k * nbytes for k, i in enumerate(imgs))
            if contiguous_run:
                images_dst.copy_(torch.as_strided(base, (len(imgs), 3, hp, wp), (nbytes, hp * wp, wp, 1)), non_blocking=True)
            else:
                # separately allocated images (what a detectron2 dataloader hands over): one asynchronous copy each, no host-side gather;
                # the driver stages pageable memory through its own pinned buffers
                for k, im in enumerate(imgs):
                    images_dst[k].copy_(im, non_blocking=True)
        else:
            if not getattr(eng, "device_pad", True):  # a plan that reads images_u8 as is: the padding value goes in here
                images_dst.fill_(int(round(self.padded_value)))
            for k, im in enumerate(imgs):
                images_dst[k, :, :im.shape[-2], :im.shape[-1]].copy_(im if im.dtype == torch.uint8 else im.round().clamp_(0, 255).to(torch.uint8), non_blocking=True)  # pixel values are integers 0..255 (detectron2 mappers emit uint8); a float image is rounded, never truncated
        hw_dst.copy_(torch.tensor([[i.shape[-2], i.shape[-1]] for i in imgs], dtype=torch.int32), non_blocking=True)
        if training:
            self._stage_labels(batched_inputs, labels_dst)

    def _stage_labels(self, batched_inputs, labels_dst):
        """[B, max_boxes, 5] = (cls, cx, cy, w, h), zero padded (yolox.py:150-162, BoxModeMy XYXY_ABS -> cxcywh boxes.py:547-551).
        One concatenation + one scatter on whichever device the ground truth lives on: no per-image device->host round trip (the
        reference pays one per image, yolox.py:157).  Row counts come from tensor shapes, which are host-side metadata."""
        boxes, classes, bi, ji = [], [], [], []
        for k, x in enumerate(batched_inputs):
            inst = x.get("instances", x.get("targets"))
            if inst is None:
                continue
            b = inst.gt_boxes.tensor[: self.max_boxes_num]
            n = b.shape[0]
            if n == 0:
                continue
            boxes.append(b.detach())
            classes.append(inst.gt_classes[:n].detach())
            bi.append(torch.full((n,), k, dtype=torch.int64))
            ji.append(torch.arange(n, dtype=torch.int64))
        labels_dst.zero_()
        if not boxes:
            return
        on_dev = boxes[0].is_cuda
        bx = torch.cat(boxes).float()
        cl = torch.cat(classes).float()
        rows = torch.stack([cl, (bx[:, 0] + bx[:, 2]) / 2, (bx[:, 1] + bx[:, 3]) / 2, bx[:, 2] - bx[:, 0], bx[:, 3] - bx[:, 1]], 1)
        flat_idx = torch.cat(bi) * self.max_boxes_num + torch.cat(ji)
        if on_dev:
            labels_dst.view(-1, 5).index_copy_(0, flat_idx.to(labels_dst.device, non_blocking=True), rows.to(labels_dst.device))
        else:
            host = torch.zeros(labels_dst.shape[0] * self.max_boxes_num, 5)
            host.index_copy_(0, flat_idx, rows)
            labels_dst.copy_(host.view_as(labels_dst), non_blocking=True)

    def prefetch(self, batched_inputs):
        """Input-side pipelining (SURVEY.md par.8f rank 2): start the host->device copies of the NEXT batch on a copy stream while the
        current step is still running; the following `forward(batched_inputs)` with this same list only copies device-to-device into the plan's
        static buffers.  The copies go into the plan's alternate buffers as soon as their previous contents have been consumed.  Optional: forward() alone behaves exactly like the reference (copy, then compute)."""
        eng, imgs, hp, wp = self._plan_for(batched_inputs)
        if self._copy_stream is None:
            self._copy_stream = torch.cuda.Stream(device=self.device)
            self._copy_done = torch.cuda.Event()
        cur = torch.cuda.current_stream()
        if getattr(eng, "_alt", None) is None:
            eng._alt = (torch.empty_like(eng.images_u8), torch.empty_like(eng.labels), torch.empty_like(eng.hw_valid))
            # the caching allocator may hand these out from blocks that work queued on the current stream still reads or writes (a
            # temporary freed by the step in flight): the copy stream must not write them before that work is done (once per plan)
            self._copy_stream.wait_stream(cur)
        # inputs that live on the device were produced on the caller's stream: read them after it, and keep their memory from being reused
        # before the copy stream is done with it, so that the caller may drop its references as soon as prefetch() returns.  Host inputs
        # add no wait: their copies overlap the step in flight.
        dev_inputs = self._device_inputs(batched_inputs, imgs)
        if dev_inputs:
            self._copy_stream.wait_stream(cur)
            for t in dev_inputs:
                t.record_stream(self._copy_stream)
        with torch.cuda.stream(self._copy_stream):
            # the alternate buffers were last READ by the device-to-device copy at the head of the step that consumed the previous prefetch
            # (preprocess_image records `_alt_free` there): wait for that, not for the whole step in flight -- the DMA overlaps its kernels
            free = getattr(eng, "_alt_free", None)
            if free is not None:
                self._copy_stream.wait_event(free)
            self._stage_batch(batched_inputs, self.training, eng, imgs, hp, wp, *eng._alt)
            self._copy_done.record(self._copy_stream)
        self._prefetched = (batched_inputs, eng)

    def _device_inputs(self, batched_inputs, imgs):
        """the caller's CUDA tensors that staging a batch reads: images, and the ground truth when training"""
        out = [i for i in imgs if i.is_cuda]
        if self.training:
            for x in batched_inputs:
                inst = x.get("instances", x.get("targets"))
                if inst is not None:
                    out += [t for t in (inst.gt_boxes.tensor, inst.gt_classes) if t.is_cuda]
        return out

    def preprocess_image(self, batched_inputs, training):
        eng, imgs, hp, wp = self._plan_for(batched_inputs)
        image_sizes = [(i.shape[-2], i.shape[-1]) for i in imgs]
        pre = self._prefetched
        if pre is not None and pre[0] is batched_inputs and pre[1] is eng:
            # the batch already sits in the alternate device buffers: move it into the plan's static buffers (captured graphs read fixed
            # addresses); 79 MB device-to-device, ~50 us
            torch.cuda.current_stream().wait_event(self._copy_done)
            alt = eng._alt
            eng.images_u8.copy_(alt[0], non_blocking=True)
            eng.labels.copy_(alt[1], non_blocking=True)
            eng.hw_valid.copy_(alt[2], non_blocking=True)
            if getattr(eng, "_alt_free", None) is None:
                eng._alt_free = torch.cuda.Event()
            eng._alt_free.record(torch.cuda.current_stream())
            self._prefetched = None
            return eng, image_sizes
        self._stage_batch(batched_inputs, training, eng, imgs, hp, wp, eng.images_u8, eng.labels, eng.hw_valid)
        return eng, image_sizes

    # -- forward ---------------------------------------------------------------------------------
    def forward(self, batched_inputs):
        eng, image_sizes = self.preprocess_image(batched_inputs, self.training)
        if self.training:
            if self._flat_grads:
                self._ensure_flat_grads()
            self._maybe_enable_l1()
            target = getattr(eng, "yx", eng)  # the YOLOX-ConvNeXt composite keeps the head in its YoloxEngine
            target.use_l1 = bool(self.use_l1)
            total, iou, conf, cls, l1 = _TrainStep.apply(eng, self._flat_grads, *self._params_in_engine_order())
            out = {"total_loss": total, "iou_loss": iou, "conf_loss": conf, "cls_loss": cls}
            if self.use_l1:
                out["l1_loss"] = l1  # yolox.py:207-208
            return out
        with torch.no_grad():
            outputs = eng.eval_forward()
            detections = postprocess(outputs, self.num_classes, self.conf_threshold, self.nms_threshold)
        results = []
        for idx, (out, inp) in enumerate(zip(detections, batched_inputs)):
            if out is None:
                out = outputs.new_zeros((0, 7))
            res = Instances(image_sizes[idx])
            res.pred_boxes = Boxes(out[:, :4])
            res.scores = out[:, 5] * out[:, 4]
            res.pred_classes = out[:, -1]
            h, w = inp.get("height", image_sizes[idx][0]), inp.get("width", image_sizes[idx][1])
            results.append({"instances": detector_postprocess(res, h, w)})
        return results
