"""SparseInst InstanceContextEncoder on the H100 kernels, forward and backward.

Reference: yolov7/modeling/transcoders/encoder_sparseinst.py -- `MyAdaptiveAvgPool2d` :18-39, `PyramidPoolingModule` :42-68,
`InstanceContextEncoder` :71-127.  `InstanceContextEncoder(cfg, input_shape)` below keeps the reference's constructor (cfg.MODEL.SPARSE_INST.ENCODER
NUM_CHANNELS / IN_FEATURES; NORM is read by nothing upstream), its parameter names / shapes (`fpn_laterals.{0,1,2}.*`, `fpn_outputs.{0,1,2}.*`
with index 0 the coarsest level, `ppm.stages.{0..3}.1.*`, `ppm.bottleneck.*`, `fusion.*`), its initialisation (c2_xavier_fill on the laterals
and outputs, c2_msra_fill on fusion, torch's Conv2d default on the PPM convolutions) and `forward(features: dict) -> fp32 NCHW [B, C, H3, W3]`,
the decoder's input.

Kernel sequence (NHWC bf16 inside; DESIGN.md par.7):
  lat0 = 1x1(res5) written into cat512[..., C:2C]  |  per PPM size s: avg_pool2d with window (ceil(H/s), ceil(W/s)), floor mode (the reference's
  MyAdaptiveAvgPool2d is not adaptive pooling), 1x1 + bias + ReLU, bilinear resize into cat512[..., s*C/4 : (s+1)*C/4]  |  prev0 = ReLU(1x1(cat512))
  out0 = 3x3(prev0)  |  per finer level: prev = 1x1(res) + nearest x2(prev), out = 3x3(prev); the finest out is written into cat768[..., 0:C]
  bilinear resize of out1 / out0 into cat768[..., C:2C] / [..., 2C:3C]  |  fusion = 1x1(cat768) -> bf16, returned as fp32 NCHW
The pooled maps and the PPM priors are tiny ([B, 1..6, 1..6, C]); their 1x1 convolutions run on one row block [1, 1, rows, C] with the rows
padded to a multiple of 16 by zeros, which change neither a weight gradient nor a column sum.
Training: with autograd recording and an input or a parameter requiring grad, the encoder is one autograd node (`_EncoderFn`) that issues the
same forward calls and keeps the intermediates; its backward returns every parameter's fp32 gradient and d res3 / res4 / res5 (fp32 NCHW, only
for the inputs that require grad) on this library's kernels.  Sums run in a fixed order (no float atomics): two backward calls give the same bits.
"""
import ctypes
import math

import torch
import torch.nn as nn

from . import capi

PPM_SIZES = (1, 2, 3, 6)


def _pad16(c):
    return (c + 15) // 16 * 16


def _conv(cin, cout, k, device):
    """nn.Conv2d as the holder of `weight` / `bias` (torch's default initialisation); the convolution itself runs on the kernels"""
    return nn.Conv2d(cin, cout, k, padding=(k - 1) // 2, device=device)


def _xavier_fill(m):
    """fvcore's c2_xavier_fill"""
    nn.init.kaiming_uniform_(m.weight, a=1)
    nn.init.zeros_(m.bias)


def _msra_fill(m):
    """fvcore's c2_msra_fill"""
    nn.init.kaiming_normal_(m.weight, mode="fan_out", nonlinearity="relu")
    nn.init.zeros_(m.bias)


def ppm_windows(h, w):
    """MyAdaptiveAvgPool2d (:18-39): window = stride = (ceil(H/s), ceil(W/s)) per size; the pooled map is (H // kh, W // kw)"""
    return [(math.ceil(h / s), math.ceil(w / s)) for s in PPM_SIZES]


class InstanceContextEncoder(nn.Module):
    def __init__(self, cfg, input_shape, device="cuda"):
        super().__init__()
        enc = cfg.MODEL.SPARSE_INST.ENCODER
        self.num_channels = enc.NUM_CHANNELS
        self.in_features = list(enc.IN_FEATURES)
        self.in_channels = [input_shape[f].channels for f in self.in_features]
        if len(self.in_features) != 3:
            raise capi.Yb200Error(f"InstanceContextEncoder: the fusion reads three levels (IN_FEATURES {self.in_features})")
        if self.num_channels % 64:
            raise capi.Yb200Error(f"InstanceContextEncoder: NUM_CHANNELS {self.num_channels} must be a multiple of 64 (the PPM width NUM_CHANNELS / 4 "
                                  "is a GEMM dimension, a multiple of 16)")
        if any(c % 16 for c in self.in_channels):
            raise capi.Yb200Error(f"InstanceContextEncoder: input channels {self.in_channels} must be multiples of 16")
        dev = torch.device(device)
        c = self.num_channels
        self.fpn_laterals, self.fpn_outputs = nn.ModuleList(), nn.ModuleList()
        for cin in reversed(self.in_channels):                    # :88-97: index 0 is the coarsest level
            lat, out = _conv(cin, c, 1, dev), _conv(c, c, 3, dev)
            _xavier_fill(lat)
            _xavier_fill(out)
            self.fpn_laterals.append(lat)
            self.fpn_outputs.append(out)
        self.ppm = nn.Module()                                    # PyramidPoolingModule(c, c // 4) (:42-54, :101)
        self.ppm.stages = nn.ModuleList()
        for _ in PPM_SIZES:
            st = nn.Module()
            st.add_module("1", _conv(c, c // 4, 1, dev))         # Sequential(MyAdaptiveAvgPool2d, Conv2d): the pool has no parameters
            self.ppm.stages.append(st)
        self.ppm.bottleneck = _conv(c + len(PPM_SIZES) * (c // 4), c, 1, dev)
        self.fusion = _conv(3 * c, c, 1, dev)                     # :103-104
        _msra_fill(self.fusion)
        self.L = capi.lib()

    # ---- helpers -----------------------------------------------------------------------------------------------------------------
    def _pack(self, w, dgrad=False):
        """fp32 OIHW -> the bf16 GEMM operand: [cout][k*k][cin] (forward, weight gradient) or [cin][k*k][cout] (data gradient)"""
        cout, cin, k = w.shape[0], w.shape[1], w.shape[2]
        shape = (cin, k * k, cout) if dgrad else (cout, k * k, cin)
        wp = torch.empty(shape, dtype=torch.bfloat16, device=w.device)
        fwd, dg = (None, wp) if dgrad else (wp, None)
        capi.check(self.L.yb200_pack_conv_weight(capi.ptr(w.detach().contiguous()), cout, cin, k, cout, cin, capi.ptr(fwd), capi.ptr(dg),
                                                 capi.stream_ptr()), "pack")
        return wp

    def _affine(self, xa, conv, oa, k):
        """oa = bf16(conv(x) + bias) (nn.Conv2d with bias: the affine epilogue with the bias as shift)"""
        capi.check(self.L.yb200_conv2d_affine_fwd(ctypes.byref(xa), capi.ptr(self._pack(conv.weight)), None, capi.ptr(conv.bias.detach()), None,
                                                  ctypes.byref(oa), k, 1, capi.stream_ptr()), "conv")

    def _relu(self, xa, conv, oa):
        """oa = bf16(max(conv1x1(x) + bias, 0))"""
        capi.check(self.L.yb200_conv2d_relu_fwd(ctypes.byref(xa), capi.ptr(self._pack(conv.weight)), capi.ptr(conv.bias.detach()), ctypes.byref(oa), 1,
                                                1, capi.stream_ptr()), "conv + relu")

    def _check(self, features):
        """Yb200Error before any kernel runs: missing keys, CPU inputs, channel counts, levels not 2x apart; returns the inputs coarsest first"""
        missing = [f for f in self.in_features if f not in features]
        if missing:
            raise capi.Yb200Error(f"InstanceContextEncoder: features {missing} (IN_FEATURES) missing from the input")
        xs = [features[f] for f in self.in_features]
        for f, x, c in zip(self.in_features, xs, self.in_channels):
            if not x.is_cuda:
                raise capi.Yb200Error(f"InstanceContextEncoder: {f} must be a CUDA tensor (no CPU path)")
            if x.dim() != 4 or x.shape[1] != c:
                raise capi.Yb200Error(f"InstanceContextEncoder: {f} has shape {tuple(x.shape)}, expected [B, {c}, H, W]")
        for (fa, a), (fb, b) in zip(zip(self.in_features, xs), zip(self.in_features[1:], xs[1:])):
            if a.shape[0] != b.shape[0] or a.shape[2] != 2 * b.shape[2] or a.shape[3] != 2 * b.shape[3]:
                raise capi.Yb200Error(f"InstanceContextEncoder: {fa} {tuple(a.shape[2:])} must be exactly twice {fb} {tuple(b.shape[2:])} "
                                      "(pad the images to a multiple of 32)")
        return xs[::-1]

    # ---- forward -----------------------------------------------------------------------------------------------------------------
    def forward(self, features):
        """fp32 NCHW [B, NUM_CHANNELS, H, W] at the finest input level.  With autograd recording and an input or a parameter requiring grad,
        the encoder is one autograd node (`_EncoderFn`)"""
        xs = self._check(features)
        params = [p for _, p in self.named_parameters()]
        if torch.is_grad_enabled() and (any(x.requires_grad for x in xs) or any(p.requires_grad for p in params)):
            return _EncoderFn.apply(self, len(xs), *xs, *params)
        with torch.no_grad():
            return self._run(xs)

    def _run(self, xs, save=None):
        """the forward kernels on the inputs coarsest first; `save` (a dict) receives what the backward reads"""
        L, sp = self.L, capi.stream_ptr()
        c, c4 = self.num_channels, self.num_channels // 4
        bf16 = torch.bfloat16
        x = [t.detach().permute(0, 2, 3, 1).to(bf16).contiguous() for t in xs]  # NCHW fp32 -> NHWC bf16 (layout plumbing)
        b, h0, w0, _ = x[0].shape
        dev = x[0].device
        # lateral 0 straight into the PPM's concat (:109), then the pyramid pooling (:56-68)
        cat512 = torch.empty(b, h0, w0, len(PPM_SIZES) * c4 + c, dtype=bf16, device=dev)
        lat0 = capi.act(cat512, len(PPM_SIZES) * c4, c)
        self._affine(capi.act(x[0]), self.fpn_laterals[0], lat0, 1)
        pooled, priors = [], []
        for i, (kh, kw) in enumerate(ppm_windows(h0, w0)):
            ph, pw = h0 // kh, w0 // kw
            rows = b * ph * pw
            pool = torch.zeros(1, 1, _pad16(rows), c, dtype=bf16, device=dev)          # zero rows up to a multiple of 16
            pa = capi.act(pool.view(-1)[:rows * c].view(b, ph, pw, c))
            capi.check(L.yb200_avg_pool2d(ctypes.byref(lat0), kh, kw, ctypes.byref(pa), sp), "ppm pool")
            prior = torch.empty(1, 1, _pad16(rows), c4, dtype=bf16, device=dev)
            self._relu(capi.act(pool), self.ppm.stages[i]._modules["1"], capi.act(prior))
            ra, ca = capi.act(prior.view(-1)[:rows * c4].view(b, ph, pw, c4)), capi.act(cat512, i * c4, c4)
            capi.check(L.yb200_resize_bilinear(ctypes.byref(ra), ctypes.byref(ca), sp), "ppm prior resize")
            pooled.append(pool)
            priors.append(prior)
        prev = torch.empty(b, h0, w0, c, dtype=bf16, device=dev)
        self._relu(capi.act(cat512), self.ppm.bottleneck, capi.act(prev))
        # top-down path (:110-119); the finest level's output goes straight into the fusion's concat
        hf, wf = x[-1].shape[1:3]
        cat768 = torch.empty(b, hf, wf, 3 * c, dtype=bf16, device=dev)
        prevs, outs = [prev], []
        for lvl in range(len(x)):
            if lvl:
                prev = torch.empty(b, *x[lvl].shape[1:3], c, dtype=bf16, device=dev)
                pa = capi.act(prev)
                self._affine(capi.act(x[lvl]), self.fpn_laterals[lvl], pa, 1)
                ca = capi.act(prevs[-1])
                capi.check(L.yb200_upsample_nearest2x_add(ctypes.byref(pa), ctypes.byref(ca), ctypes.byref(pa), sp), "top-down add")
                prevs.append(prev)
            last = lvl == len(x) - 1
            out = cat768 if last else torch.empty_like(prev)
            oa = capi.act(cat768, 0, c) if last else capi.act(out)
            self._affine(capi.act(prev), self.fpn_outputs[lvl], oa, 3)
            outs.append(out)
        # the coarser outputs bilinearly resized to the finest map (:120-125), then fusion (:126)
        for j, lvl in enumerate((1, 0)):
            oa, ca = capi.act(outs[lvl]), capi.act(cat768, (j + 1) * c, c)
            capi.check(L.yb200_resize_bilinear(ctypes.byref(oa), ctypes.byref(ca), sp), "fusion resize")
        y = torch.empty(b, hf, wf, c, dtype=bf16, device=dev)
        self._affine(capi.act(cat768), self.fusion, capi.act(y), 1)
        if save is not None:
            save.update(x=x, cat512=cat512, pooled=pooled, priors=priors, prevs=prevs, outs=outs, cat768=cat768)
        return y.permute(0, 3, 1, 2).float()

    # ---- backward ----------------------------------------------------------------------------------------------------------------
    def _wgrad(self, xa, dza, k, out):
        L = self.L
        ws = torch.empty(max(int(L.yb200_conv2d_wgrad_workspace(ctypes.byref(xa), ctypes.byref(dza), k, 1)), 16), dtype=torch.uint8, device=out.device)
        capi.check(L.yb200_conv2d_wgrad(ctypes.byref(xa), ctypes.byref(dza), k, 1, out.shape[1], capi.ptr(out), 0, capi.ptr(ws), ctypes.c_int64(ws.numel()),
                                        capi.stream_ptr()), "wgrad")
        return out

    def _colsum(self, dza, out):
        ws = torch.empty(max(int(self.L.yb200_colsum_workspace(ctypes.byref(dza))), 16), dtype=torch.uint8, device=out.device)
        capi.check(self.L.yb200_colsum(ctypes.byref(dza), ctypes.c_float(1.0), capi.ptr(out), 0, capi.ptr(ws), capi.stream_ptr()), "colsum")
        return out

    def _conv_grads(self, xa, dza, conv, name, grads, need, k):
        """weight and bias gradients of `conv` (input view xa, output-gradient view dza) for the parameters that require grad"""
        dev = conv.weight.device
        if need[name + ".weight"]:
            grads[name + ".weight"] = self._wgrad(xa, dza, k, torch.empty(conv.weight.shape, device=dev))
        if need[name + ".bias"]:
            grads[name + ".bias"] = self._colsum(dza, torch.empty(conv.bias.shape, device=dev))

    def _dgrad(self, dza, conv, dxa, addend, k):
        capi.check(self.L.yb200_conv2d_dgrad(ctypes.byref(dza), capi.ptr(self._pack(conv.weight, dgrad=True)), ctypes.byref(dxa),
                                             ctypes.byref(addend) if addend is not None else None, k, 1, capi.stream_ptr()), "dgrad")

    def _backward(self, s, g, need_x, need):
        """gradients of the encoder (DESIGN.md par.7): {parameter name: fp32 gradient} for the names with need[name], and d input (fp32 NCHW)
        per level, coarsest first, for the levels with need_x[level] (None for the others)"""
        L, sp = self.L, capi.stream_ptr()
        c, c4 = self.num_channels, self.num_channels // 4
        x, cat512, cat768, prevs, outs = s["x"], s["cat512"], s["cat768"], s["prevs"], s["outs"]
        b, h0, w0, _ = x[0].shape
        bf16 = torch.bfloat16
        grads = {}
        # 1-2. d out (fp32 NCHW) -> bf16 NHWC; fusion: weight / bias gradients, data gradient into d cat768
        dy = g.permute(0, 2, 3, 1).to(bf16).contiguous()
        dya = capi.act(dy)
        self._conv_grads(capi.act(cat768), dya, self.fusion, "fusion", grads, need, 1)
        dcat768 = torch.empty_like(cat768)
        self._dgrad(dya, self.fusion, capi.act(dcat768), None, 1)
        # 3. the resize adjoints of slices 1 and 2: d out1, d out0
        douts = [torch.empty_like(o) for o in outs[:-1]] + [dcat768]          # d out1 / d out0 own buffers; d out2 is a slice of d cat768
        dout_acts = [capi.act(d) for d in douts[:-1]] + [capi.act(dcat768, 0, c)]
        for j, lvl in enumerate((1, 0)):
            sa = capi.act(dcat768, (j + 1) * c, c)
            capi.check(L.yb200_resize_bilinear_bwd(ctypes.byref(sa), None, ctypes.byref(dout_acts[lvl]), sp), "fusion resize bwd")
        # 4-6. the output convolutions, finest first: d prev = dgrad(d out) + the 2x2 sums of the finer level's d prev (masked by the ReLU at
        # level 0, where d prev is the bottleneck's pre-activation gradient)
        dprevs = [None] * len(x)
        for lvl in range(len(x) - 1, -1, -1):
            conv = self.fpn_outputs[lvl]
            pa = capi.act(prevs[lvl])
            self._conv_grads(pa, dout_acts[lvl], conv, f"fpn_outputs.{lvl}", grads, need, 3)
            dp = torch.empty_like(prevs[lvl])
            dpa = capi.act(dp)
            add = None
            if lvl + 1 < len(x):
                addend = torch.empty_like(prevs[lvl])
                add, fa = capi.act(addend), capi.act(dprevs[lvl + 1])
                capi.check(L.yb200_upsample_nearest2x_bwd(ctypes.byref(fa), ctypes.byref(pa) if lvl == 0 else None, ctypes.byref(add), sp), "top-down bwd")
            if lvl == 0:
                capi.check(L.yb200_conv2d_dgrad_relu(ctypes.byref(dout_acts[lvl]), capi.ptr(self._pack(conv.weight, dgrad=True)), ctypes.byref(pa),
                                                     ctypes.byref(dpa), ctypes.byref(add) if add is not None else None, 3, 1, sp), "dgrad + relu bwd")
            else:
                self._dgrad(dout_acts[lvl], conv, dpa, add, 3)
            dprevs[lvl] = dp
        # 7. bottleneck: gradients, data gradient into d cat512
        dza = capi.act(dprevs[0])
        self._conv_grads(capi.act(cat512), dza, self.ppm.bottleneck, "ppm.bottleneck", grads, need, 1)
        dcat512 = torch.empty_like(cat512)
        self._dgrad(dza, self.ppm.bottleneck, capi.act(dcat512), None, 1)
        # 8. per stage: masked resize adjoint = the stage conv's pre-activation gradient; its gradients and d pooled
        dpooled, keep = [], []  # keep: the d pooled buffers stay allocated until the input-gradient kernel has read them
        windows = ppm_windows(h0, w0)
        for i, (kh, kw) in enumerate(windows):
            ph, pw = h0 // kh, w0 // kw
            rows = b * ph * pw
            pool, prior = s["pooled"][i], s["priors"][i]
            conv = self.ppm.stages[i]._modules["1"]
            dz = torch.zeros_like(prior)                                                 # padded rows stay zero
            sa, ha = capi.act(dcat512, i * c4, c4), capi.act(prior.view(-1)[:rows * c4].view(b, ph, pw, c4))
            da = capi.act(dz.view(-1)[:rows * c4].view(b, ph, pw, c4))
            capi.check(L.yb200_resize_bilinear_bwd(ctypes.byref(sa), ctypes.byref(ha), ctypes.byref(da), sp), "ppm prior resize bwd")
            za = capi.act(dz)
            self._conv_grads(capi.act(pool), za, conv, f"ppm.stages.{i}.1", grads, need, 1)
            dp = torch.empty_like(pool)
            self._dgrad(za, conv, capi.act(dp), None, 1)
            keep.append(dp)
            dpooled.append(capi.act(dp.view(-1)[:rows * c].view(b, ph, pw, c)))
        # 9. d lat0 = d cat512[..., C:2C] + the pools' adjoints, one launch
        dlat0 = torch.empty(b, h0, w0, c, dtype=bf16, device=cat512.device)
        la, ca = capi.act(dlat0), capi.act(dcat512, len(windows) * c4, c)
        views = (capi.Act * len(dpooled))(*dpooled)
        khw = (ctypes.c_int32 * (2 * len(windows)))(*[v for kk in windows for v in kk])
        capi.check(L.yb200_ppm_input_grad(ctypes.byref(ca), views, khw, len(windows), ctypes.byref(la), sp), "ppm input grad")
        # 10. laterals: gradients, and d input only for the inputs that require grad
        dlats = [dlat0] + dprevs[1:]
        dxs = [None] * len(x)
        for lvl, (xl, dl) in enumerate(zip(x, dlats)):
            conv = self.fpn_laterals[lvl]
            xa, dla = capi.act(xl), capi.act(dl)
            self._conv_grads(xa, dla, conv, f"fpn_laterals.{lvl}", grads, need, 1)
            if need_x[lvl]:
                dx = torch.empty_like(xl)
                self._dgrad(dla, conv, capi.act(dx), None, 1)
                dxs[lvl] = dx.permute(0, 3, 1, 2).float()
        return grads, dxs


class _EncoderFn(torch.autograd.Function):
    """one InstanceContextEncoder as one autograd node: args (encoder, number of levels, *inputs coarsest first, *parameters in
    named_parameters() order) -> the fp32 NCHW output; the backward returns d inputs (fp32 NCHW) and every parameter's fp32 gradient"""

    @staticmethod
    def forward(ctx, enc, nlev, *args):
        saved = {}
        out = enc._run(list(args[:nlev]), saved)
        ctx.enc, ctx.nlev, ctx.saved = enc, nlev, saved
        return out

    @staticmethod
    def backward(ctx, g):
        enc, nlev = ctx.enc, ctx.nlev
        names = [n for n, _ in enc.named_parameters()]
        need = dict(zip(names, ctx.needs_input_grad[2 + nlev:]))
        grads, dxs = enc._backward(ctx.saved, g.float(), ctx.needs_input_grad[2:2 + nlev], need)
        ctx.saved = None
        return (None, None) + tuple(dxs) + tuple(grads.get(n) for n in names)


def _register():
    try:
        from detectron2.utils.registry import Registry  # noqa: F401  pragma: no cover
    except Exception:  # noqa: BLE001
        return
    try:  # pragma: no cover
        from yolov7.modeling.transcoders.encoder_sparseinst import SPARSE_INST_ENCODER_REGISTRY
        SPARSE_INST_ENCODER_REGISTRY._obj_map["InstanceContextEncoder"] = InstanceContextEncoder
    except Exception:  # noqa: BLE001
        pass


_register()
