"""Static execution plan of the YOLOX hot path on one H100: every tensor of the forward and backward pass is
allocated once (NHWC bf16 activations, concat buffers addressed through channel-slice views, fp32 flat parameter /
gradient buffers) and a step is a fixed sequence of C-ABI kernel launches -- capturable in a CUDA graph.

Structure follows the reference (CSPDarknet darknetx.py:103-177, YOLOPAFPN yolo_pafpn.py:79-114, YOLOXHead
yolox_head.py:151-245) with three fusions the reference cannot express:
  * the two 1x1 convolutions of every CSPLayer (conv1, conv2: wrappers.py:194-195) and the first cls/reg 3x3
    convolutions of the head (yolox_head.py:160-168) read the same input and run as ONE GEMM;
  * torch.cat / nn.Upsample / Focus never materialise: producers write into channel slices of the consumer's buffer;
  * the three prediction convolutions write the [B, A, 85] head output directly.
There is no PyTorch fallback: every op is a libyb200.so call.
"""
import ctypes
import math
import os

import torch

from . import capi

BN_EPS = 1e-3       # yolox.py:85-90
BN_MOMENTUM = 0.03
STRIDES = (8, 16, 32)


def _ceil(a, b):
    return (a + b - 1) // b * b


class Buf:
    """NHWC bf16 activation buffer (+ lazily allocated gradient of the same shape)"""

    def __init__(self, name, n, h, w, c, device, dtype=torch.bfloat16, split=0):
        self.name, self.n, self.h, self.w, self.c = name, n, h, w, c
        # split (strict mode): `split` bf16 planes of c channels each in one NHWC tensor, value = their sum (csrc/strict.cu); views address
        # plane 0, plane j sits j * self.lo channels further
        self.lo = c if split else 0
        self.planes = split if split else 1
        self.t = torch.zeros(n, h, w, self.planes * c, dtype=dtype, device=device)
        self.g = None
        self.written = []  # channel ranges of .g already produced in the current backward pass

    def view(self, off=0, c=None):
        return View(self, off, self.c - off if c is None else c)

    def grad(self):
        if self.g is None:
            self.g = torch.zeros_like(self.t)
        return self.g


class View:
    def __init__(self, buf, off, c):
        self.buf, self.off, self.c = buf, off, c
        self._act = None
        self._gact = None

    def act(self):
        if self._act is None:
            self._act = capi.act(self.buf.t, self.off, self.c)
        return ctypes.byref(self._act)

    def gact(self):
        if self._gact is None:
            self._gact = capi.act(self.buf.grad(), self.off, self.c)
        return ctypes.byref(self._gact)

    @property
    def shape(self):
        return (self.buf.n, self.buf.h, self.buf.w, self.c)

    def tensor(self):
        return self.buf.t[..., self.off:self.off + self.c]

    def value(self):
        """fp32 value of the view (split buffers: hi + lo)"""
        v = self.tensor().float()
        for j in range(1, self.buf.planes):
            v = v + self.buf.t[..., j * self.buf.lo + self.off:j * self.buf.lo + self.off + self.c].float()
        return v

    def grad_tensor(self):
        return self.buf.grad()[..., self.off:self.off + self.c]


class BnHead:
    """one BatchNorm+SiLU of a (possibly merged) convolution: channel range [c0, c0+c) of the GEMM output"""

    def __init__(self, prefix, c0, c, out, residual=None, up=None):
        self.prefix, self.c0, self.c, self.out, self.residual, self.up = prefix, c0, c, out, residual, up


class ConvOp:
    def __init__(self, prefixes, x, z, heads, ksize, stride, cin_real):
        self.prefixes, self.x, self.z, self.heads = prefixes, x, z, heads
        self.ksize, self.stride, self.cin_real = ksize, stride, cin_real
        self.cin_pad, self.cout = x.c, z.c
        self.first = False  # no data gradient needed (network input)


class PredOp:
    """prediction 1x1 convolutions of one level: cls (C) and reg+obj (5), bias, fp32 output into [B, A, 5+C]"""

    def __init__(self, level, cls_feat, reg_feat):
        self.level, self.cls_feat, self.reg_feat = level, cls_feat, reg_feat


class SppOp:
    def __init__(self, views, arg):
        self.views, self.arg = views, arg


class YoloxEngine:
    def __init__(self, batch, height, width, num_classes=80, width_mul=0.5, depth_mul=0.33, max_gt=100, device="cuda", share_params_of=None,
                 strict=None):
        """strict=True (default: environment YB200_STRICT=1): forward pass in split-bf16 / fp32 arithmetic (csrc/strict.cu) for the
        1e-3 parity check against the fp32 reference; forward + SimOTA + losses only, no backward."""
        assert height % 32 == 0 and width % 32 == 0, "input must be padded to a multiple of 32 (yolox.py:100-101)"
        self.strict = (os.environ.get("YB200_STRICT", "0") == "1") if strict is None else bool(strict)
        self.group4 = os.environ.get("YB200_STEM_GROUP4", "1") == "1" and not self.strict and (width // 2) % 4 == 0
        self.planes = int(os.environ.get("YB200_STRICT_PLANES", "3"))  # bf16 planes per value in strict mode: 3 = all 24 bits of fp32, 2 = 16 bits
        assert self.planes in (2, 3)
        self.L = capi.lib()
        self.dev = torch.device(device)
        self.n, self.h, self.w, self.nc, self.max_gt = batch, height, width, num_classes, max_gt
        self.wm, self.dm = width_mul, depth_mul
        self.pad_value = 114.0  # cfg.MODEL.PADDED_VALUE; YOLOX sets it per plan (modeling.py)
        self.ops = []
        self.bufs = {}
        self.param_specs = []   # (name, shape) in flat order
        self._build()
        self._alloc_params(share_params_of)
        self._alloc_runtime()

    # ------------------------------------------------------------------ graph construction
    def _buf(self, name, h, w, c, dtype=torch.bfloat16):
        if self.strict and dtype == torch.float16:
            dtype = torch.float32  # pre-BatchNorm conv outputs stay fp32 in strict mode
        b = Buf(name, self.n, h, w, c, self.dev, dtype, split=self.planes if (self.strict and dtype == torch.bfloat16) else 0)
        self.bufs[name] = b
        return b

    def _conv(self, prefixes, x, couts, k, s, outs=None, residuals=None, ups=None, cin_real=None):
        n, h, w, _ = x.shape
        oh, ow = h // s, w // s
        ctot = sum(couts)
        z = self._buf(prefixes[0] + ".z", oh, ow, ctot, torch.float16)  # pre-BN conv output: fp16 (conv_gemm.cuh)
        heads, res = [], []
        c0 = 0
        for i, (p, c) in enumerate(zip(prefixes, couts)):
            out = outs[i] if outs and outs[i] is not None else self._buf(p + ".a", oh, ow, c).view()
            assert out.shape == (n, oh, ow, c), (p, out.shape, (n, oh, ow, c))
            heads.append(BnHead(p, c0, c, out, residuals[i] if residuals else None, ups[i] if ups else None))
            res.append(out)
            c0 += c
        op = ConvOp(prefixes, x, z.view(), heads, k, s, cin_real or x.c)
        self.ops.append(op)
        cin = op.cin_real
        for p, c in zip(prefixes, couts):
            self.param_specs.append((p + ".conv.weight", (c, cin, k, k)))
        return res

    def _csp(self, prefix, x, cout, n, shortcut, out=None):
        hdn = cout // 2
        _, h, w, _ = x.shape
        cat = self._buf(prefix + ".cat", h, w, 2 * hdn)
        y, _ = self._conv([prefix + ".conv1", prefix + ".conv2"], x, [hdn, hdn], 1, 1, outs=[None, cat.view(hdn, hdn)])
        for i in range(n):
            (t,) = self._conv([f"{prefix}.m.{i}.conv1"], y, [hdn], 1, 1)
            (y,) = self._conv([f"{prefix}.m.{i}.conv2"], t, [hdn], 3, 1, outs=[cat.view(0, hdn) if i == n - 1 else None],
                              residuals=[y if shortcut else None])
        (o,) = self._conv([prefix + ".conv3"], cat.view(), [cout], 1, 1, outs=[out])
        return o

    def _build(self):
        bc = int(self.wm * 64)
        bd = max(round(self.dm * 3), 1)
        nn_ = round(3 * self.dm)
        H, W = self.h, self.w
        c3, c4, c5 = bc * 4, bc * 8, bc * 16
        focus = self._buf("focus", H // 2, W // 2, 16)
        self.focus = focus
        # concat buffers of the neck; backbone / neck producers write straight into their slices
        cat_p4 = self._buf("neck.cat_p4", H // 16, W // 16, 2 * c4)   # [up(fpn_out0) | dark4]
        cat_p3 = self._buf("neck.cat_p3", H // 8, W // 8, 2 * c3)     # [up(fpn_out1) | dark3]
        cat_n3 = self._buf("neck.cat_n3", H // 16, W // 16, 2 * c3)   # [bu_conv2     | fpn_out1]
        cat_n4 = self._buf("neck.cat_n4", H // 32, W // 32, 2 * c4)   # [bu_conv1     | fpn_out0]
        (x,) = self._conv(["backbone.stem.conv"], focus.view(), [bc], 3, 1, cin_real=12)
        self.ops[-1].first = True
        (x,) = self._conv(["backbone.dark2.0"], x, [bc * 2], 3, 2)
        x = self._csp("backbone.dark2.1", x, bc * 2, bd, True)
        d2 = x
        (x,) = self._conv(["backbone.dark3.0"], x, [c3], 3, 2)
        d3 = self._csp("backbone.dark3.1", x, c3, bd * 3, True, out=cat_p3.view(c3, c3))
        (x,) = self._conv(["backbone.dark4.0"], d3, [c4], 3, 2)
        d4 = self._csp("backbone.dark4.1", x, c4, bd * 3, True, out=cat_p4.view(c4, c4))
        (x,) = self._conv(["backbone.dark5.0"], d4, [c5], 3, 2)
        spp_cat = self._buf("backbone.dark5.1.cat", H // 32, W // 32, 4 * c4)
        self._conv(["backbone.dark5.1.conv1"], x, [c4], 1, 1, outs=[spp_cat.view(0, c4)])
        arg = torch.empty(3, self.n, H // 32, W // 32, c4, dtype=torch.uint8, device=self.dev)
        self.ops.append(SppOp([spp_cat.view(i * c4, c4) for i in range(4)], arg))
        (x,) = self._conv(["backbone.dark5.1.conv2"], spp_cat.view(), [c5], 1, 1)
        d5 = self._csp("backbone.dark5.2", x, c5, bd, False)
        self.features = {"dark2": d2, "dark3": d3, "dark4": d4, "dark5": d5}  # CSPDarknet.forward outputs (darknetx.py:165-177)
        n_backbone = len(self.ops)
        # neck (yolo_pafpn.py:79-114)
        self._conv(["neck.lateral_conv0"], d5, [c4], 1, 1, outs=[cat_n4.view(c4, c4)], ups=[cat_p4.view(0, c4)])
        f_out0 = self._csp("neck.C3_p4", cat_p4.view(), c4, nn_, False)
        self._conv(["neck.reduce_conv1"], f_out0, [c3], 1, 1, outs=[cat_n3.view(c3, c3)], ups=[cat_p3.view(0, c3)])
        pan2 = self._csp("neck.C3_p3", cat_p3.view(), c3, nn_, False)
        self._conv(["neck.bu_conv2"], pan2, [c3], 3, 2, outs=[cat_n3.view(0, c3)])
        pan1 = self._csp("neck.C3_n3", cat_n3.view(), c4, nn_, False)
        self._conv(["neck.bu_conv1"], pan1, [c4], 3, 2, outs=[cat_n4.view(0, c4)])
        pan0 = self._csp("neck.C3_n4", cat_n4.view(), c5, nn_, False)
        self.pan = (pan2, pan1, pan0)  # YOLOPAFPN.forward outputs (yolo_pafpn.py:113-114)
        n_neck = len(self.ops)
        # head (yolox_head.py:151-175)
        hc = int(256 * self.wm)
        self.levels = []
        a_off = 0
        for k, f in enumerate((pan2, pan1, pan0)):
            _, fh, fw, _ = f.shape
            (x,) = self._conv([f"head.stems.{k}"], f, [hc], 1, 1)
            cr = self._buf(f"head.cr0.{k}", fh, fw, 2 * hc)
            self._conv([f"head.cls_convs.{k}.0", f"head.reg_convs.{k}.0"], x, [hc, hc], 3, 1, outs=[cr.view(0, hc), cr.view(hc, hc)])
            (cf,) = self._conv([f"head.cls_convs.{k}.1"], cr.view(0, hc), [hc], 3, 1)
            (rf,) = self._conv([f"head.reg_convs.{k}.1"], cr.view(hc, hc), [hc], 3, 1)
            self.ops.append(PredOp(k, cf, rf))
            self.param_specs += [(f"head.cls_preds.{k}.weight", (self.nc, hc, 1, 1)), (f"head.reg_preds.{k}.weight", (4, hc, 1, 1)),
                                 (f"head.obj_preds.{k}.weight", (1, hc, 1, 1))]
            self.levels.append((fh, fw, STRIDES[k], a_off))
            a_off += fh * fw
        self.num_anchors = a_off
        self.hc = hc
        self.ranges = {"backbone": (0, n_backbone), "neck": (n_backbone, n_neck), "head": (n_neck, len(self.ops))}  # op index ranges

    # ------------------------------------------------------------------ parameters
    def _alloc_params(self, share=None):
        """flat fp32 parameter / gradient buffers; the tensors in self.params / self.grads are views into them
        (`share`: another engine of the same architecture whose parameter storage is reused -- one set of weights, one
        plan per input shape).
        Layout: [conv + pred weights in op order][pad][bn gamma | bn beta per op][pred biases]; merged convolutions
        are adjacent so one packing / one weight-gradient launch covers them."""
        dev = self.dev
        specs = list(self.param_specs)
        for op in self.ops:
            if isinstance(op, ConvOp):
                for hd in op.heads:
                    specs.append((hd.prefix + ".bn.weight", (hd.c,)))
                for hd in op.heads:
                    specs.append((hd.prefix + ".bn.bias", (hd.c,)))
        for k in range(len(self.levels)):
            specs += [(f"head.cls_preds.{k}.bias", (self.nc,)), (f"head.reg_preds.{k}.bias", (4,)), (f"head.obj_preds.{k}.bias", (1,))]
        offs, total = {}, 0
        for name, shape in specs:
            if name.startswith("head.reg_preds") and name.endswith(".weight"):
                total = _ceil(total, 4)
            offs[name] = total
            total += math.prod(shape)
            if name.startswith("head.obj_preds") and name.endswith(".weight"):
                total += 11 * shape[1]  # room for the 16-row (padded) weight-gradient tile of reg+obj
            total = _ceil(total, 4)  # 16-byte alignment of every tensor
        if share is not None:
            assert share.flat_param.numel() == total and share.param_names == [n for n, _ in specs], "architectures differ"
        self.flat_param = share.flat_param if share is not None else torch.zeros(total, dtype=torch.float32, device=dev)
        self.flat_grad = share.flat_grad if share is not None else torch.zeros(total, dtype=torch.float32, device=dev)
        self.params, self.grads = {}, {}
        for name, shape in specs:
            n = math.prod(shape)
            self.params[name] = self.flat_param[offs[name]:offs[name] + n].view(shape)
            self.grads[name] = self.flat_grad[offs[name]:offs[name] + n].view(shape)
        self.param_names = [n for n, _ in specs]
        self.param_layout = [(n, offs[n], math.prod(shape)) for n, shape in specs]  # (name, element offset, numel); gaps are padding
        # BatchNorm buffers
        nbn = sum(hd.c for op in self.ops if isinstance(op, ConvOp) for hd in op.heads)
        self.flat_rm = share.flat_rm if share is not None else torch.zeros(nbn, device=dev)
        self.flat_rv = share.flat_rv if share is not None else torch.ones(nbn, device=dev)
        self.flat_scale = torch.empty(nbn, device=dev)
        self.flat_shift = torch.empty(nbn, device=dev)
        self.flat_mean = torch.empty(nbn, device=dev)
        self.flat_invstd = torch.empty(nbn, device=dev)
        self.flat_stats = torch.zeros(4 * nbn, dtype=torch.float64, device=dev)  # sum | sqsum | dgamma acc | dbeta acc
        self.buffers = {}
        nbt = []
        o = 0
        for op in self.ops:
            if not isinstance(op, ConvOp):
                continue
            op.bn_off = o
            for hd in op.heads:
                self.buffers[hd.prefix + ".bn.running_mean"] = self.flat_rm[o:o + hd.c]
                self.buffers[hd.prefix + ".bn.running_var"] = self.flat_rv[o:o + hd.c]
                nbt.append(hd.prefix + ".bn.num_batches_tracked")
                hd.bn_off = o
                o += hd.c
        self.nbn = nbn
        # destination of every BatchNorm channel's weight / bias gradient in the flat gradient buffer (yb200_bn_param_grads: one launch per range)
        g_off, b_off = torch.empty(nbn, dtype=torch.int32), torch.empty(nbn, dtype=torch.int32)
        for op in self.ops:
            if isinstance(op, ConvOp):
                for hd in op.heads:
                    for dst, leaf in ((g_off, ".bn.weight"), (b_off, ".bn.bias")):
                        base = (self.grads[hd.prefix + leaf].data_ptr() - self.flat_grad.data_ptr()) // 4
                        dst[hd.bn_off:hd.bn_off + hd.c] = torch.arange(base, base + hd.c, dtype=torch.int32)
        self.bn_goff, self.bn_boff = g_off.to(dev), b_off.to(dev)
        self.flat_nbt = share.flat_nbt if share is not None else torch.zeros(len(nbt), dtype=torch.int64, device=dev)
        for i, name in enumerate(nbt):
            self.buffers[name] = self.flat_nbt[i]
        # packed bf16 operands
        for op in self.ops:
            if isinstance(op, ConvOp):
                kk = op.ksize * op.ksize
                if self.strict:
                    op.w_split = torch.empty(op.cout, self.planes, kk, op.cin_pad, dtype=torch.bfloat16, device=dev)
                    op.w_fwd = op.w_dgrad = None
                elif op.first and self.group4:
                    # Stem on a pixel-grouped view (yb200_conv2d_fwd_fold): 4 horizontally adjacent Focus pixels = one pixel of 64 channels
                    # (128-byte rows for TMA instead of 32-byte ones), 4 x 32 output columns.  Expanded weight W'[(e, c)][(f, ci)][kh][t]:
                    # output pixel 4j+e reads input pixel 4(j+t-1)+f through the original tap kw = 4(t-1) + f - e + 1 when 0 <= kw <= 2.
                    g, co, ci_pad, ci_real = 4, op.cout, op.cin_pad, op.cin_real
                    idx = torch.zeros(g * co, g * ci_pad, 3, 3, dtype=torch.int64)
                    msk = torch.zeros(g * co, g * ci_pad, 3, 3)
                    for e in range(g):
                        for f in range(g):
                            for t in range(3):
                                kw = 4 * (t - 1) + f - e + 1
                                if 0 <= kw <= 2:
                                    c_i, ci_i, kh_i = torch.meshgrid(torch.arange(co), torch.arange(ci_real), torch.arange(3), indexing="ij")
                                    idx[e * co:(e + 1) * co, f * ci_pad:f * ci_pad + ci_real, :, t] = ((c_i * ci_real + ci_i) * 3 + kh_i) * 3 + kw
                                    msk[e * co:(e + 1) * co, f * ci_pad:f * ci_pad + ci_real, :, t] = 1.0
                    op.exp_idx, op.exp_mask = idx.to(dev), msk.to(dev)
                    valid = torch.nonzero(msk.flatten()).flatten()                      # positions of W' that map to a real weight
                    target = idx.flatten()[valid]                                         # ... and the flat index of that weight
                    # every real weight appears once per output pixel e of the group: row w of fold_pos lists the g positions of weight w in
                    # ascending order, so the fold is a fixed-order sum (an index_add_ adds them with atomics, in an order that varies run to run)
                    order = torch.sort(target, stable=True).indices
                    assert torch.equal(target[order], torch.arange(co * ci_real * 9).repeat_interleave(g)), "stem expansion"
                    op.fold_pos = valid[order].to(dev)
                    op.fold_parts = torch.empty(co * ci_real * 9, g, device=dev)  # gathered once per step; allocated here, not on the side stream
                    op.w_exp = torch.zeros(g * co, g * ci_pad, 3, 3, device=dev)         # fp32 OIHW of the grouped convolution
                    op.g_exp = torch.zeros_like(op.w_exp)
                    op.w_fwd = torch.empty(g * co, kk, g * ci_pad, dtype=torch.bfloat16, device=dev)
                    op.w_dgrad = None
                else:
                    op.w_fwd = torch.empty(op.cout, kk, op.cin_pad, dtype=torch.bfloat16, device=dev)
                    op.w_dgrad = None if op.first else torch.empty(op.cin_pad, kk, op.cout, dtype=torch.bfloat16, device=dev)
                op.w_src = self.params[op.prefixes[0] + ".conv.weight"]
                op.g_dst = self.grads[op.prefixes[0] + ".conv.weight"]
            elif isinstance(op, PredOp):
                k, hc = op.level, self.hc
                if self.strict:
                    op.wc_split = torch.empty(self.nc, self.planes, 1, hc, dtype=torch.bfloat16, device=dev)
                    op.wr_split = torch.empty(16, self.planes, 1, hc, dtype=torch.bfloat16, device=dev)
                op.wc_fwd = torch.empty(self.nc, 1, hc, dtype=torch.bfloat16, device=dev)
                op.wc_dgrad = torch.empty(hc, 1, self.nc, dtype=torch.bfloat16, device=dev)
                op.wr_fwd = torch.empty(16, 1, hc, dtype=torch.bfloat16, device=dev)
                op.wr_dgrad = torch.empty(hc, 1, 16, dtype=torch.bfloat16, device=dev)
                op.wc_src, op.wr_src = self.params[f"head.cls_preds.{k}.weight"], self.params[f"head.reg_preds.{k}.weight"]
                op.gc_dst, op.gr_dst = self.grads[f"head.cls_preds.{k}.weight"], self.grads[f"head.reg_preds.{k}.weight"]
                op.bc, op.br = self.params[f"head.cls_preds.{k}.bias"], self.params[f"head.reg_preds.{k}.bias"]
                assert self.params[f"head.obj_preds.{k}.weight"].data_ptr() == op.wr_src.data_ptr() + 4 * 4 * hc
                assert self.params[f"head.obj_preds.{k}.bias"].data_ptr() == op.br.data_ptr() + 16

    def init_weights(self, seed=0):
        """reference default initialisation (nn.Conv2d kaiming-uniform a=sqrt(5); BN 1/0; prior biases, yolox_head.py:140-149)"""
        g = torch.Generator().manual_seed(seed)
        for name, p in self.params.items():
            if name.endswith(".bn.weight"):
                p.fill_(1.0)
            elif name.endswith(".bias") and "preds" in name:
                p.fill_(-math.log((1 - 1e-2) / 1e-2) if ("cls_preds" in name or "obj_preds" in name) else 0.0)
            elif name.endswith(".bn.bias"):
                p.zero_()
            else:
                fan_in = p.shape[1] * p.shape[2] * p.shape[3]
                p.copy_(((torch.rand(p.shape, generator=g) * 2 - 1) / math.sqrt(fan_in)).to(self.dev))
        self.flat_rm.zero_()
        self.flat_rv.fill_(1.0)
        self.flat_nbt.zero_()

    def load_state_dict(self, sd):
        """copy a reference-layout state_dict (fp32 OIHW weights, BN tensors, prediction biases) into the flat buffers"""
        missing = []
        for name, dst in list(self.params.items()) + list(self.buffers.items()):
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

    # ------------------------------------------------------------------ runtime buffers
    def _alloc_runtime(self):
        dev, n, a, ch = self.dev, self.n, self.num_anchors, 5 + self.nc
        self.outputs = torch.zeros(n, a, ch, device=dev)
        self.labels = torch.zeros(n, self.max_gt, 5, device=dev)
        self.lv = (ctypes.c_int32 * (3 * len(self.levels)))(*[v for (h, w, s, _) in self.levels for v in (h, w, s)])
        self.simota_ws = torch.empty(self.L.yb200_simota_workspace(n, a), dtype=torch.uint8, device=dev)
        self.num_gt = torch.zeros(n, dtype=torch.int32, device=dev)
        self.fg_mask = torch.zeros(n, a, dtype=torch.uint8, device=dev)
        self.matched_gt = torch.zeros(n, a, dtype=torch.int32, device=dev)
        self.matched_iou = torch.zeros(n, a, device=dev)
        self.matched_cls = torch.zeros(n, a, dtype=torch.int32, device=dev)
        self.num_fg_img = torch.zeros(n, dtype=torch.int32, device=dev)
        self.totals = torch.zeros(2, dtype=torch.int32, device=dev)
        self.loss_acc = torch.zeros(4, dtype=torch.float64, device=dev)
        self.losses = torch.zeros(6, device=dev)
        self.loss_weights = torch.tensor([5.0, 1.0, 1.0, 1.0], device=dev)  # d objective / d (loss_iou, loss_obj, loss_cls, loss_l1)
        self.use_l1 = False       # YOLOXHead.use_l1 (yolox_head.py:131): the L1 term on the raw regression outputs, switched on late in training
        self.raw_reg = None       # [B, A, 4] fp32 `origin_preds`, allocated on first use
        self.bias_acc = torch.zeros(len(self.levels), ch, dtype=torch.float64, device=dev)
        self.d_cls = [torch.zeros(n, h, w, self.nc, dtype=torch.bfloat16, device=dev) for (h, w, _, _) in self.levels]
        self.d_ro = [torch.zeros(n, h, w, 16, dtype=torch.bfloat16, device=dev) for (h, w, _, _) in self.levels]
        self.p_dcls = (ctypes.c_void_p * len(self.levels))(*[t.data_ptr() for t in self.d_cls])
        self.p_dro = (ctypes.c_void_p * len(self.levels))(*[t.data_ptr() for t in self.d_ro])
        self.images_u8 = torch.zeros(n, 3, self.h, self.w, dtype=torch.uint8, device=dev)
        self.hw_valid = torch.tensor([[self.h, self.w]] * n, dtype=torch.int32, device=dev)
        self.ws_bytes = 0
        self.ws = None
        self.spp_scratch = None
        self._dz = {}
        self.kernel_launches = 0
        self.overlap_wgrad = True
        self._side = torch.cuda.Stream(device=dev)
        self._fork_evt = torch.cuda.Event()
        self.trace = None  # set to [] to record (label, launches) per call for tools/summarize_launches.py
        self._ev = None    # profile_step(): (label, class, launches, bytes, flops, event) per call
        self._pack_table = None

    def _count(self, k=1, label=None, cls=None, nbytes=0.0, flops=0.0):
        """k = number of kernels the preceding C-ABI call(s) launched (memsets excluded); label feeds the per-layer profile.
        cls / nbytes / flops: kernel class and ALGORITHMIC bytes / FLOPs of the call (what an ideal fused implementation must move /
        compute: every tensor read or written once, 16-bit activations) -- the numerators of bench.py's roofline."""
        self.kernel_launches += k
        if self.trace is not None:
            self.trace.append((label or "?", k))
        if self._ev is not None:
            ev = torch.cuda.Event(enable_timing=True)
            ev.record()
            self._ev.append((label or "?", cls or "other", k, float(nbytes), float(flops), ev))

    def _alg_conv(self, op):
        n, h, w, _ = op.x.shape
        oh, ow = h // op.stride, w // op.stride
        kk = op.ksize * op.ksize
        nbytes = 2.0 * n * (h * w * op.cin_pad + oh * ow * op.cout) + 2.0 * op.cout * kk * op.cin_pad
        return nbytes, 2.0 * n * oh * ow * op.cout * op.cin_real * kk

    def profile_step(self, reps=3):
        """Warm CUDA-event duration of every C-ABI call of one training step: eager launches on the current stream with the weight
        gradients serialised on it (no side stream), an event after each call, median over `reps` steps.  Returns a list of dicts
        (label, cls, launches, bytes, flops, ms).  Tiny kernels include the launch gap in front of them."""
        import statistics
        saved = self.overlap_wgrad
        self.overlap_wgrad = False
        runs = []
        try:
            self.train_step()
            for _ in range(reps):
                torch.cuda.synchronize()
                self._ev = []
                start = torch.cuda.Event(enable_timing=True)
                start.record()
                self.train_step()
                torch.cuda.synchronize()
                prev, row = start, []
                for label, cls, k, nb, fl, ev in self._ev:
                    row.append((label, cls, k, nb, fl, prev.elapsed_time(ev)))
                    prev = ev
                runs.append(row)
        finally:
            self._ev = None
            self.overlap_wgrad = saved
        out = []
        for i, (label, cls, k, nb, fl, _) in enumerate(runs[0]):
            out.append(dict(label=label, cls=cls, launches=k, bytes=nb, flops=fl, ms=statistics.median(r[i][5] for r in runs)))
        return out

    @staticmethod
    def _desc(op):
        n, h, w, _ = op.x.shape
        return "%dx%dx%dx%d->%d k%d s%d" % (n, h, w, op.cin_pad, op.cout, op.ksize, op.stride)

    def _ensure_ws(self, nbytes):
        if nbytes > self.ws_bytes:
            self._side.synchronize()  # the side stream may still be reading the old workspace (first step only)
            self.ws = torch.empty(nbytes, dtype=torch.uint8, device=self.dev)
            self.ws.record_stream(self._side)
            self.ws_bytes = nbytes

    # ------------------------------------------------------------------ forward
    def pack_weights(self):
        L, sp = self.L, capi.stream_ptr()
        if self.strict:
            for op in self.ops:
                if isinstance(op, ConvOp):
                    capi.check(L.yb200_pack_conv_weight_split(capi.ptr(op.w_src), op.cout, op.cin_real, op.ksize, op.cout, op.cin_pad, self.planes,
                                                              capi.ptr(op.w_split), sp), "pack split")
                    self._count(1, "pack split " + op.prefixes[0])
                elif isinstance(op, PredOp):
                    capi.check(L.yb200_pack_conv_weight_split(capi.ptr(op.wc_src), self.nc, self.hc, 1, self.nc, self.hc, self.planes, capi.ptr(op.wc_split), sp), "pack cls")
                    capi.check(L.yb200_pack_conv_weight_split(capi.ptr(op.wr_src), 5, self.hc, 1, 16, self.hc, self.planes, capi.ptr(op.wr_split), sp), "pack reg+obj")
                    self._count(2, "pack split preds")
            return
        if self._pack_table is None:
            # one launch for every layer of the plan: the layer table lives in device memory (built once; the pointers are plan constants)
            rows = []
            for op in self.ops:
                if isinstance(op, ConvOp) and op.first and self.group4:
                    rows.append((op.w_exp, op.w_fwd, None, 4 * op.cout, 4 * op.cin_pad, 3, 4 * op.cout, 4 * op.cin_pad))
                elif isinstance(op, ConvOp):
                    rows.append((op.w_src, op.w_fwd, op.w_dgrad, op.cout, op.cin_real, op.ksize, op.cout, op.cin_pad))
                elif isinstance(op, PredOp):
                    rows.append((op.wc_src, op.wc_fwd, op.wc_dgrad, self.nc, self.hc, 1, self.nc, self.hc))
                    rows.append((op.wr_src, op.wr_fwd, op.wr_dgrad, 5, self.hc, 1, 16, self.hc))
            arr = (capi.PackDesc * len(rows))()
            prefix = [0]
            for d, (src, wf, wd, cout, cin, k, cop, cip) in zip(arr, rows):
                d.w_oihw, d.w_fwd, d.w_dgrad = src.data_ptr(), wf.data_ptr(), (wd.data_ptr() if wd is not None else None)
                d.cout, d.cin, d.ksize, d.cout_pad, d.cin_pad = cout, cin, k, cop, cip
                prefix.append(prefix[-1] + cop * k * k * cip)
            raw = torch.frombuffer(bytearray(bytes(arr)), dtype=torch.uint8).to(self.dev)
            self._pack_table = (raw, torch.tensor(prefix, dtype=torch.int64, device=self.dev), len(rows), prefix[-1],
                                4.0 * sum(r[0].numel() for r in rows) + 2.0 * sum(prefix[-1:]) * 2)
        raw, prefix, n, total, nbytes = self._pack_table
        if self.group4:  # refresh the expanded stem weights from the parameter (two tiny torch kernels)
            st = self.ops[0]
            torch.mul(st.w_src.reshape(-1)[st.exp_idx], st.exp_mask, out=st.w_exp)
            self._count(2, "expand stem weights (torch gather, mul)", "pack_weights")
        capi.check(L.yb200_pack_conv_weights_batched(capi.ptr(raw), capi.ptr(prefix), n, ctypes.c_int64(total), sp), "pack weights")
        self._count(1, "pack all weights", "pack_weights", nbytes)

    def preprocess(self):
        """images_u8 [N,3,H,W] (device) -> focus buffer"""
        capi.check(self.L.yb200_preprocess_focus(capi.ptr(self.images_u8), self.n, self.h, self.w, capi.ptr(self.hw_valid), ctypes.c_float(self.pad_value),
                                                 self.focus.view().act(), capi.stream_ptr()), "preprocess_focus")
        self._count(1, "preprocess", "preprocess_focus", self.n * self.h * self.w * (3.0 + 8.0))

    def _forward_features_strict(self, training):
        """the same plan in split-bf16 / fp32 arithmetic: conv (3 operand-split terms on the tensor cores) -> fp32 z -> fp64 batch
        statistics -> SiLU(BN(z)) (+ shortcut, + upsampled copy) stored as split pairs -> fp32 head outputs"""
        L, sp = self.L, capi.stream_ptr()
        nb, f8 = self.nbn, self.flat_stats
        pf = lambda t, off: ctypes.c_void_p(t.data_ptr() + 4 * off)
        for op in self.ops:
            if isinstance(op, ConvOp):
                zb = op.z.buf
                capi.check(L.yb200_conv2d_fwd_split(op.x.act(), op.x.buf.lo, self.planes, capi.ptr(op.w_split), op.cout, op.ksize, op.stride, capi.ptr(zb.t), zb.c, 0,
                                                    sp), "conv split " + op.prefixes[0])
                o = op.bn_off
                gamma = self.params[op.prefixes[0] + ".bn.weight"]
                beta = self.params[op.heads[0].prefix + ".bn.bias"]
                npix = zb.n * zb.h * zb.w
                if training:
                    ssum, ssq = ctypes.c_void_p(f8.data_ptr() + 8 * o), ctypes.c_void_p(f8.data_ptr() + 8 * (nb + o))
                    capi.check(L.yb200_strict_bn_stats(capi.ptr(zb.t), ctypes.c_int64(npix), zb.c, 0, op.cout, ssum, ssq, sp), "strict_bn_stats")
                    capi.check(L.yb200_bn_finalize(ssum, ssq, op.cout, ctypes.c_int64(npix), capi.ptr(gamma), capi.ptr(beta), ctypes.c_float(BN_EPS),
                                                   ctypes.c_float(BN_MOMENTUM), pf(self.flat_rm, o), pf(self.flat_rv, o), None, pf(self.flat_scale, o),
                                                   pf(self.flat_shift, o), pf(self.flat_mean, o), pf(self.flat_invstd, o), sp), "bn_finalize")
                else:
                    capi.check(L.yb200_bn_eval_affine(op.cout, capi.ptr(gamma), capi.ptr(beta), pf(self.flat_rm, o), pf(self.flat_rv, o),
                                                      ctypes.c_float(BN_EPS), pf(self.flat_scale, o), pf(self.flat_shift, o), sp), "bn_eval_affine")
                self._count(3 if training else 2, "strict conv+stats+finalize %s %s" % (op.prefixes[0], self._desc(op)))
                for hd in op.heads:
                    capi.check(L.yb200_strict_bn_apply_silu(capi.ptr(zb.t), zb.c, hd.c0, pf(self.flat_scale, hd.bn_off), pf(self.flat_shift, hd.bn_off),
                                                            hd.residual.act() if hd.residual else None, hd.residual.buf.lo if hd.residual else 0,
                                                            hd.out.act(), hd.out.buf.lo, hd.up.act() if hd.up else None, hd.up.buf.lo if hd.up else 0, self.planes, sp),
                               "strict_bn_apply_silu " + hd.prefix)
                    self._count(1, "strict bn_apply " + hd.prefix)
            elif isinstance(op, SppOp):
                v = op.views
                capi.check(L.yb200_strict_spp_pool(v[0].act(), v[1].act(), v[2].act(), v[3].act(), v[0].buf.lo, self.planes, sp), "strict_spp_pool")
                self._count(1, "strict spp_pool")
            else:
                h, w, s, a_off = self.levels[op.level]
                ch = 5 + self.nc
                capi.check(L.yb200_conv1x1_bias_f32_split(op.cls_feat.act(), op.cls_feat.buf.lo, self.planes, capi.ptr(op.wc_split), capi.ptr(op.bc), self.nc,
                                                          capi.ptr(self.outputs), self.num_anchors, a_off, ch, 5, sp), "cls_pred split")
                capi.check(L.yb200_conv1x1_bias_f32_split(op.reg_feat.act(), op.reg_feat.buf.lo, self.planes, capi.ptr(op.wr_split), capi.ptr(op.br), 5,
                                                          capi.ptr(self.outputs), self.num_anchors, a_off, ch, 0, sp), "reg_obj_pred split")
                self._count(2, "strict pred convs level %d" % op.level)
        if training:
            self.flat_nbt += 1
        self._decode(training)
        self._count(1, "decode")

    def forward_features(self, training=True, op_range=None):
        """op_range = (lo, hi): run only self.ops[lo:hi] (standalone backbone / neck / head execution, modeling.py); the head decode
        runs when the range reaches the end of the plan"""
        if self.strict:
            assert op_range is None
            return self._forward_features_strict(training)
        L, sp = self.L, capi.stream_ptr()
        nb = self.nbn
        f8 = self.flat_stats
        lo_i, hi_i = op_range if op_range is not None else (0, len(self.ops))
        if training:
            f8[:2 * nb].zero_()  # BatchNorm sum / sum-of-squares accumulators of every layer: cleared once per forward (one memset)
            self._count(1, "clear BatchNorm accumulators (memset)")
        for op in self.ops[lo_i:hi_i]:
            if isinstance(op, ConvOp):
                o = op.bn_off
                gamma = self.params[op.prefixes[0] + ".bn.weight"]
                beta = self.params[op.heads[0].prefix + ".bn.bias"]
                pf = lambda t, off=o: ctypes.c_void_p(t.data_ptr() + 4 * off)
                if not training and all(hd.up is None for hd in op.heads) and not (op.first and self.group4):
                    # eval: BatchNorm (running statistics) + SiLU + shortcut folded into the convolution's epilogue
                    capi.check(L.yb200_bn_eval_affine(op.cout, capi.ptr(gamma), capi.ptr(beta), pf(self.flat_rm), pf(self.flat_rv),
                                                      ctypes.c_float(BN_EPS), pf(self.flat_scale), pf(self.flat_shift), sp), "bn_eval_affine")
                    self._count(1, "bn_eval_affine " + op.prefixes[0])
                    kk = op.ksize * op.ksize
                    for hd in op.heads:
                        w_head = ctypes.c_void_p(op.w_fwd.data_ptr() + 2 * hd.c0 * kk * op.cin_pad)
                        capi.check(L.yb200_conv2d_bn_silu_fwd(op.x.act(), w_head, pf(self.flat_scale, hd.bn_off), pf(self.flat_shift, hd.bn_off),
                                                             hd.residual.act() if hd.residual else None, hd.out.act(), op.ksize, op.stride, sp),
                                   "conv_bn_silu " + hd.prefix)
                        self._count(1, "conv+bn+silu (eval) %s %s" % (hd.prefix, self._desc(op)))
                    continue
                ssum = ctypes.c_void_p(f8.data_ptr() + 8 * o) if training else None
                ssq = ctypes.c_void_p(f8.data_ptr() + 8 * (nb + o)) if training else None
                if op.first and self.group4:
                    xg, zg = self._grouped_views(op)
                    if training:
                        capi.check(L.yb200_conv2d_fwd_fold(ctypes.byref(xg), capi.ptr(op.w_fwd), ctypes.byref(zg), 3, 1, ssum, ssq, op.cout, sp), op.prefixes[0])
                    else:
                        capi.check(L.yb200_conv2d_fwd(ctypes.byref(xg), capi.ptr(op.w_fwd), ctypes.byref(zg), 3, 1, None, None, sp), op.prefixes[0])
                else:
                    capi.check(L.yb200_conv2d_fwd(op.x.act(), capi.ptr(op.w_fwd), op.z.act(), op.ksize, op.stride, ssum, ssq, sp), op.prefixes[0])
                npx = op.z.buf.n * op.z.buf.h * op.z.buf.w
                if not training:
                    capi.check(L.yb200_bn_eval_affine(op.cout, capi.ptr(gamma), capi.ptr(beta), pf(self.flat_rm), pf(self.flat_rv),
                                                      ctypes.c_float(BN_EPS), pf(self.flat_scale), pf(self.flat_shift), sp), "bn_eval_affine")
                self._count(1 if training else 2, "conv_fwd %s %s" % (op.prefixes[0], self._desc(op)), "conv_fwd (conv_gemm, BN statistics in the epilogue)",
                            *self._alg_conv(op))
                for hd in op.heads:
                    zv = op.z.buf.view(hd.c0, hd.c)
                    if training:  # finalize (scale / shift, running statistics, saved mean / invstd) folded into the apply pass: one launch
                        ho = hd.bn_off
                        capi.check(L.yb200_bn_train_apply_silu(zv.act(), ctypes.c_void_p(f8.data_ptr() + 8 * ho), ctypes.c_void_p(f8.data_ptr() + 8 * (nb + ho)),
                                                               ctypes.c_int64(npx), pf(gamma, hd.c0), pf(beta, hd.c0), ctypes.c_float(BN_EPS),
                                                               ctypes.c_float(BN_MOMENTUM), pf(self.flat_rm, ho), pf(self.flat_rv, ho), pf(self.flat_scale, ho),
                                                               pf(self.flat_shift, ho), pf(self.flat_mean, ho), pf(self.flat_invstd, ho),
                                                               hd.residual.act() if hd.residual else None, hd.out.act(), hd.up.act() if hd.up else None, sp),
                                   "bn_train_apply_silu " + hd.prefix)
                    else:
                        capi.check(L.yb200_bn_apply_silu(zv.act(), pf(self.flat_scale, hd.bn_off), pf(self.flat_shift, hd.bn_off),
                                                         hd.residual.act() if hd.residual else None, hd.out.act(), hd.up.act() if hd.up else None, sp),
                                   "bn_apply_silu " + hd.prefix)
                    self._count(1, "bn_apply %s c=%d px=%d" % (hd.prefix, hd.c, npx), "bn_apply_silu (+ finalize)",
                                2.0 * npx * hd.c * (2 + (1 if hd.residual else 0) + (4 if hd.up else 0)))
            elif isinstance(op, SppOp):
                v = op.views
                capi.check(L.yb200_spp_pool(v[0].act(), v[1].act(), v[2].act(), v[3].act(), capi.ptr(op.arg) if training else None, sp), "spp_pool")
                self._count(1, "spp_pool", "spp_pool", 2.0 * 4 * v[0].buf.n * v[0].buf.h * v[0].buf.w * v[0].c)
            else:
                h, w, s, a_off = self.levels[op.level]
                ch = 5 + self.nc
                capi.check(L.yb200_conv1x1_bias_f32(op.cls_feat.act(), capi.ptr(op.wc_fwd), capi.ptr(op.bc), self.nc, capi.ptr(self.outputs),
                                                    self.num_anchors, a_off, ch, 5, sp), "cls_pred")
                capi.check(L.yb200_conv1x1_bias_f32(op.reg_feat.act(), capi.ptr(op.wr_fwd), capi.ptr(op.br), 5, capi.ptr(self.outputs),
                                                    self.num_anchors, a_off, ch, 0, sp), "reg_obj_pred")
                self._count(2, "pred convs level %d" % op.level, "pred_conv fwd", self.n * h * w * (2.0 * 2 * self.hc + 4.0 * ch),
                            2.0 * self.n * h * w * self.hc * ch)
        if training:
            if op_range is None:
                self.flat_nbt += 1
            else:  # only the BatchNorm layers that ran
                i0 = sum(len(o.heads) for o in self.ops[:lo_i] if isinstance(o, ConvOp))
                i1 = i0 + sum(len(o.heads) for o in self.ops[lo_i:hi_i] if isinstance(o, ConvOp))
                self.flat_nbt[i0:i1] += 1
            self._count(1, "num_batches_tracked += 1 (torch)")
        if hi_i < len(self.ops):
            return
        self._decode(training)
        self._count(1, "decode", "decode", 8.0 * self.n * self.num_anchors * 4)

    def _decode(self, training):
        L, sp = self.L, capi.stream_ptr()
        if training and self.use_l1:
            if self.raw_reg is None:
                self.raw_reg = torch.zeros(self.n, self.num_anchors, 4, device=self.dev)
            capi.check(L.yb200_yolox_decode_keep_raw(capi.ptr(self.outputs), self.n, self.num_anchors, 5 + self.nc, self.lv, len(self.levels),
                                                     capi.ptr(self.raw_reg), sp), "decode (+ origin_preds)")
        else:
            capi.check(L.yb200_yolox_decode(capi.ptr(self.outputs), self.n, self.num_anchors, 5 + self.nc, self.lv, len(self.levels),
                                            0 if training else 1, sp), "decode")

    def assign_and_loss(self, with_grad=True):
        L, sp = self.L, capi.stream_ptr()
        n, a, ch = self.n, self.num_anchors, 5 + self.nc
        capi.check(L.yb200_simota_assign(capi.ptr(self.outputs), capi.ptr(self.labels), n, a, ch, self.max_gt, self.lv, len(self.levels),
                                         capi.ptr(self.simota_ws), capi.ptr(self.num_gt), capi.ptr(self.fg_mask), capi.ptr(self.matched_gt),
                                         capi.ptr(self.matched_iou), capi.ptr(self.matched_cls), capi.ptr(self.num_fg_img), capi.ptr(self.totals), sp),
                   "simota_assign")
        self._count(4, "simota (count_gt, prep, match, resolve)", "simota_assign", 4.0 * n * a * ch)
        self._loss(capi.ptr(self.loss_weights) if with_grad else None, capi.ptr(self.losses), self.p_dcls if with_grad else None,
                   self.p_dro if with_grad else None, capi.ptr(self.bias_acc) if with_grad else None, "yolox_loss")
        self._count(2, "yolox_loss + finish", "yolox_loss", n * a * ch * (4.0 + (2.0 if with_grad else 0.0)))

    def loss_grad_only(self):
        """recompute d loss / d head outputs with the current loss_weights (autograd path: upstream gradients arrive late)"""
        L, sp = self.L, capi.stream_ptr()
        n, a, ch = self.n, self.num_anchors, 5 + self.nc
        self._loss(capi.ptr(self.loss_weights), None, self.p_dcls, self.p_dro, capi.ptr(self.bias_acc), "yolox_loss grad")
        self._count(1, "yolox_loss grad")

    def _loss(self, weights, losses, p_dcls, p_dro, bias_acc, what):
        """get_losses (yolox_head.py:412-441), with the L1 term when `use_l1` (the decode of this step kept the raw regression outputs)"""
        L, sp = self.L, capi.stream_ptr()
        n, a, ch = self.n, self.num_anchors, 5 + self.nc
        lab, fg, mgt, miou, mcls = capi.ptr(self.labels), capi.ptr(self.fg_mask), capi.ptr(self.matched_gt), capi.ptr(self.matched_iou), capi.ptr(self.matched_cls)
        tot, acc, nl = capi.ptr(self.totals), capi.ptr(self.loss_acc), len(self.levels)
        if self.use_l1:
            if self.raw_reg is None:
                raise capi.Yb200Error("use_l1 was switched on after this step's forward: run the forward pass again")
            capi.check(L.yb200_yolox_loss_l1(capi.ptr(self.outputs), capi.ptr(self.raw_reg), lab, n, a, ch, self.max_gt, self.lv, nl, fg, mgt, miou, mcls, tot,
                                             weights, acc, losses, p_dcls, p_dro, None, bias_acc, sp), what + " (+ L1)")
        else:
            capi.check(L.yb200_yolox_loss(capi.ptr(self.outputs), lab, n, a, ch, self.max_gt, self.lv, nl, fg, mgt, miou, mcls, tot, weights, acc, losses,
                                          p_dcls, p_dro, None, bias_acc, sp), what)

    # ------------------------------------------------------------------ backward
    def _grouped_views(self, op, dz=None):
        """the stem's input / output (or output gradient) seen as [N, H, W/4, 4C]: same memory, 4 pixels per row"""
        xb = op.x.buf
        xg = capi.act(xb.t.view(xb.n, xb.h, xb.w // 4, 4 * xb.c))
        zt = op.z.buf.t if dz is None else dz
        zg = capi.act(zt.view(zt.shape[0], zt.shape[1], zt.shape[2] // 4, 4 * zt.shape[3]))
        return xg, zg

    def _wgrad_stem_grouped(self, op, dz_t, acc):
        """weight gradient of the grouped stem convolution, folded back onto the [32, 12, 3, 3] parameter (side stream)"""
        L = self.L
        xg, dzg = self._grouped_views(op, dz_t)
        need = L.yb200_conv2d_wgrad_workspace(ctypes.byref(xg), ctypes.byref(dzg), 3, 1)
        assert need > 0, L.yb200_last_error()
        self._ensure_ws(need)

        def run():
            capi.check(L.yb200_conv2d_wgrad_grouped(ctypes.byref(xg), ctypes.byref(dzg), 3, 1, 4 * op.cin_pad, 4, capi.ptr(op.g_exp), 0, capi.ptr(self.ws),
                                                    ctypes.c_int64(self.ws_bytes), capi.stream_ptr()), "wgrad stem (grouped)")
            g = op.g_dst.reshape(-1)
            parts = op.fold_parts  # every real weight appears in several (e, f, t) positions
            torch.index_select(op.g_exp.reshape(-1), 0, op.fold_pos, out=parts.view(-1))
            for i in range(parts.shape[1]):  # added one position at a time, in ascending position order
                if i == 0 and not acc:
                    g.copy_(parts[:, 0])
                else:
                    g.add_(parts[:, i])

        if self.overlap_wgrad:
            main = torch.cuda.current_stream()
            self._fork_evt.record(main)
            with torch.cuda.stream(self._side):
                self._side.wait_event(self._fork_evt)
                run()
        else:
            run()

    def _dz_buf(self, op):
        b = self._dz.get(id(op))
        if b is None:
            zb = op.z.buf
            b = Buf(zb.name + ".dz", zb.n, zb.h, zb.w, zb.c, self.dev)
            self._dz[id(op)] = b
        return b

    def _grad_target(self, view):
        """returns (addend or None) for a data-gradient that lands in view's gradient: first producer writes, later ones accumulate"""
        buf = view.buf
        lo, hi = view.off, view.off + view.c
        covered = any(a <= lo and hi <= b for a, b in buf.written)
        overlap = any(not (hi <= a or b <= lo) for a, b in buf.written)
        if covered:
            return view
        assert not overlap, f"partial overlap of gradient writes on {buf.name}"
        buf.written.append((lo, hi))
        return None

    def _wgrad(self, x_act, dz_act, ksize, stride, cin_real, gdst, acc, label):
        """Weight gradients are off the backward critical path (nothing downstream reads them): they run on a side stream,
        overlapping the next layers' data-gradient / BatchNorm-backward chain.  All of them are serialised on that one
        stream, so a single split-K workspace suffices."""
        L = self.L
        need = L.yb200_conv2d_wgrad_workspace(x_act, dz_act, ksize, stride)
        assert need > 0, L.yb200_last_error()
        self._ensure_ws(need)
        if self.overlap_wgrad:
            main = torch.cuda.current_stream()
            self._fork_evt.record(main)
            with torch.cuda.stream(self._side):
                self._side.wait_event(self._fork_evt)
                capi.check(L.yb200_conv2d_wgrad(x_act, dz_act, ksize, stride, cin_real, capi.ptr(gdst), acc, capi.ptr(self.ws),
                                                ctypes.c_int64(self.ws_bytes), capi.stream_ptr()), "wgrad " + label)
        else:
            capi.check(L.yb200_conv2d_wgrad(x_act, dz_act, ksize, stride, cin_real, capi.ptr(gdst), acc, capi.ptr(self.ws),
                                            ctypes.c_int64(self.ws_bytes), capi.stream_ptr()), "wgrad " + label)

    def backward(self, accumulate=False, op_range=None, seeded=(), fresh=True):
        """op_range = (lo, hi): backward of self.ops[lo:hi] only, from gradients the caller has already stored in the gradient buffers of
        the `seeded` views (standalone backbone / neck / head, modeling.py), or -- fresh=False -- continuing a backward pass that earlier
        calls ran over the later ranges (dist.GradientBuckets: the gradient bucket of a finished range is all-reduced while the next range
        computes)."""
        if self.strict:
            raise capi.Yb200Error("strict mode is a forward / loss verification mode: no backward (use the default engine for training)")
        L, sp = self.L, capi.stream_ptr()
        nb = self.nbn
        f8 = self.flat_stats
        acc = 1 if accumulate else 0
        if fresh:
            for b in self.bufs.values():
                b.written = []
        for v in seeded:
            v.buf.written.append((v.off, v.off + v.c))
        lo_i, hi_i = op_range if op_range is not None else (0, len(self.ops))
        pending_res = {}  # id(view.buf), off -> gradient view of the residual sum
        for op in reversed(self.ops[lo_i:hi_i]):
            if isinstance(op, PredOp):
                k = op.level
                h, w, s, a_off = self.levels[k]
                dcls = capi.act(self.d_cls[k])
                dro = capi.act(self.d_ro[k])
                capi.check(L.yb200_head_bias_grad(capi.ptr(self.bias_acc), len(self.levels), 5 + self.nc, k, capi.ptr(self.grads[f"head.reg_preds.{k}.bias"]),
                                                  capi.ptr(self.grads[f"head.obj_preds.{k}.bias"]), capi.ptr(self.grads[f"head.cls_preds.{k}.bias"]),
                                                  acc, sp), "head_bias_grad")
                for which, feat, dz, gdst, wd in (("cls", op.cls_feat, dcls, op.gc_dst, op.wc_dgrad), ("reg", op.reg_feat, dro, op.gr_dst, op.wr_dgrad)):
                    self._wgrad(feat.act(), ctypes.byref(dz), 1, 1, self.hc, gdst, acc, "pred")
                    add = self._grad_target(feat)
                    capi.check(L.yb200_conv2d_dgrad(ctypes.byref(dz), capi.ptr(wd), feat.gact(), add.gact() if add else None, 1, 1, sp), "pred dgrad")
                self._count(7, "pred level %d: bias_grad, 2x(wgrad, reduce, dgrad)" % k, "pred_conv bwd", self.n * h * w * 2.0 * (4 * self.hc + self.nc + 16),
                            4.0 * self.n * h * w * self.hc * (self.nc + 5))
            elif isinstance(op, SppOp):
                v = op.views
                if self.spp_scratch is None:
                    self.spp_scratch = torch.empty(v[0].buf.n * v[0].buf.h * v[0].buf.w * v[0].c, device=self.dev)
                # in place: the identity slice of the concat gradient receives the pooled gradients
                capi.check(L.yb200_spp_pool_bwd(v[0].gact(), v[1].gact(), v[2].gact(), v[3].gact(), capi.ptr(op.arg), capi.ptr(self.spp_scratch),
                                                v[0].gact(), sp), "spp_pool_bwd")
                self._count(2, "spp_pool_bwd (scatter, finish)", "spp_pool_bwd", 2.0 * 5 * v[0].buf.n * v[0].buf.h * v[0].buf.w * v[0].c)
            else:
                dzb = self._dz_buf(op)
                pf = lambda t, off: ctypes.c_void_p(t.data_ptr() + 4 * off)
                for hd in op.heads:
                    zv = op.z.buf.view(hd.c0, hd.c)
                    dzv = dzb.view(hd.c0, hd.c)
                    o = hd.bn_off
                    npx = op.z.buf.n * op.z.buf.h * op.z.buf.w
                    capi.check(L.yb200_bn_silu_bwd(zv.act(), hd.out.gact(), None, hd.up.gact() if hd.up else None, pf(self.flat_scale, o),
                                                   pf(self.flat_shift, o), pf(self.flat_mean, o), pf(self.flat_invstd, o),
                                                   ctypes.c_void_p(f8.data_ptr() + 8 * (2 * nb + o)), ctypes.c_void_p(f8.data_ptr() + 8 * (3 * nb + o)),
                                                   dzv.act(), None, None, acc, sp), "bn_silu_bwd " + hd.prefix)
                    self._count(2, "bn_bwd (reduce, apply) %s c=%d px=%d" % (hd.prefix, hd.c, npx), "bn_silu_bwd",
                                2.0 * npx * hd.c * (3 + (4 if hd.up else 0)))
                    if hd.residual is not None:
                        pending_res[(id(hd.residual.buf), hd.residual.off)] = hd.out
                dz = dzb.view()
                if op.first and self.group4:
                    self._wgrad_stem_grouped(op, dzb.t, acc)
                else:
                    self._wgrad(op.x.act(), dz.act(), op.ksize, op.stride, op.cin_real, op.g_dst, acc, op.prefixes[0])
                self._count(2, "wgrad+reduce %s %s" % (op.prefixes[0], self._desc(op)), "wgrad (wgrad_gemm + reduce)", *self._alg_conv(op))
                if not op.first:
                    res = pending_res.pop((id(op.x.buf), op.x.off), None)
                    add = self._grad_target(op.x)
                    assert not (res is not None and add is not None), "residual + fan-out on the same activation"
                    addend = res.gact() if res is not None else (add.gact() if add is not None else None)
                    capi.check(L.yb200_conv2d_dgrad(dz.act(), capi.ptr(op.w_dgrad), op.x.gact(), addend, op.ksize, op.stride, sp), "dgrad " + op.prefixes[0])
                    self._count(1, "dgrad %s %s" % (op.prefixes[0], self._desc(op)), "dgrad (conv_gemm)", *self._alg_conv(op))
        # BatchNorm weight / bias gradients of the whole range out of the fp64 accumulators: one launch (the per-layer kernels left them there)
        heads = [hd for op in self.ops[lo_i:hi_i] if isinstance(op, ConvOp) for hd in op.heads]
        if heads:
            b0, b1 = min(hd.bn_off for hd in heads), max(hd.bn_off + hd.c for hd in heads)
            assert b1 - b0 == sum(hd.c for hd in heads), "BatchNorm channels of an op range are one run of the flat statistics buffers"
            i4 = lambda t: ctypes.c_void_p(t.data_ptr() + 4 * b0)
            capi.check(L.yb200_bn_param_grads(ctypes.c_void_p(f8.data_ptr() + 8 * (2 * nb + b0)), ctypes.c_void_p(f8.data_ptr() + 8 * (3 * nb + b0)), b1 - b0,
                                              i4(self.bn_goff), i4(self.bn_boff), capi.ptr(self.flat_grad), acc, sp), "bn_param_grads")
            self._count(1, "bn param grads of %d layers" % len(heads), "bn_silu_bwd")
        if self.overlap_wgrad:
            torch.cuda.current_stream().wait_stream(self._side)  # join: gradients are complete when backward() returns

    # ------------------------------------------------------------------ whole steps
    def train_step(self, accumulate=False):
        """forward + backward on the resident batch (images_u8 / labels already on the device)"""
        self.pack_weights()
        self.preprocess()
        self.forward_features(True)
        self.assign_and_loss(not self.strict)
        if not self.strict:
            self.backward(accumulate)
        return self.losses

    def eval_forward(self):
        self.pack_weights()
        self.preprocess()
        self.forward_features(False)
        return self.outputs
