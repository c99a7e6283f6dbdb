"""SparseInst IAM decoder on the H100 kernels, forward and backward (SURVEY.md par.8a row S1).

Reference: yolov7/modeling/transcoders/decoder_sparseinst.py -- `InstanceBranch` :27-81, `MaskBranch` :84-104, `BaseIAMDecoder` :107-169.
`BaseIAMDecoder(cfg)` below keeps the reference's constructor (the same `cfg.MODEL.SPARSE_INST.*` keys), parameter names / shapes
(`inst_branch.inst_convs.{0,2,..}.weight`, `inst_branch.iam_conv.*`, `inst_branch.{cls_score,mask_kernel,objectness}.*`,
`mask_branch.mask_convs.*`, `mask_branch.projection.*`) and `forward(features NCHW fp32) -> {"pred_logits", "pred_masks", "pred_scores"[, "pred_iam"]}`.

Kernel sequence (NHWC bf16 inside):
  coordinates + features -> [B,H,W,Cpad]  |  4x conv3x3+bias+ReLU (wgmma implicit GEMM, `EPI_BF16_BIAS_RELU`) per branch
  iam = conv3x3+bias -> sigmoid -> per image:  raw = iam_prob^T features  (the pixel-contraction GEMM of the weight-gradient kernel: MN-major
  wgmma descriptors straight on the NHWC tiles), normaliser = column sums, inst = raw / max(norm, 1e-6)
  heads: three small GEMMs with fp32 output (`yb200_conv1x1_bias_f32`)  |  mask projection 1x1
  pred_masks = per-image 1x1 convolution of the mask features with pred_kernel[b] as weights, fp32 NCHW written by the GEMM epilogue
The final bilinear x2 up-sampling (decoder_sparseinst.py:148-153) is `yb200_upsample_bilinear2x_f32` (other scale factors: F.interpolate).
Training: with autograd recording and `features` or a parameter requiring grad, the decoder runs as one autograd node (`_DecoderFn`) that
issues the same forward calls and keeps the intermediates; its backward (`BaseIAMDecoder._backward`, DESIGN.md par.7) returns every parameter's
fp32 gradient and d features (fp32 NCHW) on this library's kernels: the bilinear x2 adjoint, the mask GEMM's weight / data gradients, data
gradients through the ReLUs (`yb200_conv2d_dgrad_relu`), weight gradients, fixed-order column sums for the biases, the normalisation and sigmoid
backward kernels.  Sums run in a fixed order (no float atomics): two backward calls give the same bits.  SCALE_FACTOR != 2 keeps torch's
interpolate forward and has no backward (Yb200Error).  `pred_iam` (OUTPUT_IAM) carries no gradient.  The matcher and the losses of
sparseinst_loss.py, with their gradients w.r.t. this module's outputs, are `sparseinst_criterion.py`.
Instance / kernel counts are padded to multiples of 16 internally (100 -> 112: padded IAM channels get bias -30, i.e. probability 0).
"""
import ctypes

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import capi


def _pad16(c):
    return (c + 15) // 16 * 16


class _Conv(nn.Module):
    def __init__(self, cin, cout, k, device, std):
        super().__init__()
        self.weight = nn.Parameter(torch.randn(cout, cin, k, k, device=device) * std)
        self.bias = nn.Parameter(torch.zeros(cout, device=device))


class _Linear(nn.Module):
    def __init__(self, cin, cout, device, std=0.01, bias=0.0):
        super().__init__()
        self.weight = nn.Parameter(torch.randn(cout, cin, device=device) * std)
        self.bias = nn.Parameter(torch.full((cout,), float(bias), device=device))


def _stack(num_convs, cin, cout, device):
    """`_make_stack_3x3_convs` (decoder_sparseinst.py:18-24): Sequential(Conv2d, ReLU, Conv2d, ReLU, ...) -> parameters at even indices"""
    seq = nn.Module()
    for i in range(num_convs):
        seq.add_module(str(2 * i), _Conv(cin, cout, 3, device, (2.0 / (9 * cout)) ** 0.5))  # c2_msra_fill: kaiming normal, fan_out
        cin = cout
    return seq


class BaseIAMDecoder(nn.Module):
    def __init__(self, cfg, device="cuda"):
        super().__init__()
        sp = cfg.MODEL.SPARSE_INST
        dec = sp.DECODER
        self.in_channels = sp.ENCODER.NUM_CHANNELS + 2  # + coordinates (:111-112)
        self.scale_factor, self.output_iam = dec.SCALE_FACTOR, dec.OUTPUT_IAM
        self.dim, self.num_convs = dec.INST.DIM, dec.INST.CONVS
        self.mask_dim, self.mask_convs_n = dec.MASK.DIM, dec.MASK.CONVS
        self.num_masks, self.kernel_dim, self.num_classes = dec.NUM_MASKS, dec.KERNEL_DIM, dec.NUM_CLASSES
        if self.dim % 16 or self.mask_dim % 16 or self.kernel_dim % 16 or self.kernel_dim > 128 or self.num_classes > 128:
            raise capi.Yb200Error("BaseIAMDecoder: branch widths must be multiples of 16, kernel_dim and num_classes at most 128")
        dev = torch.device(device)
        prior = -4.59511985013459  # -log((1 - 0.01) / 0.01)   (:45, :54)
        self.inst_branch = nn.Module()
        self.inst_branch.inst_convs = _stack(self.num_convs, self.in_channels, self.dim, dev)
        self.head_dim = self._build_iam(dev, prior)  # width of the per-instance feature the heads read
        self.inst_branch.cls_score = _Linear(self.head_dim, self.num_classes, dev, bias=prior)
        self.inst_branch.mask_kernel = _Linear(self.head_dim, self.kernel_dim, dev)
        self.inst_branch.objectness = _Linear(self.head_dim, 1, dev)
        self.mask_branch = nn.Module()
        self.mask_branch.mask_convs = _stack(self.mask_convs_n, self.in_channels, self.mask_dim, dev)
        self.mask_branch.projection = _Conv(self.mask_dim, self.kernel_dim, 1, dev, (2.0 / self.kernel_dim) ** 0.5)
        self.L = capi.lib()

    def _build_iam(self, dev, prior):
        """InstanceBranch (:27-60): one 3x3 convolution dim -> num_masks"""
        self.inst_branch.iam_conv = _Conv(self.dim, self.num_masks, 3, dev, 0.01)
        with torch.no_grad():
            self.inst_branch.iam_conv.bias.fill_(prior)
        return self.dim

    # ---- helpers -----------------------------------------------------------------------------------------------------------------
    def _pack(self, w, cout_pad, cin_pad):
        cout, cin, k = w.shape[0], w.shape[1], (w.shape[2] if w.dim() == 4 else 1)
        wf = torch.empty(cout_pad, k * k, cin_pad, dtype=torch.bfloat16, device=w.device)
        capi.check(self.L.yb200_pack_conv_weight(capi.ptr(w.detach().contiguous()), cout, cin, k, cout_pad, cin_pad, capi.ptr(wf), None, capi.stream_ptr()), "pack")
        return wf

    def _conv_relu(self, x, conv, cin_pad):
        b, h, w, _ = x.shape
        cout = conv.weight.shape[0]
        out = torch.empty(b, h, w, cout, dtype=torch.bfloat16, device=x.device)
        xa, oa = capi.act(x), capi.act(out)
        capi.check(self.L.yb200_conv2d_relu_fwd(ctypes.byref(xa), capi.ptr(self._pack(conv.weight, cout, cin_pad)), capi.ptr(conv.bias.detach()), ctypes.byref(oa), 3, 1,
                                                capi.stream_ptr()), "conv3x3+relu")
        return out

    def _branch(self, x, seq, n, acts=None):
        """the 3x3 + ReLU stack; `acts` (a list) receives every layer's output for the backward"""
        cin_pad = x.shape[-1]
        for i in range(n):
            x = self._conv_relu(x, getattr(seq, str(2 * i)), cin_pad)
            cin_pad = x.shape[-1]
            if acts is not None:
                acts.append(x)
        return x

    def _heads_f32(self, inst, lin, cout):
        """inst: bf16 [B,1,Npad,dim] -> fp32 [B, Npad, cout]"""
        b, _, npad, _ = inst.shape
        cpad = max(16, _pad16(cout))
        out = torch.empty(b, npad, cout, device=inst.device)
        xa = capi.act(inst)
        capi.check(self.L.yb200_conv1x1_bias_f32(ctypes.byref(xa), capi.ptr(self._pack(lin.weight, cpad, inst.shape[-1])), capi.ptr(lin.bias.detach()), cout, capi.ptr(out),
                                                 npad, 0, cout, 0, capi.stream_ptr()), "head")
        return out

    def _aggregate(self, f, prob, save=None):
        """inst[b] = prob[b]^T f[b] / clamp(sum prob[b], 1e-6)   (:70-76): the pixel contraction is the weight-gradient GEMM (MN-major wgmma
        descriptors on the NHWC tiles), per image; returns bf16 [B, 1, C_prob, dim].  raw = prob^T f and the normalisers are kept per image
        (fp32 [B, C_prob, dim] and [B, C_prob]): the backward reads them"""
        L, sp = self.L, capi.stream_ptr()
        b, dev, npad = f.shape[0], f.device, prob.shape[-1]
        inst = torch.empty(b, 1, npad, self.dim, dtype=torch.bfloat16, device=dev)
        raw = torch.empty(b, npad, self.dim, device=dev)
        norm = torch.empty(b, npad, device=dev)
        f1, p1 = capi.act(f[0:1]), capi.act(prob[0:1])
        ws_g = torch.empty(max(int(L.yb200_conv2d_wgrad_workspace(ctypes.byref(f1), ctypes.byref(p1), 1, 1)), 16), dtype=torch.uint8, device=dev)
        ws_c = torch.empty(max(int(L.yb200_colsum_workspace(ctypes.byref(p1))), 16), dtype=torch.uint8, device=dev)
        for i in range(b):
            fi, pi, oi = capi.act(f[i:i + 1]), capi.act(prob[i:i + 1]), capi.act(inst[i:i + 1])
            capi.check(L.yb200_conv2d_wgrad(ctypes.byref(fi), ctypes.byref(pi), 1, 1, self.dim, capi.ptr(raw[i]), 0, capi.ptr(ws_g), ctypes.c_int64(ws_g.numel()),
                                            sp), "iam bmm")
            capi.check(L.yb200_colsum(ctypes.byref(pi), ctypes.c_float(1.0), capi.ptr(norm[i]), 0, capi.ptr(ws_c), sp), "iam normaliser")
            capi.check(L.yb200_iam_normalize(capi.ptr(raw[i]), capi.ptr(norm[i]), npad, self.dim, ctypes.byref(oi), sp), "iam normalise")
        if save is not None:
            save.update(prob=prob, raw=raw, norm=norm)
        return inst

    def _instances(self, f, save=None):
        """InstanceBranch.forward (:62-81) up to the aggregated instance features"""
        L, sp = self.L, capi.stream_ptr()
        b, h, w, _ = f.shape
        dev = f.device
        n, npad = self.num_masks, _pad16(self.num_masks)
        iam_conv = self.inst_branch.iam_conv
        bias = torch.full((npad,), -30.0, device=dev)
        bias[:n] = iam_conv.bias.detach()
        iam = torch.empty(b, h, w, npad, dtype=torch.bfloat16, device=dev)
        fa, ia = capi.act(f), capi.act(iam)
        capi.check(L.yb200_conv2d_affine_fwd(ctypes.byref(fa), capi.ptr(self._pack(iam_conv.weight, npad, self.dim)), None, capi.ptr(bias), None, ctypes.byref(ia), 3, 1, sp),
                   "iam_conv")
        prob = torch.empty_like(iam)
        pa = capi.act(prob)
        capi.check(L.yb200_sigmoid(ctypes.byref(ia), ctypes.byref(pa), sp), "sigmoid")
        inst = self._aggregate(f, prob, save)
        if save is not None:
            save.update(iam=iam, inst=inst)
        return inst, iam[..., :n]

    # ---- forward -----------------------------------------------------------------------------------------------------------------
    def forward(self, features):
        """{"pred_logits", "pred_masks", "pred_scores"[, "pred_iam"]}.  With autograd recording and `features` or a parameter requiring grad,
        the decoder is one autograd node (`_DecoderFn`): the same kernel calls forward, the backward of `_backward` on the kernels.
        `pred_iam` carries no gradient."""
        if not features.is_cuda:
            raise capi.Yb200Error("BaseIAMDecoder: input must be a CUDA tensor (no CPU path)")
        params = [p for _, p in self.named_parameters()]
        if torch.is_grad_enabled() and (features.requires_grad or any(p.requires_grad for p in params)):
            logits, pred_masks, scores = _DecoderFn.apply(self, features, *params)
            out = {"pred_logits": logits, "pred_masks": pred_masks, "pred_scores": scores}
        else:
            with torch.no_grad():
                out = self._run(features)
        if self.output_iam:
            with torch.no_grad():
                out["pred_iam"] = F.interpolate(self.last["iam"].permute(0, 3, 1, 2).float(), scale_factor=self.scale_factor, mode="bilinear",
                                                align_corners=False)
        return out

    def _run(self, features, save=None):
        """the forward kernels; `save` (a dict) receives what the backward reads"""
        L, sp = self.L, capi.stream_ptr()
        b, c, h, w = features.shape
        assert c + 2 == self.in_channels, (c, self.in_channels)
        dev = features.device
        cpad = _pad16(self.in_channels)
        # coordinates (x_loc, y_loc) in [-1, 1] in front of the features (:118-132), NHWC bf16, zero padded to a multiple of 16 channels
        x = torch.zeros(b, h, w, cpad, dtype=torch.bfloat16, device=dev)
        x[..., 0] = torch.linspace(-1, 1, w, device=dev).view(1, 1, w)
        x[..., 1] = torch.linspace(-1, 1, h, device=dev).view(1, h, 1)
        x[..., 2:2 + c] = features.detach().permute(0, 2, 3, 1)
        acts_f, acts_m = ([], []) if save is not None else (None, None)
        # instance branch
        f = self._branch(x, self.inst_branch.inst_convs, self.num_convs, acts_f)
        n = self.num_masks
        inst, iam = self._instances(f, save)  # [B, 1, Npad, head_dim] bf16 instance features; iam logits [B, n, H, W]-shaped source (NHWC slice)
        npad = inst.shape[2]
        ib = self.inst_branch
        logits = self._heads_f32(inst, ib.cls_score, self.num_classes)[:, :n]
        kernel = self._heads_f32(inst, ib.mask_kernel, self.kernel_dim)            # [B, Npad, kernel_dim] (padded instances: bias only)
        scores = self._heads_f32(inst, ib.objectness, 1)[:, :n]
        # mask branch
        m = self._branch(x, self.mask_branch.mask_convs, self.mask_convs_n, acts_m)
        proj = self.mask_branch.projection
        mf = torch.empty(b, h, w, self.kernel_dim, dtype=torch.bfloat16, device=dev)
        ma, mfa = capi.act(m), capi.act(mf)
        capi.check(L.yb200_conv2d_affine_fwd(ctypes.byref(ma), capi.ptr(self._pack(proj.weight, self.kernel_dim, self.mask_dim)), None, capi.ptr(proj.bias.detach()), None,
                                             ctypes.byref(mfa), 1, 1, sp), "projection")
        masks = torch.empty(b, npad, h, w, device=dev)
        # torch.bmm(pred_kernel, mask_features) (:143-146): an image's predicted kernels are the weights of a 1x1 convolution over its mask features.
        # One launch for the batch when a 128-pixel tile stays inside one image (the [B * Npad, kernel_dim] kernels are packed to bf16 by one launch too)
        rc = L.yb200_conv1x1_nchw_f32_batched(ctypes.byref(mfa), capi.ptr(self._pack(kernel.reshape(b * npad, self.kernel_dim), b * npad, self.kernel_dim)), npad,
                                              capi.ptr(masks), sp)
        if rc == capi.ERR_UNSUPPORTED:  # small maps (tiles would span images): one launch per image
            for i in range(b):
                mi = capi.act(mf[i:i + 1])
                capi.check(L.yb200_conv1x1_nchw_f32(ctypes.byref(mi), capi.ptr(self._pack(kernel[i], npad, self.kernel_dim)), None, npad, capi.ptr(masks[i]), sp), "mask bmm")
        else:
            capi.check(rc, "mask bmm (batched)")
        if self.scale_factor == 2:  # bilinear x2 (:148-153) on the device kernel; other factors keep torch's interpolate
            m_lo = masks[:, :n].contiguous()
            pred_masks = torch.empty(b, n, 2 * h, 2 * w, device=dev)
            capi.check(L.yb200_upsample_bilinear2x_f32(capi.ptr(m_lo), capi.ptr(pred_masks), ctypes.c_int64(b * n), h, w, sp), "bilinear x2")
        else:
            pred_masks = F.interpolate(masks[:, :n], scale_factor=self.scale_factor, mode="bilinear", align_corners=False)
        # kept for tests / callers that want the un-interpolated tensors
        self.last = {"pred_kernel": kernel[:, :n], "iam": iam, "masks_lowres": masks[:, :n]}
        if save is not None:
            save.update(x=x, f=acts_f, m=acts_m, mf=mf, kernel=kernel)
        return {"pred_logits": logits, "pred_masks": pred_masks, "pred_scores": scores}

    # ---- backward ----------------------------------------------------------------------------------------------------------------
    def _pack_dgrad(self, w, cout_pad, cin_pad):
        """fp32 OIHW (or [out, in]) -> the data-gradient operand [cin_pad][k*k][cout_pad] bf16"""
        cout, cin, k = w.shape[0], w.shape[1], (w.shape[2] if w.dim() == 4 else 1)
        wd = torch.empty(cin_pad, k * k, cout_pad, dtype=torch.bfloat16, device=w.device)
        capi.check(self.L.yb200_pack_conv_weight(capi.ptr(w.detach().contiguous()), cout, cin, k, cout_pad, cin_pad, None, capi.ptr(wd), capi.stream_ptr()),
                   "pack dgrad")
        return wd

    def _wgrad(self, xa, dza, k, out):
        """out (fp32 [cout][cin_real][k][k] or [cout][cin_real], contiguous) = the weight gradient of the convolution x -> dz"""
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
            grads[name + ".weight"] = self._wgrad(xa, dza, k, torch.empty(dza.c, *conv.weight.shape[1:], device=dev))
        if need[name + ".bias"]:
            grads[name + ".bias"] = self._colsum(dza, torch.empty(dza.c, device=dev))

    def _stack_bwd(self, x, acts, dz, seq, prefix, grads, need):
        """backward of the 3x3 + ReLU stack from dz = the gradient of the last layer's pre-activation; returns the first layer's"""
        L, sp = self.L, capi.stream_ptr()
        for i in range(len(acts) - 1, -1, -1):
            inp = acts[i - 1] if i else x
            conv = getattr(seq, str(2 * i))
            self._conv_grads(capi.act(inp), capi.act(dz), conv, f"{prefix}{2 * i}", grads, need, 3)
            if i:
                dzi = torch.empty_like(inp)
                za, ha, da = capi.act(dz), capi.act(inp), capi.act(dzi)
                capi.check(L.yb200_conv2d_dgrad_relu(ctypes.byref(za), capi.ptr(self._pack_dgrad(conv.weight, dz.shape[-1], inp.shape[-1])), ctypes.byref(ha),
                                                     ctypes.byref(da), None, 3, 1, sp), "conv3x3 dgrad + relu bwd")
                dz = dzi
        return dz

    def _iam_grads(self, f, diam, dfagg, grads, need):
        """stage 8 of `_backward` for the single IAM convolution: d F (masked by F > 0, plus the aggregation's share) and the conv's gradients"""
        L, sp = self.L, capi.stream_ptr()
        npad, n = diam.shape[-1], self.num_masks
        conv = self.inst_branch.iam_conv
        df = torch.empty_like(f)
        za, fa, da, aa = capi.act(diam), capi.act(f), capi.act(df), capi.act(dfagg)
        capi.check(L.yb200_conv2d_dgrad_relu(ctypes.byref(za), capi.ptr(self._pack_dgrad(conv.weight, npad, self.dim)), ctypes.byref(fa), ctypes.byref(da),
                                             ctypes.byref(aa), 3, 1, sp), "iam_conv dgrad + relu bwd")
        if need["inst_branch.iam_conv.weight"]:
            gw = self._wgrad(capi.act(f), capi.act(diam), 3, torch.empty(npad, self.dim, 3, 3, device=f.device))
            grads["inst_branch.iam_conv.weight"] = gw[:n]
        if need["inst_branch.iam_conv.bias"]:
            grads["inst_branch.iam_conv.bias"] = self._colsum(capi.act(diam), torch.empty(npad, device=f.device))[:n]
        return df

    def _iam_layout(self):
        """(maps per group in the forward's IAM tensor, in the backward's d iam, groups)"""
        npad = _pad16(self.num_masks)
        return npad, npad, 1

    def _backward(self, s, g_logits, g_masks, g_scores, need_x, need):
        """gradients of the decoder (see DESIGN.md par.7 for the stages): {parameter name: fp32 gradient} for the names with need[name], and
        d features (fp32 NCHW) when need_x"""
        if self.scale_factor != 2:
            raise capi.Yb200Error(f"{type(self).__name__}: backward implemented for SCALE_FACTOR 2 (got {self.scale_factor})")
        L, sp = self.L, capi.stream_ptr()
        x, f, mf, kernel = s["x"], s["f"][-1], s["mf"], s["kernel"]
        b, h, w, cpad = x.shape
        dev = x.device
        n, npad, kd, ncls = self.num_masks, kernel.shape[1], self.kernel_dim, self.num_classes
        bf16 = torch.bfloat16
        grads = {}
        # 1. bilinear x2 adjoint -> d masks as the bf16 NHWC operand [B, H, W, Npad] (maps >= n zero)
        dm_lo = torch.empty(b, h, w, npad, dtype=bf16, device=dev)
        dma = capi.act(dm_lo)
        capi.check(L.yb200_upsample_bilinear2x_bwd_f32(capi.ptr(g_masks.float().contiguous()), n, ctypes.byref(dma), sp), "bilinear x2 bwd")
        # 2. mask GEMM, per image: d kernel = dM^T mf (pixel contraction), d mf = dM kernel
        dkernel = torch.empty(b, npad, kd, device=dev)
        dmf = torch.empty_like(mf)
        for i in range(b):
            ma, da, oa = capi.act(mf[i:i + 1]), capi.act(dm_lo[i:i + 1]), capi.act(dmf[i:i + 1])
            self._wgrad(ma, da, 1, dkernel[i])
            capi.check(L.yb200_conv2d_dgrad(ctypes.byref(da), capi.ptr(self._pack_dgrad(kernel[i], npad, kd)), ctypes.byref(oa), None, 1, 1, sp), "mask bmm dgrad")
        # 3. projection (1x1, its input is the last mask conv's ReLU output) and the mask convs
        m = s["m"]
        proj = self.mask_branch.projection
        dz = torch.empty_like(m[-1])
        fa, ma, za = capi.act(dmf), capi.act(m[-1]), capi.act(dz)
        capi.check(L.yb200_linear_dgrad_relu(ctypes.byref(fa), capi.ptr(self._pack_dgrad(proj.weight, kd, self.mask_dim)), ctypes.byref(ma), ctypes.byref(za), None, sp),
                   "projection dgrad + relu bwd")
        self._conv_grads(ma, fa, proj, "mask_branch.projection", grads, need, 1)
        dz0_mask = self._stack_bwd(x, m, dz, self.mask_branch.mask_convs, "mask_branch.mask_convs.", grads, need)
        # 4. heads: d logits | d kernel | d scores as one bf16 [B, 1, Npad, 224] operand (rows >= n zero)
        ib = self.inst_branch
        head_in = s["inst"]
        hd = head_in.shape[-1]
        ncat = ncls + kd + 1
        dh = torch.zeros(b, 1, npad, _pad16(ncat), dtype=bf16, device=dev)
        dh[:, 0, :n, :ncls] = g_logits
        dh[:, 0, :, ncls:ncls + kd] = dkernel
        dh[:, 0, :n, ncls + kd] = g_scores.reshape(b, n)
        wcat = torch.cat([ib.cls_score.weight.detach(), ib.mask_kernel.weight.detach(), ib.objectness.weight.detach()])
        d_in = self._heads_bwd(dh, self._pack_dgrad(wcat, dh.shape[-1], hd), head_in)
        heads = (("cls_score", 0, ncls), ("mask_kernel", ncls, ncls + kd), ("objectness", ncls + kd, ncat))
        ha, dha = capi.act(head_in), capi.act(dh)
        if any(need[f"inst_branch.{k}.weight"] for k, _, _ in heads):
            gw = self._wgrad(ha, dha, 1, torch.empty(dh.shape[-1], hd, device=dev))
            grads.update({f"inst_branch.{k}.weight": gw[lo:hi] for k, lo, hi in heads if need[f"inst_branch.{k}.weight"]})
        if any(need[f"inst_branch.{k}.bias"] for k, _, _ in heads):
            gb = self._colsum(dha, torch.empty(dh.shape[-1], device=dev))
            grads.update({f"inst_branch.{k}.bias": gb[lo:hi] for k, lo, hi in heads if need[f"inst_branch.{k}.bias"]})
        g_inst = self._fc_bwd(d_in, s, grads, need)
        # 5. normalisation: d raw (two bf16 operand layouts) and d normaliser, one launch for the batch
        raw, norm, prob, iam = s["raw"], s["norm"], s["prob"], s["iam"]
        rows = raw.shape[1]
        gin, gout, groups = self._iam_layout()
        if rows != gin * groups:
            raise capi.Yb200Error(f"{type(self).__name__}: backward needs NUM_MASKS * GROUPS maps padded to a multiple of 16 without extra channels")
        draw = torch.empty(b, rows, self.dim, dtype=bf16, device=dev)
        draw_t = torch.empty(b, self.dim, rows, dtype=bf16, device=dev)
        dnorm = torch.empty(b, rows, device=dev)
        ga = capi.act(g_inst)
        capi.check(L.yb200_iam_normalize_bwd(ctypes.byref(ga), capi.ptr(raw), capi.ptr(norm), rows, self.dim, gin, capi.ptr(draw), capi.ptr(draw_t), capi.ptr(dnorm), sp),
                   "iam normalise bwd")
        # 6. aggregation, per image: d prob = F d raw^T + d normaliser;  d F (aggregation) = prob d raw, masked by F > 0
        dprob = torch.empty_like(prob)
        dfagg = torch.empty_like(f)
        for i in range(b):
            fa, pa, qa, ga = capi.act(f[i:i + 1]), capi.act(prob[i:i + 1]), capi.act(dprob[i:i + 1]), capi.act(dfagg[i:i + 1])
            capi.check(L.yb200_conv2d_affine_fwd(ctypes.byref(fa), capi.ptr(draw[i]), None, capi.ptr(dnorm[i]), None, ctypes.byref(qa), 1, 1, sp), "d prob")
            capi.check(L.yb200_linear_dgrad_relu(ctypes.byref(pa), capi.ptr(draw_t[i]), ctypes.byref(fa), ctypes.byref(ga), None, sp), "d F (aggregation)")
        # 7. sigmoid backward into the backward's layout (gout maps per group)
        diam = torch.empty(b, h, w, gout * groups, dtype=bf16, device=dev)
        pa, ia, da = capi.act(dprob, 0, rows), capi.act(iam, 0, rows), capi.act(diam)
        capi.check(L.yb200_sigmoid_bwd(ctypes.byref(pa), ctypes.byref(ia), ctypes.byref(da), gin, gout, sp), "sigmoid bwd")
        # 8. IAM convolution, then the instance convs
        df = self._iam_grads(f, diam, dfagg, grads, need)
        dz0_inst = self._stack_bwd(x, s["f"], df, ib.inst_convs, "inst_branch.inst_convs.", grads, need)
        # 9. d features: the two first-layer data gradients summed (no ReLU: the input is not a ReLU output)
        if not need_x:
            return grads, None
        dxi, dx = torch.empty_like(x), torch.empty_like(x)
        ia, xa, ma, oa = capi.act(dz0_inst), capi.act(dxi), capi.act(dz0_mask), capi.act(dx)
        w_inst, w_mask = ib.inst_convs._modules["0"].weight, self.mask_branch.mask_convs._modules["0"].weight
        capi.check(L.yb200_conv2d_dgrad(ctypes.byref(ia), capi.ptr(self._pack_dgrad(w_inst, self.dim, cpad)), ctypes.byref(xa), None, 3, 1, sp), "input dgrad")
        capi.check(L.yb200_conv2d_dgrad(ctypes.byref(ma), capi.ptr(self._pack_dgrad(w_mask, self.mask_dim, cpad)), ctypes.byref(oa), ctypes.byref(xa), 3, 1, sp),
                   "input dgrad")
        return grads, dx[..., 2:self.in_channels].permute(0, 3, 1, 2).float().contiguous()

    def _heads_bwd(self, dh, wd, head_in):
        """d head input = dh W_heads (the instance features are no ReLU output)"""
        d_in = torch.empty_like(head_in)
        za, oa = capi.act(dh), capi.act(d_in)
        capi.check(self.L.yb200_conv2d_dgrad(ctypes.byref(za), capi.ptr(wd), ctypes.byref(oa), None, 1, 1, capi.stream_ptr()), "heads dgrad")
        return d_in

    def _fc_bwd(self, d_in, s, grads, need):
        """the gradient of the aggregated instance features (Base: the heads' input itself)"""
        return d_in


class _DecoderFn(torch.autograd.Function):
    """one SparseInst decoder as one autograd node: args (decoder, features, *parameters in named_parameters() order) -> (pred_logits,
    pred_masks, pred_scores); the backward returns d features (fp32 NCHW) and every parameter's fp32 gradient"""

    @staticmethod
    def forward(ctx, dec, features, *params):
        saved = {}
        out = dec._run(features, saved)
        ctx.dec, ctx.saved = dec, saved
        return out["pred_logits"], out["pred_masks"], out["pred_scores"]

    @staticmethod
    def backward(ctx, g_logits, g_masks, g_scores):
        dec = ctx.dec
        names = [n for n, _ in dec.named_parameters()]
        need = dict(zip(names, ctx.needs_input_grad[2:]))
        grads, dfeat = dec._backward(ctx.saved, g_logits, g_masks, g_scores, ctx.needs_input_grad[1], need)
        ctx.saved = None
        return (None, dfeat) + tuple(grads.get(n) for n in names)


class GroupIAMDecoder(BaseIAMDecoder):
    """decoder_sparseinst.py:172-250: `GroupInstanceBranch` -- a GROUPED 3x3 IAM convolution (G groups of dim/G input channels, N maps each), the
    aggregation over all N*G maps, the G features of one instance concatenated ([B, N, G*dim]), fc + ReLU, then the heads.  Extra cfg key
    MODEL.SPARSE_INST.DECODER.GROUPS.  The grouped convolution is G implicit-GEMM launches on channel-slice views of the same tensors
    (each group padded to a multiple of 8 maps with bias -30, i.e. probability 0)."""

    def _build_iam(self, dev, prior):
        self.groups = int(self._cfg_groups)
        if self.dim % (16 * self.groups):
            raise capi.Yb200Error("GroupIAMDecoder: INST.DIM / GROUPS must be a multiple of 16")
        self.inst_branch.iam_conv = _Conv(self.dim // self.groups, self.num_masks * self.groups, 3, dev, 0.01)
        with torch.no_grad():
            self.inst_branch.iam_conv.bias.fill_(prior)
        expand = self.dim * self.groups
        self.inst_branch.fc = _Linear(expand, expand, dev, std=(1.0 / expand) ** 0.5)
        return expand

    def __init__(self, cfg, device="cuda"):
        self._cfg_groups = cfg.MODEL.SPARSE_INST.DECODER.GROUPS
        super().__init__(cfg, device)

    def _instances(self, f, save=None):
        L, sp = self.L, capi.stream_ptr()
        b, h, w, _ = f.shape
        dev = f.device
        n, g = self.num_masks, self.groups
        np8 = (n + 7) // 8 * 8                   # maps per group, padded
        ctot = _pad16(np8 * g)
        cg = self.dim // g
        conv = self.inst_branch.iam_conv
        iam = torch.zeros(b, h, w, ctot, dtype=torch.bfloat16, device=dev)
        for k in range(g):                       # nn.Conv2d(dim, N*G, 3, padding=1, groups=G) (:186-188): group k reads channels [k*cg, (k+1)*cg)
            bias = torch.full((np8,), -30.0, device=dev)
            bias[:n] = conv.bias.detach()[k * n:(k + 1) * n]
            wk = self._pack(conv.weight[k * n:(k + 1) * n], np8, cg)
            fa, ia = capi.act(f, k * cg, cg), capi.act(iam, k * np8, np8)
            capi.check(L.yb200_conv2d_affine_fwd(ctypes.byref(fa), capi.ptr(wk), None, capi.ptr(bias), None, ctypes.byref(ia), 3, 1, sp), "grouped iam_conv")
        if ctot > np8 * g:
            iam[..., np8 * g:] = -30.0           # alignment padding of the channel count: probability 0
        prob = torch.empty_like(iam)
        ia, pa = capi.act(iam), capi.act(prob)
        capi.check(L.yb200_sigmoid(ctypes.byref(ia), ctypes.byref(pa), sp), "sigmoid")
        inst = self._aggregate(f, prob, save)    # [B, 1, ctot, dim]; row k*np8 + i = map i of group k
        # reshape(B, 4, N, C).transpose(1, 2).reshape(B, N, 4C) (:231-235): the G features of instance i side by side
        v = inst[:, 0, :np8 * g].view(b, g, np8, self.dim)[:, :, :n].permute(0, 2, 1, 3).reshape(b, n, g * self.dim)
        npad = _pad16(n)
        x = torch.zeros(b, 1, npad, g * self.dim, dtype=torch.bfloat16, device=dev)
        x[:, 0, :n] = v
        fc = self.inst_branch.fc
        y = torch.empty_like(x)
        xa, ya = capi.act(x), capi.act(y)
        capi.check(L.yb200_conv2d_relu_fwd(ctypes.byref(xa), capi.ptr(self._pack(fc.weight, fc.weight.shape[0], x.shape[-1])), capi.ptr(fc.bias.detach()), ctypes.byref(ya),
                                           1, 1, sp), "fc + relu")
        iam_out = torch.cat([iam[..., k * np8:k * np8 + n] for k in range(g)], -1)  # the reference's channel order: group-major, N per group
        if save is not None:
            save.update(iam=iam, xg=x, inst=y)
        return y, iam_out

    # ---- backward ----------------------------------------------------------------------------------------------------------------
    def _iam_layout(self):
        """the forward's IAM maps are np8 per group (a multiple of 8); the backward's d iam has gout per group, a width the data- and
        weight-gradient GEMMs take as a channel slice (16, 32 or a multiple of 64: 128 for 100 masks); maps >= N of each group are zero"""
        np8 = (self.num_masks + 7) // 8 * 8
        gout = 16 if np8 <= 16 else (32 if np8 <= 32 else (np8 + 63) // 64 * 64)
        return np8, gout, self.groups

    def _heads_bwd(self, dh, wd, head_in):
        """d fc pre-activation = dh W_heads masked by the fc's ReLU output"""
        d_in = torch.empty_like(head_in)
        za, ha, oa = capi.act(dh), capi.act(head_in), capi.act(d_in)
        capi.check(self.L.yb200_linear_dgrad_relu(ctypes.byref(za), capi.ptr(wd), ctypes.byref(ha), ctypes.byref(oa), None, capi.stream_ptr()), "heads dgrad + relu bwd")
        return d_in

    def _fc_bwd(self, d_in, s, grads, need):
        """fc's gradients and the gradient of its input [B, 1, Npad, G*dim] (instance i, group k at columns k*dim: the normalisation backward
        reads it through its row map)"""
        xg, fc = s["xg"], self.inst_branch.fc
        za = capi.act(d_in)
        self._conv_grads(capi.act(xg), za, fc, "inst_branch.fc", grads, need, 1)
        g = torch.empty_like(xg)
        oa = capi.act(g)
        capi.check(self.L.yb200_conv2d_dgrad(ctypes.byref(za), capi.ptr(self._pack_dgrad(fc.weight, fc.weight.shape[0], xg.shape[-1])), ctypes.byref(oa), None, 1, 1,
                                             capi.stream_ptr()), "fc dgrad")
        return g

    def _iam_grads(self, f, diam, dfagg, grads, need):
        """the grouped IAM convolution: one data-gradient launch per group on channel slices (gout-wide slices of d iam, cg-wide of F)"""
        L, sp = self.L, capi.stream_ptr()
        n, g = self.num_masks, self.groups
        _, gout, _ = self._iam_layout()
        cg = self.dim // g
        conv = self.inst_branch.iam_conv
        df = torch.empty_like(f)
        gw = torch.empty(g * n, cg, 3, 3, device=f.device) if need["inst_branch.iam_conv.weight"] else None
        for k in range(g):
            za, fa, da, aa = capi.act(diam, k * gout, gout), capi.act(f, k * cg, cg), capi.act(df, k * cg, cg), capi.act(dfagg, k * cg, cg)
            capi.check(L.yb200_conv2d_dgrad_relu(ctypes.byref(za), capi.ptr(self._pack_dgrad(conv.weight[k * n:(k + 1) * n], gout, cg)), ctypes.byref(fa),
                                                 ctypes.byref(da), ctypes.byref(aa), 3, 1, sp), "grouped iam_conv dgrad + relu bwd")
            if gw is not None:
                gw[k * n:(k + 1) * n] = self._wgrad(fa, za, 3, torch.empty(gout, cg, 3, 3, device=f.device))[:n]
        if gw is not None:
            grads["inst_branch.iam_conv.weight"] = gw
        if need["inst_branch.iam_conv.bias"]:
            gb = self._colsum(capi.act(diam), torch.empty(g * gout, device=f.device))
            grads["inst_branch.iam_conv.bias"] = gb.view(g, gout)[:, :n].reshape(g * n)
        return df


def _register():
    try:
        from detectron2.utils.registry import Registry  # pragma: no cover
    except Exception:  # noqa: BLE001
        return
    try:  # pragma: no cover
        from yolov7.modeling.transcoders.decoder_sparseinst import SPARSE_INST_DECODER_REGISTRY
        SPARSE_INST_DECODER_REGISTRY._obj_map["BaseIAMDecoder"] = BaseIAMDecoder
        SPARSE_INST_DECODER_REGISTRY._obj_map["GroupIAMDecoder"] = GroupIAMDecoder
    except Exception:  # noqa: BLE001
        pass


_register()
