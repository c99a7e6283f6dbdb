"""SparseInst IAM decoder on the H100 kernels (forward path; SURVEY.md par.8a row S1).

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
Scope: forward (inference; the decoder backward is not built): runs under no_grad.  The matcher and the losses of sparseinst_loss.py, with
their gradients w.r.t. this module's outputs, are `sparseinst_criterion.py`.
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

    def _branch(self, x, seq, n):
        cin_pad = x.shape[-1]
        for i in range(n):
            x = self._conv_relu(x, getattr(seq, str(2 * i)), cin_pad)
            cin_pad = x.shape[-1]
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

    def _aggregate(self, f, prob):
        """inst[b] = prob[b]^T f[b] / clamp(sum prob[b], 1e-6)   (:70-76): the pixel contraction is the weight-gradient GEMM (MN-major wgmma
        descriptors on the NHWC tiles), per image; returns bf16 [B, 1, C_prob, dim]"""
        L, sp = self.L, capi.stream_ptr()
        b, dev, npad = f.shape[0], f.device, prob.shape[-1]
        inst = torch.empty(b, 1, npad, self.dim, dtype=torch.bfloat16, device=dev)
        raw = torch.empty(npad, self.dim, device=dev)
        norm = torch.empty(npad, device=dev)
        f1, p1 = capi.act(f[0:1]), capi.act(prob[0:1])
        ws_g = torch.empty(max(int(L.yb200_conv2d_wgrad_workspace(ctypes.byref(f1), ctypes.byref(p1), 1, 1)), 16), dtype=torch.uint8, device=dev)
        ws_c = torch.empty(max(int(L.yb200_colsum_workspace(ctypes.byref(p1))), 16), dtype=torch.uint8, device=dev)
        for i in range(b):
            fi, pi, oi = capi.act(f[i:i + 1]), capi.act(prob[i:i + 1]), capi.act(inst[i:i + 1])
            capi.check(L.yb200_conv2d_wgrad(ctypes.byref(fi), ctypes.byref(pi), 1, 1, self.dim, capi.ptr(raw), 0, capi.ptr(ws_g), ctypes.c_int64(ws_g.numel()), sp), "iam bmm")
            capi.check(L.yb200_colsum(ctypes.byref(pi), ctypes.c_float(1.0), capi.ptr(norm), 0, capi.ptr(ws_c), sp), "iam normaliser")
            capi.check(L.yb200_iam_normalize(capi.ptr(raw), capi.ptr(norm), npad, self.dim, ctypes.byref(oi), sp), "iam normalise")
        return inst

    def _instances(self, f):
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
        return self._aggregate(f, prob), iam[..., :n]

    # ---- forward -----------------------------------------------------------------------------------------------------------------
    @torch.no_grad()
    def forward(self, features):
        if not features.is_cuda:
            raise capi.Yb200Error("BaseIAMDecoder: input must be a CUDA tensor (no CPU path)")
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
        # instance branch
        f = self._branch(x, self.inst_branch.inst_convs, self.num_convs)
        n = self.num_masks
        inst, iam = self._instances(f)  # [B, 1, Npad, head_dim] bf16 instance features; iam logits [B, n, H, W]-shaped source (NHWC slice)
        npad = inst.shape[2]
        ib = self.inst_branch
        logits = self._heads_f32(inst, ib.cls_score, self.num_classes)[:, :n]
        kernel = self._heads_f32(inst, ib.mask_kernel, self.kernel_dim)            # [B, Npad, kernel_dim] (padded instances: bias only)
        scores = self._heads_f32(inst, ib.objectness, 1)[:, :n]
        # mask branch
        m = self._branch(x, self.mask_branch.mask_convs, self.mask_convs_n)
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
        out = {"pred_logits": logits, "pred_masks": pred_masks, "pred_scores": scores}
        if self.output_iam:
            out["pred_iam"] = F.interpolate(iam.permute(0, 3, 1, 2).float(), scale_factor=self.scale_factor, mode="bilinear", align_corners=False)
        # kept for tests / callers that want the un-interpolated tensors
        self.last = {"pred_kernel": kernel[:, :n], "iam": iam, "masks_lowres": masks[:, :n]}
        return out


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

    def _instances(self, f):
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
        inst = self._aggregate(f, prob)          # [B, 1, ctot, dim]; row k*np8 + i = map i of group k
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
        return y, iam_out


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
