"""TEST INFRASTRUCTURE -- the SparseInst IAM decoder of oracle/sparseinst_oracle.py with bf16 storage emulated: values, and the gradients flowing
back through them, are rounded to bf16 at the points where the kernels store bf16 (the input, every convolution's output and its gradient, the IAM
probabilities, the instance features, the mask features, the GEMM weights and the bf16 gradient operands of the heads and of the masks before
up-sampling).  Run in float64, it is the yardstick of what 16-bit storage alone costs against the fp64 oracle, as EMULATE_STORAGE of
oracle/yolox_oracle.py is for YOLOX.  Same arguments and outputs as sparseinst_oracle.decoder_forward (without masks_lowres).
Only tests/ and tools/ may import it.
"""
import torch
import torch.nn.functional as F

from .sparseinst_oracle import coordinates


class _Bf16(torch.autograd.Function):
    """bf16 rounding of a stored value and of its gradient"""

    @staticmethod
    def forward(ctx, x):
        return x.to(torch.bfloat16).to(x.dtype)

    @staticmethod
    def backward(ctx, g):
        return g.to(torch.bfloat16).to(g.dtype)


class _GradBf16(torch.autograd.Function):
    """identity forward (an fp32 output), bf16 rounding of the gradient (a bf16 gradient operand)"""

    @staticmethod
    def forward(ctx, x):
        return x.view_as(x)

    @staticmethod
    def backward(ctx, g):
        return g.to(torch.bfloat16).to(g.dtype)


class _WeightBf16(torch.autograd.Function):
    """bf16 rounding of a GEMM operand packed from fp32 (the weights, the predicted mask kernels); its gradient stays fp32"""

    @staticmethod
    def forward(ctx, x):
        return x.to(torch.bfloat16).to(x.dtype)

    @staticmethod
    def backward(ctx, g):
        return g


_s, _sg, _w = _Bf16.apply, _GradBf16.apply, _WeightBf16.apply


def _stack(x, sd, prefix, n):
    for i in range(n):
        x = F.relu(_s(F.conv2d(x, _w(sd[f"{prefix}{2 * i}.weight"]), sd[f"{prefix}{2 * i}.bias"], padding=1)))
    return x


def _heads(inst, sd, prefix):
    return tuple(_sg(F.linear(inst, _w(sd[prefix + k + ".weight"]), sd[prefix + k + ".bias"])) for k in ("cls_score", "mask_kernel", "objectness"))


def _instances(f, sd, prefix, groups):
    """InstanceBranch (:62-81) / GroupInstanceBranch (:212-242) after the instance convs"""
    iam = _s(F.conv2d(f, _w(sd[prefix + "iam_conv.weight"]), sd[prefix + "iam_conv.bias"], padding=1, groups=groups or 1))
    prob = _s(iam.sigmoid())
    b, n = prob.shape[:2]
    c = f.shape[1]
    prob = prob.view(b, n, -1)
    inst = torch.bmm(prob, _sg(f).view(b, c, -1).permute(0, 2, 1))
    norm = prob.sum(-1).clamp(min=1e-6, max=1e5) if groups else prob.sum(-1).clamp(min=1e-6)
    inst = _s(inst / norm[:, :, None])
    if groups:
        inst = inst.reshape(b, 4, n // 4, -1).transpose(1, 2).reshape(b, n // 4, -1)
        inst = F.relu(_s(F.linear(inst, _w(sd[prefix + "fc.weight"]), sd[prefix + "fc.bias"])))
    return _heads(inst, sd, prefix) + (iam,)


def decoder_forward(features, sd, scale_factor=2.0, num_convs=4, groups=0):
    """BaseIAMDecoder.forward (:130-169; groups > 0: GroupIAMDecoder) with the kernels' bf16 storage points"""
    x = _s(torch.cat([coordinates(features), features], 1))
    logits, kernel, scores, iam = _instances(_stack(x, sd, "inst_branch.inst_convs.", num_convs), sd, "inst_branch.", groups)
    m = _stack(x, sd, "mask_branch.mask_convs.", num_convs)
    mf = _s(F.conv2d(m, _w(sd["mask_branch.projection.weight"]), sd["mask_branch.projection.bias"]))
    b, c, h, w = mf.shape
    masks = _sg(torch.bmm(_w(kernel), mf.view(b, c, h * w)).view(b, kernel.shape[1], h, w))
    masks = F.interpolate(masks, scale_factor=scale_factor, mode="bilinear", align_corners=False)
    return {"pred_logits": logits, "pred_masks": masks, "pred_scores": scores, "pred_kernel": kernel, "iam": iam}
