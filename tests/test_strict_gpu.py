"""north_star: "fp32 losses and logits within 1e-3 relative" -- checked literally, on the GPU, in STRICT mode.

YoloxEngine(strict=True) (or YB200_STRICT=1) runs the same plan on the same wgmma implicit-GEMM kernel, but every activation and
weight is a sum of three bf16 planes (a0 + a1 + a2 = all 24 significant bits of the fp32 value; csrc/strict.cu; YB200_STRICT_PLANES=2 keeps
16 bits) multiplied as the six products a_i * w_j with i + j < 3 into the fp32 accumulator, with fp32 pre-BatchNorm outputs and fp64
batch statistics.  The result is compared with the fp32 CPU oracle
(oracle/yolox_oracle.py, pinned to the reference by tests/golden/*):
    head outputs (decoded boxes, objectness and class logits): |err| <= 1e-3 * max(1, |ref|)   elementwise
    the four losses:                                            relative 1e-3
    SimOTA assignment:                                          identical to the oracle's on the oracle's own head outputs
Weights are full fp32 values (NOT bf16-representable), so the lo planes carry signal.
"""
import numpy as np
import pytest
import torch

from oracle import yolox_oracle as orc

pytestmark = pytest.mark.gpu
TOL = 1e-3  # north_star: "fp32 losses and logits within 1e-3 relative"


def _fp32_state_dict(seed):
    sd = orc.yolox_state_dict(seed)
    g = torch.Generator().manual_seed(seed + 99)
    for k in sd:
        if k.endswith(".conv.weight") or ("preds" in k and k.endswith(".weight")):
            sd[k] = sd[k] * (1 + 3e-3 * torch.randn(sd[k].shape, generator=g))  # no longer representable in bf16
        if k.endswith(".bn.weight"):
            sd[k] = torch.rand(sd[k].shape, generator=g) * 0.5 + 0.75
        if k.endswith(".bn.bias"):
            sd[k] = torch.randn(sd[k].shape, generator=g) * 0.1
    assert not torch.equal(sd["backbone.dark3.0.conv.weight"], sd["backbone.dark3.0.conv.weight"].to(torch.bfloat16).float())
    return sd


def _run(cuda, batch, size, seed, max_gt):
    from yolov7_d2_b200.engine import YoloxEngine

    sd = _fp32_state_dict(seed)
    images, labels = orc.synthetic_batch(batch, size, seed + 1, max_gt=max_gt, empty_every=4)
    eng = YoloxEngine(batch, size, size, device=cuda, strict=True)
    eng.load_state_dict(sd)
    eng.images_u8.copy_(images.to(cuda))
    eng.labels.copy_(labels.to(cuda))
    eng.train_step()
    torch.cuda.synchronize()
    with torch.no_grad():
        total, iou5, lobj, lcls, ratio, ref_out = orc.yolox_forward_train(images.float(), labels, {k: v.clone() for k, v in sd.items()})
    return eng, labels, np.array([float(total), float(iou5), float(lobj), float(lcls)]), float(ratio), ref_out


@pytest.mark.parametrize("batch,size,max_gt", [(8, 256, 6), (4, 640, 12)])
def test_strict_logits_and_losses_within_1e3(cuda, batch, size, max_gt):
    eng, labels, ref_losses, ref_ratio, ref_out = _run(cuda, batch, size, 31 + size, max_gt)
    out = eng.outputs.cpu()
    # LOGITS = the raw head outputs: objectness / class logits as stored, box regression outputs with the (exact, monotonic) decode
    # undone -- raw_xy = xy / stride - grid, raw_wh = log(wh / stride)   (yolox_head.py:226-245)
    xs, ys, ss = orc.anchor_grid([(h, w) for h, w, _, _ in eng.levels])
    xs, ys, ss = xs[None, :, None].double(), ys[None, :, None].double(), ss.double()
    ss3 = ss[None, :, None]
    def raw(o):
        o = o.double()
        return torch.cat([o[..., 0:1] / ss3 - xs, o[..., 1:2] / ss3 - ys, torch.log(o[..., 2:4] / ss3), o[..., 4:]], -1)

    r_out, r_ref = raw(out), raw(ref_out)
    err = (r_out - r_ref).abs()
    rel = err / r_ref.abs().clamp(min=1.0)
    print("strict %dx%d bs%d (%d bf16 planes): max relative error of the raw box outputs %.2e, of the obj/cls logits %.2e (mean %.2e); the 16-bit "
          "training engine sits near 3e-2" % (size, size, batch, eng.planes, rel[..., :4].max(), rel[..., 4:].max(), rel.mean()))
    assert bool((err <= TOL * r_ref.abs().clamp(min=1.0)).all()), "raw head outputs deviate from the fp32 oracle by more than 1e-3: max rel %.3e" % rel.max()
    # decoded boxes in pixels: 1e-3 of the anchor stride (xy) / 1e-3 relative (wh)
    assert bool(((out[..., :2] - ref_out[..., :2]).abs() <= TOL * ss3.float() * (ref_out[..., :2].abs() / ss3.float()).clamp(min=1.0)).all())
    assert bool(((out[..., 2:4] - ref_out[..., 2:4]).abs() <= 2 * TOL * ref_out[..., 2:4].abs() * r_ref[..., 2:4].abs().clamp(min=1.0).float()).all())
    got = eng.losses.cpu().double().numpy()
    print("losses strict", got[:4], "oracle", ref_losses)
    assert np.allclose(got[:4], ref_losses, rtol=1e-3, atol=0.0), (got, ref_losses)
    assert abs(got[5] - ref_ratio) <= 1e-3 * max(ref_ratio, 1.0)
    # the assignment made on the strict head outputs is the one the oracle makes on ITS head outputs
    xs, ys, ss = orc.anchor_grid([(h, w) for h, w, _, _ in eng.levels])
    assigns = orc.yolox_losses(ref_out, labels, xs, ys, ss, return_assign=True)[-1]
    fg = eng.fg_mask.cpu().bool()
    same = sum(int(torch.equal(fg[b], a[0])) for b, a in enumerate(assigns))
    assert same == len(assigns), f"SimOTA foreground masks differ on {len(assigns) - same} of {len(assigns)} images"


def test_strict_eval_probabilities_within_1e3(cuda):
    from yolov7_d2_b200.engine import YoloxEngine

    sd = _fp32_state_dict(77)
    g = torch.Generator().manual_seed(5)
    for k in sd:  # non-trivial running statistics
        if k.endswith("running_mean"):
            sd[k] = torch.randn(sd[k].shape, generator=g) * 0.1
        if k.endswith("running_var"):
            sd[k] = torch.rand(sd[k].shape, generator=g) * 0.5 + 0.75
    images, _ = orc.synthetic_batch(4, 256, 78)
    eng = YoloxEngine(4, 256, 256, device=cuda, strict=True)
    eng.load_state_dict(sd)
    eng.images_u8.copy_(images.to(cuda))
    out = eng.eval_forward().cpu()
    with torch.no_grad():
        ref = orc.yolox_forward_eval(images.float(), sd)
    err = (out - ref).abs()
    assert bool((err <= 1e-3 * ref.abs().clamp(min=1.0)).all()), float((err / ref.abs().clamp(min=1.0)).max())


def test_strict_has_no_backward(cuda):
    from yolov7_d2_b200 import capi
    from yolov7_d2_b200.engine import YoloxEngine

    eng = YoloxEngine(1, 64, 64, device=cuda, strict=True)
    with pytest.raises(capi.Yb200Error):
        eng.backward()
