"""End-to-end GPU parity of the YOLOX-s engine (forward, SimOTA + loss, backward) against the CPU oracle.

The engine stores activations in 16 bits (pre-BN conv outputs fp16, activations / gradients bf16).  A randomly initialised
BatchNorm network amplifies storage rounding (BatchNorm divides by small batch standard deviations), so the fp32 oracle
cannot be matched to 1e-3 end to end by ANY 16-bit implementation.  The yardstick is therefore the storage-emulating
oracle (`orc.EMULATE_STORAGE`: identical math in fp32 but rounded at the engine's storage points):
  * forward: |engine - fp32 oracle| must not exceed 1.5 x |emulating oracle - fp32 oracle| (mean abs error of the head logits);
  * loss / SimOTA on the engine's own head outputs: indices bit-exact, losses 1e-4 (the kernels under test are fp32);
  * parameter gradients: cosine similarity to the fp32 oracle within 0.05 of the emulating oracle's, and >= 0.9.
"""
import numpy as np
import pytest
import torch

from oracle import yolox_oracle as orc

pytestmark = pytest.mark.gpu


def _oracle_step(sd, images, labels, emulate):
    orc.EMULATE_STORAGE = emulate
    try:
        sd = {k: v.clone() for k, v in sd.items()}
        for k, v in sd.items():
            if v.dtype == torch.float32 and "running" not in k:
                v.requires_grad_(True)
        total, iou5, lobj, lcls, ratio, outputs = orc.yolox_forward_train(images.float(), labels, sd)
        total.backward()
    finally:
        orc.EMULATE_STORAGE = False
    return dict(losses=np.array([float(total), float(iou5), float(lobj), float(lcls), float(ratio)]), outputs=outputs.detach(), sd=sd)


@pytest.fixture(scope="module")
def step(cuda):
    from yolov7_d2_b200.engine import YoloxEngine

    batch, size = 8, 256
    sd = orc.yolox_state_dict(3)
    g = torch.Generator().manual_seed(9)
    for k in sd:  # non-trivial BN affine parameters so that the gamma/beta gradients and scale/shift paths are exercised
        if k.endswith(".bn.weight"):
            sd[k] = (torch.rand(sd[k].shape, generator=g) * 0.5 + 0.75)
        if k.endswith(".bn.bias"):
            sd[k] = torch.randn(sd[k].shape, generator=g) * 0.1
    images, labels = orc.synthetic_batch(batch, size, 5, max_gt=6, empty_every=4)
    eng = YoloxEngine(batch, size, size, device=cuda)
    eng.load_state_dict(sd)
    eng.images_u8.copy_(images.to(cuda))
    eng.labels.copy_(labels.to(cuda))
    eng.train_step()
    torch.cuda.synchronize()
    torch.set_num_threads(max(1, torch.get_num_threads()))
    ref = _oracle_step(sd, images, labels, False)
    emu = _oracle_step(sd, images, labels, True)
    return dict(eng=eng, ref=ref, emu=emu, images=images, labels=labels, sd0=sd)


def test_forward_logits(step):
    eng, ref, emu = step["eng"], step["ref"], step["emu"]
    out = eng.outputs.cpu()
    e_eng = (out - ref["outputs"]).abs()[..., 4:]
    e_emu = (emu["outputs"] - ref["outputs"]).abs()[..., 4:]
    print("logit error vs fp32 oracle: engine mean %.5f max %.4f | emulating oracle mean %.5f max %.4f" %
          (e_eng.mean(), e_eng.max(), e_emu.mean(), e_emu.max()))
    assert e_eng.mean() <= 1.5 * e_emu.mean() + 1e-4
    def corr(t):
        a, b = t[..., 4:].flatten().double(), ref["outputs"][..., 4:].flatten().double()
        return float(((a - a.mean()) * (b - b.mean())).mean() / (a.std() * b.std()))

    c_eng, c_emu = corr(out), corr(emu["outputs"])
    print("logit correlation with the fp32 oracle: engine %.5f, emulating oracle %.5f" % (c_eng, c_emu))
    assert c_eng >= c_emu - 0.003 and c_eng >= 0.99


def test_loss_and_simota_on_engine_outputs(step):
    """same inputs -> bit-exact assignment and fp32 losses (the reference's parity rule for SimOTA / losses)"""
    eng, labels = step["eng"], step["labels"]
    out = eng.outputs.cpu()
    xs, ys, ss = orc.anchor_grid([(h, w) for h, w, _, _ in eng.levels])
    total, iou5, lobj, lcls, ratio, assigns = orc.yolox_losses(out, labels, xs, ys, ss, return_assign=True)
    fg = eng.fg_mask.cpu().bool()
    for b, (rfg, mgt, mcls, miou) in enumerate(assigns):
        assert torch.equal(fg[b], rfg), f"image {b}"
        assert torch.equal(eng.matched_gt.cpu()[b][rfg].long(), mgt)
        assert torch.equal(eng.matched_iou.cpu()[b][rfg], miou)
    got = eng.losses.cpu().double().numpy()
    ref = np.array([float(total), float(iou5), float(lobj), float(lcls), 0.0, float(ratio)])
    assert np.allclose(got, ref, rtol=1e-4, atol=1e-5), (got, ref)


def test_losses_close_to_fp32_model(step):
    got = step["eng"].losses.cpu().double().numpy()[[0, 1, 2, 3, 5]]
    ref, emu = step["ref"]["losses"], step["emu"]["losses"]
    print("losses engine", got, "fp32", ref, "emulating", emu)
    assert np.all(np.abs(got - ref) <= 1.5 * np.abs(emu - ref) + 2e-2 * np.abs(ref) + 1e-3), (got, ref, emu)


def test_bn_running_stats(step):
    eng, ref_sd = step["eng"], step["ref"]["sd"]
    for name in ("backbone.stem.conv.bn", "backbone.dark3.1.m.1.conv2.bn", "neck.C3_n4.conv3.bn", "head.reg_convs.2.1.bn"):
        rm, rv = eng.buffers[name + ".running_mean"].cpu(), eng.buffers[name + ".running_var"].cpu()
        assert torch.allclose(rm, ref_sd[name + ".running_mean"], rtol=3e-2, atol=3e-3), name
        assert torch.allclose(rv, ref_sd[name + ".running_var"], rtol=3e-2, atol=3e-3), name
        assert int(eng.buffers[name + ".num_batches_tracked"]) == 1


def _linear_functional_grads(sd, images, g_raw, emulate):
    """d/d params of  sum(G * raw head outputs)  -- no discrete decision (SimOTA) between parameters and objective"""
    orc.EMULATE_STORAGE = emulate
    try:
        sd = {k: v.clone() for k, v in sd.items()}
        for k, v in sd.items():
            if v.dtype == torch.float32 and "running" not in k:
                v.requires_grad_(True)
        raw = orc.head_raw(orc.pafpn(orc.csp_darknet(images.float(), sd, True), sd, True), sd, True)
        flat = torch.cat([r.permute(0, 2, 3, 1).reshape(r.shape[0], -1, r.shape[1]) for r in raw], 1)
        (flat * g_raw).sum().backward()
    finally:
        orc.EMULATE_STORAGE = False
    return {k: v.grad for k, v in sd.items() if v.requires_grad}


def test_backward_against_oracle(step, cuda):
    """conv / BatchNorm / SPP / upsample / residual backward of the whole network for a fixed upstream gradient G on the raw
    head outputs (the loss kernel's own gradient is verified bit-level against the reference in test_simota_gpu.py)."""
    eng, images, sd0 = step["eng"], step["images"], step["sd0"]
    gen = torch.Generator().manual_seed(77)
    n, a, ch = eng.outputs.shape
    g_raw = (torch.randn(n, a, ch, generator=gen) * 1e-2).to(torch.bfloat16).float()
    eng.load_state_dict(sd0)
    eng.pack_weights()
    eng.preprocess()
    eng.forward_features(True)
    for k, (h, w, s, a_off) in enumerate(eng.levels):
        gl = g_raw[:, a_off:a_off + h * w]
        eng.d_cls[k].copy_(gl[..., 5:].reshape(n, h, w, ch - 5).to(cuda))
        eng.d_ro[k].zero_()
        eng.d_ro[k][..., :5].copy_(gl[..., :5].reshape(n, h, w, 5).to(cuda))
        eng.bias_acc[k].copy_(gl.double().sum((0, 1)).to(cuda))
    eng.backward()
    torch.cuda.synchronize()
    ref = _linear_functional_grads(sd0, images, g_raw, False)
    emu = _linear_functional_grads(sd0, images, g_raw, True)
    rows = []
    for name in eng.param_names:
        g = eng.grads[name].cpu().flatten().double()
        r, e = ref[name].flatten().double(), emu[name].flatten().double()
        cos = float((g @ r) / (g.norm() * r.norm() + 1e-30))
        cos_e = float((e @ r) / (e.norm() * r.norm() + 1e-30))
        rows.append((cos, cos_e, float(g.norm() / (r.norm() + 1e-30)), name))
    rows.sort()
    print("lowest cosine similarity to the fp32 oracle (engine, emulating oracle, norm ratio):")
    for r in rows[:10]:
        print("   %.4f %.4f %.3f %s" % r)
    for cos, cos_e, ratio, name in rows:
        assert cos >= cos_e - 0.03 and cos >= 0.9 and 0.85 <= ratio <= 1.18, (name, cos, cos_e, ratio)


def test_second_step_is_reproducible(step):
    """a second identical step reproduces the same result (no stale accumulators; fp64 atomics are the only reordering)"""
    eng = step["eng"]
    eng.load_state_dict(step["sd0"])
    eng.train_step()
    torch.cuda.synchronize()
    g1, l1 = eng.flat_grad.clone(), eng.losses.clone()
    eng.load_state_dict(step["sd0"])
    eng.train_step()
    torch.cuda.synchronize()
    assert torch.allclose(l1, eng.losses, rtol=1e-6)
    rel = (g1 - eng.flat_grad).abs().max() / g1.abs().max()
    # block reductions run in a fixed order; only fp64 atomics are unordered (1e-16) -- but a single flipped bf16 rounding is
    # amplified by the backward chain of BatchNorms, so allow a small residue rather than demanding bit equality
    assert rel <= 2e-3, rel.item()


def test_eval_forward_matches_oracle(step):
    eng, images = step["eng"], step["images"]
    sd = {k: v.detach() for k, v in step["ref"]["sd"].items()}  # running statistics after the oracle's training step
    eng.load_state_dict(sd)
    out = eng.eval_forward().cpu()
    with torch.no_grad():
        ref = orc.yolox_forward_eval(images.float(), sd)
        orc.EMULATE_STORAGE = True
        try:
            emu = orc.yolox_forward_eval(images.float(), sd)
        finally:
            orc.EMULATE_STORAGE = False
    e_eng, e_emu = (out - ref).abs()[..., 4:], (emu - ref).abs()[..., 4:]
    print("eval prob error: engine mean %.6f | emulating %.6f" % (e_eng.mean(), e_emu.mean()))
    assert e_eng.mean() <= 1.5 * e_emu.mean() + 1e-5


def test_pixel_grouped_stem_equals_plain_stem(step, cuda, monkeypatch):
    """YB200_STEM_GROUP4 (default on): the stem convolution and its weight gradient run on [N, H, W/4, 64] views (128-byte TMA rows) with an
    expanded weight matrix; same pre-BatchNorm output, statistics and parameter gradient as the plain 16-channel formulation"""
    from yolov7_d2_b200.engine import YoloxEngine

    sd0 = step["sd0"]
    engs = []
    for flag in ("1", "0"):
        monkeypatch.setenv("YB200_STEM_GROUP4", flag)
        e = YoloxEngine(step["eng"].n, step["eng"].h, step["eng"].w, device=cuda)
        assert e.group4 == (flag == "1")
        e.load_state_dict(sd0)
        e.images_u8.copy_(step["images"].to(cuda))
        e.labels.copy_(step["labels"].to(cuda))
        e.train_step()
        torch.cuda.synchronize()
        engs.append(e)
    a, b = engs
    za, zb = a.ops[0].z.buf.t.float(), b.ops[0].z.buf.t.float()
    assert (za - zb).abs().max() <= 2.0 ** -9 * zb.abs().max(), "stem pre-BN output"
    n = a.ops[0].cout
    assert torch.allclose(a.flat_mean[:n], b.flat_mean[:n], rtol=1e-4, atol=1e-4) and torch.allclose(a.flat_invstd[:n], b.flat_invstd[:n], rtol=1e-3)
    assert torch.allclose(a.losses, b.losses, rtol=2e-2)
    # weight gradient of the stem alone on IDENTICAL operands (the two plans' whole-step gradients differ by the 16-bit storage noise that the
    # 2^-9 difference above seeds -- cosine ~0.95 between any two noisy runs of this random-weight net, see test_backward_against_oracle)
    sa, sb = a.ops[0], b.ops[0]
    dza, dzb = a._dz_buf(sa), b._dz_buf(sb)
    dzb.t.copy_(dza.t)
    sb.x.buf.t.copy_(sa.x.buf.t)
    for e in engs:
        e.overlap_wgrad = False
    a._wgrad_stem_grouped(sa, dza.t, 0)
    b._wgrad(sb.x.act(), dzb.view().act(), sb.ksize, sb.stride, sb.cin_real, sb.g_dst, 0, "stem")
    torch.cuda.synchronize()
    ga, gb = a.grads["backbone.stem.conv.conv.weight"].flatten().double(), b.grads["backbone.stem.conv.conv.weight"].flatten().double()
    cos = float((ga @ gb) / (ga.norm() * gb.norm()))
    assert cos >= 0.99999 and abs(float(ga.norm() / gb.norm()) - 1) <= 1e-3, (cos, float(ga.norm() / gb.norm()))
