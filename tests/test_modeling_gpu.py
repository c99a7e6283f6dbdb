"""The drop-in surface: registry entries, state_dict layout, YOLOX.forward contract in training and eval mode."""
import numpy as np
import pytest
import torch

from oracle import yolox_oracle as orc


def test_registry_entries_exist_without_gpu():
    from yolov7_d2_b200 import modeling

    assert modeling.META_ARCH_REGISTRY.get("YOLOX") is modeling.YOLOX
    assert modeling.BACKBONE_REGISTRY.get("build_cspdarknetx_backbone") is modeling.build_cspdarknetx_backbone
    with pytest.raises(KeyError):
        modeling.META_ARCH_REGISTRY.get("NoSuchArch")


def test_postprocess_rejects_cpu_tensors():
    from yolov7_d2_b200 import capi, modeling

    with pytest.raises(capi.Yb200Error):
        modeling.postprocess(torch.zeros(1, 10, 85), 80)


@pytest.fixture(scope="module")
def model(cuda):
    import bench
    from yolov7_d2_b200.modeling import YOLOX

    m = YOLOX(bench.yolox_s_cfg("cuda"))
    sd = orc.yolox_state_dict(4)
    m.load_state_dict(sd, strict=True)
    return m, sd


@pytest.mark.gpu
def test_state_dict_layout_matches_reference(model):
    m, sd = model
    got = m.state_dict()
    assert set(got.keys()) == set(sd.keys())
    for k, v in sd.items():
        assert tuple(got[k].shape) == tuple(v.shape), k
        assert torch.equal(got[k].cpu(), v), k
    n_params = sum(p.numel() for p in m.parameters())
    assert abs(n_params - 8.97e6) < 2e4
    assert m.size_divisibility == 32 and m.backbone.size_divisibility == 32
    assert m.backbone.output_shape()["dark5"].channels == 512


@pytest.mark.gpu
def test_forward_training_contract_and_autograd(model, cuda):
    import bench

    m, _ = model
    m.train()
    images, labels = orc.synthetic_batch(2, 128, 11, max_gt=4)
    bi = bench.batched_inputs_from(images, labels)
    out = m(bi)
    assert set(out.keys()) == {"total_loss", "iou_loss", "conf_loss", "cls_loss"}
    total = float(out["total_loss"])
    assert abs(total - float(out["iou_loss"] + out["conf_loss"] + out["cls_loss"])) < 1e-4 * abs(total)
    m.zero_grad(set_to_none=True)
    sum(out.values()).backward()   # detectron2's SimpleTrainer objective: every entry of the dict (= 2 x total)
    g2 = {k: p.grad.clone() for k, p in m.named_parameters()}
    assert all(p.grad is not None and torch.isfinite(p.grad).all() for p in m.parameters())
    m.zero_grad(set_to_none=True)
    out = m(bi)
    out["total_loss"].backward()
    for k, p in m.named_parameters():
        assert torch.allclose(g2[k], 2 * p.grad, rtol=2e-2, atol=1e-3 * float(g2[k].abs().max()) + 1e-8), k


@pytest.mark.gpu
def test_forward_eval_contract(model):
    import bench

    m, _ = model
    m.eval()
    images, labels = orc.synthetic_batch(2, 160, 12, max_gt=4)
    bi = bench.batched_inputs_from(images, labels)
    for b in bi:
        b["height"], b["width"] = 320, 320     # detector_postprocess rescales to the original image size
    res = m(bi)
    assert len(res) == 2 and all("instances" in r for r in res)
    inst = res[0]["instances"]
    n = inst.pred_boxes.tensor.shape[0]
    assert inst.scores.shape == (n,) and inst.pred_classes.shape == (n,)
    assert (inst.pred_boxes.tensor[:, 2] <= 320 + 1e-3).all()
    m.train()


@pytest.mark.gpu
def test_prefetch_gives_identical_steps_and_flat_optimizer_trains(model, cuda):
    """model.prefetch(next) + forward(next) equals forward(next) alone (same buffers content, same kernels); the flat optimizer built by
    the reference-named mapper updates the very tensors the module exposes"""
    import bench
    from yolov7_d2_b200 import optim

    m, _ = model
    m.train()
    ba = bench.batched_inputs_from(*orc.synthetic_batch(2, 160, 31, max_gt=4))
    bb = bench.batched_inputs_from(*orc.synthetic_batch(2, 160, 32, max_gt=4))
    with torch.no_grad():
        ref_a = float(m(ba)["total_loss"])
        ref_b = float(m(bb)["total_loss"])
        la = m(ba)["total_loss"]
        m.prefetch(bb)                  # copies run behind forward(ba)
        lb = m(bb)["total_loss"]        # swaps buffers
        m.prefetch(ba)
        la2 = m(ba)["total_loss"]
    assert float(la) == ref_a and float(lb) == ref_b and float(la2) == ref_a
    # a stale prefetch (different list object) is ignored
    m.prefetch(bb)
    with torch.no_grad():
        assert float(m(bench.batched_inputs_from(*orc.synthetic_batch(2, 160, 31, max_gt=4)))["total_loss"]) == ref_a

    class S:
        OPTIMIZER, BASE_LR, MOMENTUM, NESTEROV, WEIGHT_DECAY, WEIGHT_DECAY_NORM = "SGD", 1e-3, 0.9, False, 5e-4, 0.0

    class C:
        SOLVER = S()

    opt = optim.build_optimizer_mapper(C(), m)
    w = dict(m.named_parameters())["head.cls_preds.0.bias"]
    before = w.detach().clone()
    losses = []
    for _ in range(3):
        opt.zero_grad()
        out = m(ba)
        out["total_loss"].backward()
        assert w.grad.data_ptr() == m.engine.grads["head.cls_preds.0.bias"].data_ptr()  # gradients land in the flat buffer
        opt.step()
        losses.append(float(out["total_loss"].detach()))
    assert not torch.equal(before, w.detach()) and losses[-1] < losses[0]


@pytest.mark.gpu
def test_standalone_backbone_neck_head_like_a_yolov5_caller(model, cuda):
    """The YOLOV5 / YOLOV7P / YOLOMask architectures build `build_cspdarknetx_backbone` through BACKBONE_REGISTRY and call
    `backbone(x)["dark3"]` themselves (darknetx.py:165-213, yolo_pafpn.py:79-114, yolox_head.py:197-224).  The registered modules run on
    their own; chained, they reproduce the fused YOLOX evaluation exactly (same kernels, same 16-bit storage)."""
    import bench
    from yolov7_d2_b200 import modeling

    m, sd = model
    m.load_state_dict(sd, strict=True)  # earlier tests trained this fixture: restore the running statistics of the state_dict
    m.eval()
    cfg = bench.yolox_s_cfg("cuda")
    bb = modeling.BACKBONE_REGISTRY.get("build_cspdarknetx_backbone")(cfg, None)   # standalone: owns its parameters
    neck = modeling.YOLOPAFPN(depth=0.33, width=0.5, in_features=["dark3", "dark4", "dark5"])
    head = modeling.YOLOXHead(80, width=0.5)
    bb.load_state_dict({k[len("backbone."):]: v for k, v in sd.items() if k.startswith("backbone.")}, strict=True)
    neck.load_state_dict({k[len("neck."):]: v for k, v in sd.items() if k.startswith("neck.")}, strict=True)
    head.load_state_dict({k[len("head."):]: v for k, v in sd.items() if k.startswith("head.")}, strict=True)
    for mod in (bb, neck, head):
        mod.eval()
    images, _ = orc.synthetic_batch(2, 160, 31)
    x = images.float().to(cuda)
    feats = bb(x)
    assert set(feats.keys()) == {"dark3", "dark4", "dark5"}
    assert tuple(feats["dark3"].shape) == (2, 128, 20, 20) and feats["dark3"].dtype == torch.float32
    with torch.no_grad():
        ref = orc.csp_darknet(images.float(), {k: v.clone() for k, v in sd.items()}, False)
    for k in feats:
        err = (feats[k].cpu() - ref[k]).abs().mean() / ref[k].abs().mean()
        assert err < 0.02, (k, float(err))
    pred = head(neck(feats))
    eng = m._plan(2, 160, 160)
    eng.images_u8.copy_(images.to(cuda))
    fused = eng.eval_forward()
    assert torch.equal(pred, fused), "standalone backbone -> neck -> head differs from the fused evaluation"


@pytest.mark.gpu
def test_standalone_backbone_trains_through_autograd(cuda):
    """a caller that owns the loss: gradients reach the backbone's parameters through the partial engine backward"""
    from yolov7_d2_b200 import modeling

    sd = orc.yolox_state_dict(6)
    bb = modeling.CSPDarknet(0.33, 0.5)
    bb.load_state_dict({k[len("backbone."):]: v for k, v in sd.items() if k.startswith("backbone.")}, strict=True)
    bb.train()
    images, _ = orc.synthetic_batch(4, 128, 32)
    x = images.float().to(cuda)
    g = torch.Generator().manual_seed(1)
    w3 = torch.randn(4, 128, 16, 16, generator=g).to(cuda) * 1e-2
    w5 = torch.randn(4, 512, 4, 4, generator=g).to(cuda) * 1e-2
    feats = bb(x)
    ((feats["dark3"] * w3).sum() + (feats["dark5"] * w5).sum()).backward()
    rsd = {k: v.clone().requires_grad_(v.dtype == torch.float32 and "running" not in k) for k, v in sd.items() if k.startswith("backbone.")}
    rf = orc.csp_darknet(images.float(), rsd, True)
    ((rf["dark3"] * w3.cpu()).sum() + (rf["dark5"] * w5.cpu()).sum()).backward()
    worst = 1.0
    for name, p in bb.named_parameters():
        assert p.grad is not None and torch.isfinite(p.grad).all(), name
        r = rsd["backbone." + name].grad.flatten().double()
        gq = p.grad.cpu().flatten().double()
        worst = min(worst, float((gq @ r) / (gq.norm() * r.norm() + 1e-30)))
    assert worst >= 0.9, worst


@pytest.mark.gpu
def test_api_cuda_graphs_reproduce_eager_training(cuda, monkeypatch):
    """YOLOX.forward / backward replay CUDA graphs after two eager calls (YB200_API_GRAPHS, default on): the same kernels on the same data as
    eager launches, so the same losses and parameters bit for bit over several optimizer steps, including a prefetched batch"""
    import bench
    from yolov7_d2_b200 import optim
    from yolov7_d2_b200.modeling import YOLOX

    images, labels = orc.synthetic_batch(2, 128, 61, max_gt=4)
    batches = [bench.batched_inputs_from(images, labels), bench.batched_inputs_from(images.flip(0).contiguous(), labels.flip(0).contiguous())]
    results = []
    for flag in ("1", "0"):
        monkeypatch.setenv("YB200_API_GRAPHS", flag)
        m = YOLOX(bench.yolox_s_cfg("cuda"))
        m.load_state_dict(orc.yolox_state_dict(8), strict=True)
        m.train()
        cfg = bench.yolox_s_cfg("cuda")
        cfg.SOLVER.BASE_LR = 1e-3
        opt = optim.build_optimizer_mapper(cfg, m)
        losses = []
        for it in range(6):
            opt.zero_grad()
            out = m(batches[it & 1])
            if it == 3:
                m.prefetch(batches[(it + 1) & 1])
            sum(out.values()).backward()
            opt.step()
            losses.append(float(out["total_loss"].detach()))
        plan = m._plan(2, 128, 128)
        graphed = bool(getattr(plan, "_api_graphs", {}).get("backward", {}).get("graph"))
        assert graphed == (flag == "1"), "graph capture state"
        results.append((losses, m.engine.flat_param.clone()))
    (la, pa), (lb, pb) = results
    assert la == lb, (la, lb)
    assert torch.equal(pa, pb), float((pa - pb).abs().max())


@pytest.mark.gpu
def test_l1_loss_switches_on_after_the_augmentation_phase(cuda):
    """yolox.py:105-121, 207-208 + yolox_head.py:186-195, 389-429: once `iter > INPUT.MOSAIC_AND_MIXUP.DISABLE_AT_ITER` the loss dict gains `l1_loss`
    (L1 on the raw regression outputs), the total includes it, and it trains (eager launch, graph capture and replay)"""
    import bench
    from yolov7_d2_b200 import optim
    from yolov7_d2_b200.modeling import YOLOX

    cfg = bench.yolox_s_cfg("cuda")
    m = YOLOX(cfg)
    m.load_state_dict(orc.yolox_state_dict(6), strict=True)
    m.train()
    images, labels = orc.synthetic_batch(2, 128, 71, max_gt=4)
    bi = bench.batched_inputs_from(images, labels)
    assert "l1_loss" not in m(bi) and not m.use_l1
    m.update_iter(m.enable_l1_loss_at + 1)
    out = m(bi)
    assert m.use_l1 and m.head.use_l1 and set(out.keys()) == {"total_loss", "iou_loss", "conf_loss", "cls_loss", "l1_loss"}
    eng = m._plan(2, 128, 128)
    xs, ys, ss = orc.anchor_grid([(h, w) for h, w, _, _ in eng.levels])
    ref = orc.yolox_losses(eng.outputs.cpu(), labels, xs, ys, ss, origin_preds=eng.raw_reg.cpu())
    got = [float(out[k]) for k in ("total_loss", "iou_loss", "conf_loss", "cls_loss", "l1_loss")]
    assert np.allclose(got, [float(v) for v in ref[:5]], rtol=1e-4, atol=1e-5), (got, ref[:5])
    assert got[4] > 0.1
    cfg.SOLVER.BASE_LR = 1e-3
    opt = optim.build_optimizer_mapper(cfg, m)
    wreg = dict(m.named_parameters())["head.reg_preds.0.weight"]
    before = wreg.detach().clone()
    losses = []
    for _ in range(4):  # eager, capture, replay, replay
        opt.zero_grad()
        o = m(bi)
        sum(o.values()).backward()
        opt.step()
        losses.append(float(o["l1_loss"].detach()))
    # (the SimOTA assignment changes from step to step on two images: no monotonic decrease to expect, only finite values that move the weights)
    assert all(np.isfinite(losses)) and len(set(losses)) > 1, losses
    assert not torch.equal(before, wreg.detach())
    graphs = getattr(eng, "_api_graphs", {})
    assert graphs.get("forward+l1", {}).get("graph") is not None and graphs.get("backward+l1", {}).get("graph") is not None
