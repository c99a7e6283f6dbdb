"""DETR matching cost, SetCriterion and the DETR tail on the sm_90a kernels, against the unmodified reference (tests/golden/detr_criterion.npz)
and the plain-torch restatement (oracle/detr_criterion_oracle.py, pinned to the reference by tests/test_detr_criterion_oracle_golden.py)."""
import os

import numpy as np
import pytest
import torch
import torch.nn as nn

from oracle import detr_criterion_oracle as dco
from oracle import detr_oracle as dto
from test_detr_criterion_oracle_golden import CASES, golden_indices, load_case

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "detr_criterion.npz")
TERMS = ("loss_ce", "loss_bbox", "loss_giou")


@pytest.fixture(scope="module")
def gold():
    return np.load(GOLD, allow_pickle=False)


def _dev_case(gold, name, cuda):
    layers, targets, dims, eos, costs, w = load_case(gold, name)
    layers = [(lg.to(cuda).requires_grad_(True), bx.to(cuda).requires_grad_(True)) for lg, bx in layers]
    targets_d = [{k: v.to(cuda) for k, v in t.items()} for t in targets]
    outputs = {"pred_logits": layers[-1][0], "pred_boxes": layers[-1][1]}
    if len(layers) > 1:
        outputs["aux_outputs"] = [{"pred_logits": lg, "pred_boxes": bx} for lg, bx in layers[:-1]]
    return layers, targets, targets_d, outputs, dims, eos, costs, w


def _criterion(k1, eos, costs):
    from yolov7_d2_b200.detr_criterion import HungarianMatcher, SetCriterion

    return SetCriterion(k1 - 1, HungarianMatcher(*costs), {}, eos, ["labels", "boxes", "cardinality"])


@pytest.mark.parametrize("name", CASES)
def test_cost_kernel_against_fp64(gold, cuda, name):
    from yolov7_d2_b200 import capi
    from yolov7_d2_b200.detr_criterion import _Targets

    layers, targets, targets_d, _, (L, B, Q, K1), eos, costs, _ = _dev_case(gold, name, cuda)
    logits = torch.stack([lg.detach() for lg, _ in layers]).contiguous()
    boxes = torch.stack([bx.detach() for _, bx in layers]).contiguous()
    tg = _Targets(targets_d, cuda)
    cost = torch.full((L * Q * tg.total + 1,), float("nan"), device=cuda)
    capi.detr_match_cost(logits, boxes, tg.labels, tg.boxes, tg.offsets, tg.total, *costs, cost)
    cost = cost.cpu()
    assert int(cost[-1:].view(torch.int32)) == 0
    ref = torch.cat([blk.flatten() for lg, bx in layers for blk in dco.match_cost(lg.detach().cpu().double(), bx.detach().cpu().double(),
                                                                                       [{k: v.double() if v.is_floating_point() else v for k, v in t.items()} for t in targets], *costs)]
                    or [torch.zeros(0, dtype=torch.float64)])
    assert torch.allclose(cost[:-1].double(), ref, rtol=1e-5, atol=1e-5), (cost[:-1].double() - ref).abs().max()


@pytest.mark.parametrize("name", CASES)
def test_assignment_matches_the_reference(gold, cuda, name):
    """scipy on the kernel's cost: the golden indices, or (near-ties) an assignment whose golden-cost total is the golden optimum within 1e-5"""
    from yolov7_d2_b200.detr_criterion import HungarianMatcher, _Targets

    layers, targets, targets_d, _, (L, B, Q, K1), eos, costs, _ = _dev_case(gold, name, cuda)
    logits = torch.stack([lg.detach() for lg, _ in layers])
    boxes = torch.stack([bx.detach() for _, bx in layers])
    idx, match = HungarianMatcher(*costs).match_layers(logits, boxes, _Targets(targets_d, cuda))
    ref_idx = golden_indices(gold, name)
    cost = torch.tensor(gold[name + "/cost"])
    sizes = [len(t["labels"]) for t in targets]
    off = np.concatenate([[0], np.cumsum(sizes)])
    G = int(off[-1])
    for l in range(L):
        for b in range(B):
            (gi, gj), (ri, rj) = idx[l][b], ref_idx[l][b]
            assert gi.dtype == torch.int64 and gj.dtype == torch.int64 and len(gi) == min(Q, sizes[b])
            if not (torch.equal(gi, ri) and torch.equal(gj, rj)):
                start = l * Q * G + Q * int(off[b])
                blk = cost[start:start + Q * sizes[b]].view(Q, sizes[b])
                assert abs(dco.assignment_cost(blk, (gi, gj)) - dco.assignment_cost(blk, (ri, rj))) <= 1e-5, (name, l, b)
            m = match[l, b]
            assert (m >= 0).sum() == len(gi) and torch.equal(m[gi].long(), gj)


@pytest.mark.parametrize("name", CASES)
def test_losses_and_gradients_match_the_reference(gold, cuda, name):
    """loss values within 1e-5 relative, counts exactly, and the gradient of Σ w[l, k] · loss[l, k] (non-unit weights, every layer) within
    1e-5 of its max-norm"""
    layers, targets, targets_d, outputs, (L, B, Q, K1), eos, costs, w = _dev_case(gold, name, cuda)
    losses = _criterion(K1, eos, costs)(outputs, targets_d)
    p = name + "/"
    assert list(losses.keys()) == [str(k) for k in gold[p + "keys"]]
    ref = gold[p + "losses"]
    for l in range(L):
        sfx = "" if l == L - 1 else f"_{l}"
        for k, key in enumerate(TERMS):
            v = float(losses[key + sfx])
            assert abs(v - ref[l, k]) <= 1e-5 * abs(ref[l, k]) + 1e-7, (key + sfx, v, ref[l, k])
        assert float(losses["cardinality_error" + sfx]) == ref[l, 3]
        assert not losses["cardinality_error" + sfx].requires_grad
    assert float(losses["class_error"]) == ref[L - 1, 4] and not losses["class_error"].requires_grad
    total = sum(float(w[l, k]) * losses[key + ("" if l == L - 1 else f"_{l}")] for l in range(L) for k, key in enumerate(TERMS))
    total.backward()
    dl, rows, db = torch.tensor(gold[p + "dlogits"]), torch.tensor(gold[p + "grad_rows"]), torch.tensor(gold[p + "dboxes"])
    got = torch.stack([lg.grad.cpu() for lg, _ in layers]).reshape(-1, K1)[rows]
    assert (got - dl).abs().max() <= 1e-5 * max(dl.abs().max().item(), 1e-30), name
    for l, (lg, bx) in enumerate(layers):
        assert (bx.grad.cpu() - db[l]).abs().max() <= 1e-5 * max(db.abs().max().item(), 1e-30), (name, l)


def test_criterion_is_bit_reproducible(gold, cuda):
    layers, _, targets_d, outputs, (L, B, Q, K1), eos, costs, w = _dev_case(gold, "l6", cuda)
    crit = _criterion(K1, eos, costs)
    runs = []
    for _ in range(2):
        for lg, bx in layers:
            lg.grad = bx.grad = None
        losses = crit(outputs, targets_d)
        sum(losses[k] for k in losses if k.startswith("loss_")).backward()
        runs.append((torch.stack([v.detach() for v in losses.values()]), [lg.grad.clone() for lg, _ in layers], [bx.grad.clone() for _, bx in layers]))
    (a, al, ab), (b, bl, bb) = runs
    assert torch.equal(a, b) and all(torch.equal(x, y) for x, y in zip(al + ab, bl + bb))


def test_without_aux_loss_and_matcher_entry(gold, cuda):
    from yolov7_d2_b200.detr_criterion import HungarianMatcher

    layers, _, targets_d, _, (L, B, Q, K1), eos, costs, _ = _dev_case(gold, "l6", cuda)
    out = {"pred_logits": layers[-1][0], "pred_boxes": layers[-1][1]}
    losses = _criterion(K1, eos, costs)(out, targets_d)
    assert list(losses.keys()) == ["loss_ce", "class_error", "loss_bbox", "loss_giou", "cardinality_error"]
    ref = gold["l6/losses"][-1]
    assert abs(float(losses["loss_ce"]) - ref[0]) <= 1e-5 * ref[0]
    idx = HungarianMatcher(*costs)(out, targets_d)
    for (gi, gj), (ri, rj) in zip(idx, golden_indices(gold, "l6")[-1]):
        assert torch.equal(gi, ri) and torch.equal(gj, rj)


def test_bad_targets_raise_instead_of_faulting(gold, cuda):
    from yolov7_d2_b200 import capi

    layers, _, targets_d, outputs, (L, B, Q, K1), eos, costs, _ = _dev_case(gold, "g_over_q", cuda)
    crit = _criterion(K1, eos, costs)
    bad = [dict(t) for t in targets_d]
    bad[0]["labels"] = bad[0]["labels"].clone()
    bad[0]["labels"][3] = K1
    with pytest.raises(capi.Yb200Error, match="label"):
        crit(outputs, bad)
    bad = [dict(t) for t in targets_d]
    bad[2]["boxes"] = bad[2]["boxes"].clone()
    bad[2]["boxes"][0, 2] = -0.1
    with pytest.raises(capi.Yb200Error, match="negative width"):
        crit(outputs, bad)
    with pytest.raises(capi.Yb200Error):
        _criterion(K1, eos, costs).__class__(K1 - 1, crit.matcher, {}, eos, ["labels", "masks"])(outputs, targets_d)
    torch.cuda.synchronize()
    assert float(crit(outputs, targets_d)["loss_ce"]) > 0  # the context is healthy


def test_one_device_to_host_copy_per_criterion_call(gold, cuda):
    from torch.profiler import ProfilerActivity, profile

    layers, _, targets_d, outputs, (L, B, Q, K1), eos, costs, _ = _dev_case(gold, "l6", cuda)
    crit = _criterion(K1, eos, costs)
    crit(outputs, targets_d)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        crit(outputs, targets_d)
        torch.cuda.synchronize()
    d2h = [e for e in prof.events() if "Memcpy DtoH" in e.name]
    assert L == 6 and len(d2h) == 1, [e.name for e in d2h]


class _StandInTransformer(nn.Module):
    def __init__(self, hs):
        super().__init__()
        self.d_model, self.hs = hs.shape[-1], hs

    def forward(self, src, mask, query, pos):
        self.seen = src
        return self.hs, None


class _Nested:
    def __init__(self, t, m):
        self.t, self.m = t, m

    def decompose(self):
        return self.t, self.m


class _StandInBackbone(nn.Module):
    def __init__(self, src, mask, pos):
        super().__init__()
        self.num_channels, self.src, self.mask, self.pos = src.shape[1], src, mask, pos

    def forward(self, samples):
        return [_Nested(self.src, self.mask)], [self.pos]


def _verdict(got, ref, emu, what):
    """None, or why `got` fails the 16-bit yardstick: cosine > 0.995 and max error <= 2.5 x the storage-emulating oracle's + 2e-2 (relative to
    max |ref|).  A reference that is exactly zero (e.g. the first decoder layer's self-attention weights: its input is zero, so every value and
    score is constant over the keys) must be matched by a gradient that is zero to 1e-6 of the gradient's own scale."""
    got, ref, emu = got.detach().float().cpu(), ref.detach().float().cpu(), emu.detach().float().cpu()
    if not torch.isfinite(got).all():
        return f"{what}: not finite"
    if ref.abs().max().item() == 0:
        return None if got.abs().max().item() <= 1e-6 * max(emu.abs().max().item(), 1.0) else f"{what}: nonzero where the reference is zero"
    scale = ref.abs().max().item()
    err, yard = (got - ref).abs().max().item() / scale, (emu - ref).abs().max().item() / scale
    cos = torch.dot(got.flatten(), ref.flatten()) / (got.norm() * ref.norm())
    ok = cos > 0.995 and err <= 2.5 * yard + 2e-2
    return None if ok else f"{what}: cos {cos:.4f}, rel err {err:.4f} vs emulated-storage yardstick {yard:.4f}"


def _judge(got, ref, emu, what):
    v = _verdict(got, ref, emu, what)
    assert v is None, v


def test_detr_tail_matches_the_reference(gold, cuda):
    from yolov7_d2_b200.detr import DETR
    from yolov7_d2_b200 import capi

    t = lambda k: torch.tensor(gold["heads/" + k]).to(cuda)
    sd = {k[len("heads/sd/"):]: torch.tensor(gold[k]) for k in gold.files if k.startswith("heads/sd/")}
    tr = _StandInTransformer(t("hs"))
    k1, nq = gold["heads/pred_logits"].shape[-1], gold["heads/pred_logits"].shape[-2]
    model = DETR(_StandInBackbone(t("src"), t("mask"), t("pos")), tr, num_classes=k1 - 1, num_queries=nq, aux_loss=True).to(cuda)
    model.load_state_dict({k: v.to(cuda) for k, v in sd.items()}, strict=True)
    out = model(_Nested(None, None))
    emu_l, emu_b = dco.heads(torch.tensor(gold["heads/hs"]), sd, storage=dco.bf16)
    emu_p = dco.input_proj(torch.tensor(gold["heads/src"]), sd, storage=dco.bf16)
    _judge(tr.seen, torch.tensor(gold["heads/proj"]), emu_p, "input_proj")
    ref_l = torch.tensor(np.concatenate([gold["heads/aux_logits"], gold["heads/pred_logits"][None]]))
    ref_b = torch.tensor(np.concatenate([gold["heads/aux_boxes"], gold["heads/pred_boxes"][None]]))
    got_l = torch.stack([a["pred_logits"] for a in out["aux_outputs"]] + [out["pred_logits"]])
    got_b = torch.stack([a["pred_boxes"] for a in out["aux_outputs"]] + [out["pred_boxes"]])
    assert got_l.dtype == torch.float32 and got_b.dtype == torch.float32
    _judge(got_l, ref_l, emu_l, "pred_logits")
    _judge(got_b, ref_b, emu_b, "pred_boxes")
    with pytest.raises(capi.Yb200Error):
        model(torch.zeros(2, 3, 8, 8, device=cuda))


def test_detr_training_step_against_the_oracle_stack(cuda):
    """DETR (stand-in backbone feature [2, 2048, 20, 25] with a ragged padding mask and sine positions) -> Transformer (256, 8 heads, 6 + 6
    layers, dropout 0, intermediate outputs) -> SetCriterion: the loss dict and every parameter gradient, input_proj and the gradient into the
    backbone feature included, against the oracle stack given the device's assignment, judged with the 16-bit yardstick"""
    from yolov7_d2_b200.detr import DETR, Transformer
    from yolov7_d2_b200.detr_criterion import HungarianMatcher, SetCriterion, _Targets

    torch.manual_seed(0)
    g = torch.Generator().manual_seed(7)
    B, C, H, W, d, nq, k1 = 2, 2048, 20, 25, 256, 100, 81
    feat = (torch.randn(B, C, H, W, generator=g) * 0.5).to(cuda).requires_grad_(True)
    mask = torch.zeros(B, H, W, dtype=torch.bool)
    mask[1, 15:, :] = True
    mask[1, :, 19:] = True
    # sine positions (PositionEmbeddingSine, normalize=True) of the unpadded region
    not_mask = (~mask).float()
    y = not_mask.cumsum(1)
    x = not_mask.cumsum(2)
    y, x = y / (y[:, -1:, :] + 1e-6) * 2 * np.pi, x / (x[:, :, -1:] + 1e-6) * 2 * np.pi
    dim_t = 10000 ** (2 * (torch.arange(d // 2) // 2) / (d // 2))
    px, py = x[..., None] / dim_t, y[..., None] / dim_t
    px = torch.stack((px[..., 0::2].sin(), px[..., 1::2].cos()), 4).flatten(3)
    py = torch.stack((py[..., 0::2].sin(), py[..., 1::2].cos()), 4).flatten(3)
    pos = torch.cat((py, px), 3).permute(0, 3, 1, 2).contiguous()
    tr = Transformer(d, 8, 6, 6, dim_feedforward=2048, dropout=0.0, return_intermediate_dec=True)
    model = DETR(_StandInBackbone(feat, mask.to(cuda), pos.to(cuda)), tr, num_classes=k1 - 1, num_queries=nq, aux_loss=True).to(cuda)
    targets = []
    for n in (7, 19):
        targets.append({"labels": torch.randint(0, k1 - 1, (n,), generator=g).to(cuda),
                        "boxes": torch.cat([torch.rand(n, 2, generator=g) * 0.8 + 0.1, torch.rand(n, 2, generator=g) * 0.4 + 0.05], 1).to(cuda)})
    matcher = HungarianMatcher(1, 5, 2)
    crit = SetCriterion(k1 - 1, matcher, {}, 0.1, ["labels", "boxes", "cardinality"])
    out = model(_Nested(None, None))
    losses = crit(out, targets)
    layers = [(a["pred_logits"], a["pred_boxes"]) for a in out["aux_outputs"]] + [(out["pred_logits"], out["pred_boxes"])]
    idx, _ = matcher.match_layers(torch.stack([lg.detach() for lg, _ in layers]), torch.stack([bx.detach() for _, bx in layers]),
                                  _Targets(targets, cuda))
    wts = {"loss_ce": 1.0, "loss_bbox": 5.0, "loss_giou": 2.0}
    weight = lambda k: next(v for n, v in wts.items() if k == n or k.startswith(n + "_"))
    sum(weight(k) * v for k, v in losses.items() if k.startswith(tuple(wts))).backward()

    sd0 = {k: v.detach().cpu().float() for k, v in model.state_dict().items()}
    tg_cpu = [{k: v.cpu() for k, v in t.items()} for t in targets]

    def oracle(emulate):
        dto.EMULATE_STORAGE = emulate
        q = dco.bf16 if emulate else None
        try:
            sd = {k: v.clone().requires_grad_(v.is_floating_point()) for k, v in sd0.items()}
            f = feat.detach().cpu().requires_grad_(True)
            src = dco.input_proj(f, sd, storage=q)
            s = src.flatten(2).permute(2, 0, 1)
            p = pos.flatten(2).permute(2, 0, 1)
            qe = sd["query_embed.weight"].unsqueeze(1).repeat(1, B, 1)
            m = mask.flatten(1)
            mem = s
            for i in range(6):
                mem = dto.encoder_layer_post(mem, sd, f"transformer.encoder.layers.{i}.", 8, m, p)
            o, inter = torch.zeros_like(qe), []
            for i in range(6):
                o = dto.decoder_layer_post(o, mem, sd, f"transformer.decoder.layers.{i}.", 8, m, p, qe)
                inter.append(torch.nn.functional.layer_norm(o, (d,), sd["transformer.decoder.norm.weight"], sd["transformer.decoder.norm.bias"]))
            hs = torch.stack(inter).transpose(1, 2)
            lg, bx = dco.heads(hs, sd, storage=q)
            ls, _ = dco.criterion([(lg[l], bx[l]) for l in range(6)], tg_cpu, k1 - 1, 0.1, (1, 5, 2), indices=idx)
            sum(weight(k) * v for k, v in ls.items() if k.startswith(tuple(wts))).backward()
        finally:
            dto.EMULATE_STORAGE = False
        return ls, sd, f

    ref_l, ref_sd, ref_f = oracle(False)
    emu_l, emu_sd, emu_f = oracle(True)
    assert list(losses.keys()) == list(ref_l.keys())
    for k in losses:
        if k.startswith("loss_"):
            r, e = float(ref_l[k]), float(emu_l[k])
            assert abs(float(losses[k]) - r) <= 2.5 * abs(e - r) + 2e-2 * abs(r), (k, float(losses[k]), r, e)
    bad = [_verdict(feat.grad, ref_f.grad, emu_f.grad, "backbone feature gradient")]
    for n, prm in model.named_parameters():
        assert prm.grad is not None, n
        bad.append(_verdict(prm.grad, ref_sd[n].grad, emu_sd[n].grad, n))
    bad = [b for b in bad if b]
    assert not bad, bad
