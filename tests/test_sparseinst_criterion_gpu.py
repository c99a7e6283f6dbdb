"""SparseInst's matcher and criterion on the sm_90a kernels (yolov7_d2_b200.sparseinst_criterion, csrc/sparseinst_criterion.cu) against the
unmodified reference (tests/golden/sparseinst_criterion.npz) and the fp64 restatement (oracle/sparseinst_criterion_oracle.py, pinned to the
reference by tests/test_sparseinst_criterion_oracle_golden.py)."""
import math
import types
import warnings

import numpy as np
import pytest
import torch

from oracle import sparseinst_criterion_oracle as sco
from test_sparseinst_criterion_oracle_golden import CASES, GOLD, golden_indices, load_case

pytestmark = pytest.mark.gpu
ns = types.SimpleNamespace


@pytest.fixture(scope="module")
def gold():
    return np.load(GOLD, allow_pickle=False)


def _cfg(K, alpha=0.8, beta=0.2, weights=(2.0, 5.0, 2.0, 1.0), items=("labels", "masks"), matcher="SparseInstMatcher"):
    return ns(MODEL=ns(SPARSE_INST=ns(LOSS=ns(NAME="SparseInstCriterion", ITEMS=items, CLASS_WEIGHT=weights[0], MASK_PIXEL_WEIGHT=weights[1],
                                              MASK_DICE_WEIGHT=weights[2], OBJECTNESS_WEIGHT=weights[3]),
                                      MATCHER=ns(NAME=matcher, ALPHA=alpha, BETA=beta), DECODER=ns(NUM_CLASSES=K))))


def _criterion(c):
    from yolov7_d2_b200.sparseinst_criterion import build_sparse_inst_criterion

    return build_sparse_inst_criterion(_cfg(c["K"], c["alpha"], c["beta"], c["weights"], c["items"]))


def _dev(c, cuda):
    """(outputs with fp32 leaves that require grad, device targets)"""
    outputs = {k: c[s].float().to(cuda).requires_grad_(True) for k, s in (("pred_logits", "logits"), ("pred_masks", "masks"), ("pred_scores", "scores"))}
    off = np.concatenate([[0], np.cumsum(c["sizes"])])
    targets = [{"labels": c["labels"][off[b]:off[b + 1]].to(cuda), "masks": sco.BitMasks(m.to(cuda))} for b, m in enumerate(c["mask_list"])]
    return outputs, targets


def _run(crit, outputs, targets, input_shape, coef):
    for v in outputs.values():
        v.grad = None
    losses = crit(outputs, targets, input_shape)
    sum(coef[k] * v for k, v in losses.items()).backward()
    return losses, [outputs[k].grad for k in ("pred_logits", "pred_masks", "pred_scores")]


def _within(got, ref, tol, what):
    got, ref = got.detach().double().cpu(), torch.as_tensor(ref).double()
    err = (got - ref).abs().max().item() if ref.numel() else 0.0
    assert err <= tol * max(ref.abs().max().item() if ref.numel() else 0.0, 1e-30), f"{what}: max err {err:.3e}, max |ref| {ref.abs().max().item():.3e}"


# ---- 1. target masks ---------------------------------------------------------------------------------------------------------------------------
def _target_masks(mask_list, input_shape, size, cuda):
    from yolov7_d2_b200.sparseinst_criterion import _Targets

    targets = [{"labels": torch.zeros(m.shape[0], dtype=torch.int64, device=cuda), "masks": sco.BitMasks(m.to(cuda))} for m in mask_list]
    return _Targets(targets, input_shape, (len(mask_list), max(64, max(m.shape[0] for m in mask_list)), *size), cuda, "test")


@pytest.mark.parametrize("shape", [((640, 640), (160, 160), [(640, 640), (480, 600), (333, 517)]), ((160, 160), (40, 40), [(150, 140), (37, 160)])])
def test_target_masks_bit_exact_at_a_quarter_of_the_input(cuda, shape):
    input_shape, size, hw = shape
    g = torch.Generator().manual_seed(1)
    mask_list = [torch.rand(5, h, w, generator=g) > 0.6 for h, w in hw]
    tg = _target_masks(mask_list, input_shape, size, cuda)
    ref = sco.target_masks(mask_list, input_shape, size, torch.float32)
    assert torch.equal(tg.masks.cpu(), ref)
    _within(tg.tsq, (ref.double() ** 2).flatten(1).sum(1), 1e-6, "sum t^2")


@pytest.mark.parametrize("shape", [((100, 90), (24, 22), [(100, 90), (87, 71)]), ((97, 131), (40, 56), [(97, 131)]), ((64, 64), (80, 48), [(60, 64)])])
def test_target_masks_other_sizes(cuda, shape):
    input_shape, size, hw = shape
    g = torch.Generator().manual_seed(2)
    mask_list = [(torch.rand(3, h, w, generator=g) * 3).to(torch.uint8) for h, w in hw]  # uint8 values are taken as they are, as the reference does
    tg = _target_masks(mask_list, input_shape, size, cuda)
    ref = sco.target_masks(mask_list, input_shape, size, torch.float32)
    assert (tg.masks.cpu() - ref).abs().max() <= 1e-6


# ---- 2.-5. against the reference fixture -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", CASES)
def test_cost_blocks_against_fp64(gold, cuda, name):
    from yolov7_d2_b200 import capi
    from yolov7_d2_b200.sparseinst_criterion import _Targets

    c = load_case(gold, name)
    outputs, targets = _dev(c, cuda)
    masks = outputs["pred_masks"].detach()
    tg = _Targets(targets, c["input_shape"], masks.shape, cuda, "test")
    cost = torch.full((c["N"] * tg.total + 1,), float("nan"), device=cuda)
    capi.sparseinst_match_cost(outputs["pred_logits"].detach(), masks, tg.labels, tg.offsets, tg.masks, tg.tsq, tg.total, c["alpha"], c["beta"], cost)
    cost = cost.cpu()
    assert int(cost[-1:].view(torch.int32)) == 0
    tm = sco.target_masks(c["mask_list"], c["input_shape"], c["size"], torch.float64)
    ref = torch.cat([b.flatten() for b in sco.match_cost(c["logits"], c["masks"], tm, c["sizes"], c["labels"], c["alpha"], c["beta"])])
    assert (cost[:-1].double() - ref).abs().max() <= 1e-5
    assert torch.allclose(ref, torch.tensor(gold[name + "/cost"]), rtol=1e-12, atol=1e-14)


def _check_assignment(indices, ref_idx, blocks, N, sizes, what):
    for b, ((gi, gj), (ri, rj)) in enumerate(zip(indices, ref_idx)):
        assert gi.dtype == torch.int64 and gj.dtype == torch.int64 and len(gi) == min(N, sizes[b]), (what, b)
        if not (torch.equal(gi, ri) and torch.equal(gj, rj)):
            assert abs(sco.assignment_cost(blocks[b], (gi, gj)) - sco.assignment_cost(blocks[b], (ri, rj))) <= 1e-5, (what, b)


@pytest.mark.parametrize("name", CASES)
def test_assignment_matches_the_reference(gold, cuda, name):
    from yolov7_d2_b200.sparseinst_criterion import SparseInstMatcher

    c = load_case(gold, name)
    outputs, targets = _dev(c, cuda)
    indices = SparseInstMatcher(_cfg(c["K"], c["alpha"], c["beta"]))(outputs, targets, c["input_shape"])
    tm = sco.target_masks(c["mask_list"], c["input_shape"], c["size"], torch.float64)
    blocks = sco.match_cost(c["logits"], c["masks"], tm, c["sizes"], c["labels"], c["alpha"], c["beta"])
    _check_assignment(indices, golden_indices(gold, name), blocks, c["N"], c["sizes"], name)


@pytest.mark.parametrize("name", CASES)
def test_losses_and_gradients_match_the_reference(gold, cuda, name):
    """losses within 1e-5 relative with the reference's keys and order; the gradient of Σ coef[k] · loss[k] within 1e-5 of its max-norm; exact
    zeros on unmatched rows of d pred_masks"""
    c = load_case(gold, name)
    p = name + "/"
    outputs, targets = _dev(c, cuda)
    losses, (dl, dm, ds) = _run(_criterion(c), outputs, targets, c["input_shape"], c["coef"])
    assert list(losses.keys()) == [str(k) for k in gold[p + "keys"]]
    for k, ref in zip(losses, gold[p + "losses"]):
        assert abs(float(losses[k].detach()) - ref) <= 1e-5 * abs(ref) + 1e-7, (k, float(losses[k].detach()), ref)
    B, N, K = c["B"], c["N"], c["K"]
    rows, mrows = torch.tensor(gold[p + "grad_rows"]), torch.tensor(gold[p + "mask_rows"])
    _within(dl.cpu().reshape(B * N, K)[rows], gold[p + "dlogits"], 1e-5, "d pred_logits")
    _within(dm.cpu().reshape(B * N, -1)[mrows], gold[p + "dmasks"], 1e-5, "d pred_masks")
    _within(ds, gold[p + "dscores"], 1e-5, "d pred_scores")
    unmatched = torch.ones(B * N, dtype=torch.bool)
    unmatched[mrows] = False
    assert torch.equal(dm.cpu().reshape(B * N, -1)[unmatched], torch.zeros(int(unmatched.sum()), dm[0, 0].numel()))


def test_criterion_is_bit_reproducible(gold, cuda):
    c = load_case(gold, "a_pad")
    outputs, targets = _dev(c, cuda)
    crit = _criterion(c)
    runs = []
    for _ in range(2):
        losses, grads = _run(crit, outputs, targets, c["input_shape"], c["coef"])
        runs.append((torch.stack([v.detach() for v in losses.values()]), [g.clone() for g in grads]))
    (a, ga), (b, gb) = runs
    assert torch.equal(a, b) and all(torch.equal(x, y) for x, y in zip(ga, gb))


def test_batch_without_instances(cuda):
    """defined behaviour (the reference raises): loss_ce over all-background labels with num_instances = 1, zero mask losses and gradients"""
    g = torch.Generator().manual_seed(3)
    B, N, K, H, W = 2, 10, 6, 8, 8
    logits, masks, scores = torch.randn(B, N, K, generator=g), torch.randn(B, N, H, W, generator=g), torch.randn(B, N, 1, generator=g)
    c = dict(K=K, alpha=0.8, beta=0.2, weights=(2.0, 5.0, 2.0, 1.0), items=("labels", "masks"))
    outputs = {"pred_logits": logits.to(cuda).requires_grad_(True), "pred_masks": masks.to(cuda).requires_grad_(True),
               "pred_scores": scores.to(cuda).requires_grad_(True)}
    targets = [{"labels": torch.zeros(0, dtype=torch.int64, device=cuda), "masks": sco.BitMasks(torch.zeros(0, 32, 32, dtype=torch.bool, device=cuda))}
               for _ in range(B)]
    from yolov7_d2_b200.sparseinst_criterion import SparseInstMatcher

    assert all(len(i) == 0 and i.dtype == torch.int64 for i, _ in SparseInstMatcher(_cfg(K))(outputs, targets, (32, 32)))
    losses, (dl, dm, ds) = _run(_criterion(c), outputs, targets, (32, 32), {"loss_ce": 1.0, "loss_dice": 1.0, "loss_mask": 1.0, "loss_objectness": 1.0})
    assert list(losses.keys()) == ["loss_ce", "loss_dice", "loss_mask", "loss_objectness"]
    lg = logits.double().requires_grad_(True)
    ref = sco.sigmoid_focal_loss(lg, torch.zeros_like(lg)).sum() * 2.0
    ref.backward()
    assert abs(float(losses["loss_ce"]) - float(ref)) <= 1e-5 * float(ref)
    _within(dl, lg.grad, 1e-5, "d pred_logits")
    assert all(float(losses[k]) == 0.0 for k in ("loss_dice", "loss_mask", "loss_objectness"))
    assert not dm.any() and not ds.any()


# ---- 7. shipped size ---------------------------------------------------------------------------------------------------------------------------
def _ellipses(g, n, h, w):
    yy, xx = torch.meshgrid(torch.arange(h, dtype=torch.float32), torch.arange(w, dtype=torch.float32), indexing="ij")
    c = torch.rand(n, 4, generator=g)
    cy, cx, ry, rx = c[:, 0, None, None] * h, c[:, 1, None, None] * w, 8 + c[:, 2, None, None] * h / 4, 8 + c[:, 3, None, None] * w / 4
    return ((yy - cy) / ry) ** 2 + ((xx - cx) / rx) ** 2 <= 1


def test_shipped_size_against_fp64(cuda):
    """B = 16, N = 100, K = 80, 160 x 160 masks from a 640 x 640 input, 1-20 random ellipses per image: cost, assignment, losses and gradients
    against the fp64 oracle given the same assignment"""
    from yolov7_d2_b200.sparseinst_criterion import _Targets

    g = torch.Generator().manual_seed(4)
    B, N, K, S, IN = 16, 100, 80, 160, 640
    sizes = torch.randint(1, 21, (B,), generator=g).tolist()
    hw = [(int(torch.randint(400, IN + 1, (1,), generator=g)), int(torch.randint(400, IN + 1, (1,), generator=g))) for _ in range(B)]
    mask_list = [_ellipses(g, n, h, w) for n, (h, w) in zip(sizes, hw)]
    tm = sco.target_masks(mask_list, (IN, IN), (S, S), torch.float32)  # exact at 4x: values are multiples of 1/4
    codes = torch.round(torch.randn(B, N, S, S, generator=g) * 2.5 * 16)
    off = 0
    for b, n in enumerate(sizes):
        q = torch.randperm(N, generator=g)[:n]
        codes[b, q] += torch.round(8.0 * 16 * (tm[off:off + n] - 0.5))
        off += n
    codes = codes.clamp(-127, 127)
    codes[codes == -6.0] = -5.0  # no logit within 2^-8 of logit(0.4) = -0.405 (codes are multiples of 2^-4)
    masks = codes / 16
    logits = (torch.randn(B, N, K, generator=g) * 2 - 2)
    scores = torch.randn(B, N, 1, generator=g)
    labels = torch.randint(0, K, (sum(sizes),), generator=g)
    c = dict(K=K, alpha=0.8, beta=0.2, weights=(2.0, 5.0, 2.0, 1.0), items=("labels", "masks"), N=N, sizes=sizes, mask_list=mask_list, labels=labels)
    coef = {"loss_ce": 0.7, "loss_objectness": 1.3, "loss_dice": 0.4, "loss_mask": 1.9}
    outputs, targets = _dev(dict(c, logits=logits, masks=masks, scores=scores), cuda)
    crit = _criterion(c)
    tg = _Targets(targets, (IN, IN), masks.shape, cuda, "test")
    assert torch.equal(tg.masks.cpu(), tm)
    indices, _ = crit.matcher.match(outputs["pred_logits"].detach(), outputs["pred_masks"].detach(), tg)
    losses, (dl, dm, ds) = _run(crit, outputs, targets, (IN, IN), coef)

    tm64 = tm.double()
    blocks = sco.match_cost(logits.double(), masks.double(), tm64, sizes, labels, 0.8, 0.2)
    ref_idx = sco.assign(blocks)
    _check_assignment(indices, ref_idx, blocks, N, sizes, "shipped")
    lg, mk, sc = (t.double().requires_grad_(True) for t in (logits, masks, scores))
    ref = sco.losses(lg, mk, sc, tm64, sizes, labels, indices, dict(zip(("loss_ce", "loss_mask", "loss_dice", "loss_objectness"), c["weights"])),
                     float(sum(sizes)))
    assert list(losses.keys()) == list(ref.keys())
    for k in ref:
        r = float(ref[k].detach())
        assert abs(float(losses[k]) - r) <= 1e-5 * abs(r), (k, float(losses[k]), r)
    rdl, rdm, rds = sco.loss_gradients(lg, mk, sc, ref, coef)
    _within(dl, rdl, 1e-5, "d pred_logits")
    _within(dm, rdm, 1e-5, "d pred_masks")
    _within(ds, rds, 1e-5, "d pred_scores")
    matched = torch.zeros(B, N, dtype=torch.bool)
    for b, (i, _) in enumerate(indices):
        matched[b, i] = True
    assert not dm[matched.to(cuda)].eq(0).all() and not dm[~matched.to(cuda)].any()


# ---- 8. errors ---------------------------------------------------------------------------------------------------------------------------------
def test_errors_raise_before_any_loss_kernel(gold, cuda):
    from yolov7_d2_b200 import capi
    from yolov7_d2_b200.sparseinst_criterion import SparseInstCriterion, build_sparse_inst_criterion, build_sparse_inst_matcher

    c = load_case(gold, "b_empty_image")
    outputs, targets = _dev(c, cuda)
    crit = _criterion(c)
    shape = c["input_shape"]
    with pytest.raises(capi.Yb200Error, match="CUDA"):
        crit({k: v.detach().cpu() for k, v in outputs.items()}, targets, shape)
    with pytest.raises(capi.Yb200Error, match="CUDA"):
        crit(outputs, [{"labels": t["labels"].cpu(), "masks": t["masks"]} for t in targets], shape)
    bad = [dict(t) for t in targets]
    bad[1]["labels"] = bad[1]["labels"].clone()
    bad[1]["labels"][2] = c["K"]
    with pytest.raises(capi.Yb200Error, match="label"):
        crit(outputs, bad, shape)
    with pytest.raises(capi.Yb200Error, match="larger than input_shape"):
        crit(outputs, targets, (shape[0] - 1, shape[1]))
    too_many = [dict(t) for t in targets]
    too_many[1] = {"labels": torch.zeros(c["N"] + 1, dtype=torch.int64, device=cuda),
                   "masks": sco.BitMasks(torch.zeros(c["N"] + 1, 8, 8, dtype=torch.bool, device=cuda))}
    with pytest.raises(capi.Yb200Error, match="targets for"):
        crit(outputs, too_many, shape)
    with pytest.raises(capi.Yb200Error, match="unknown loss"):
        build_sparse_inst_criterion(_cfg(c["K"], items=("labels", "boxes")))(outputs, targets, shape)
    with pytest.raises(capi.Yb200Error, match="SparseInstMatcherV1"):
        build_sparse_inst_matcher(_cfg(c["K"], matcher="SparseInstMatcherV1"))
    with pytest.raises(capi.Yb200Error, match="matcher"):
        SparseInstCriterion(_cfg(c["K"]), object())(outputs, targets, shape)
    torch.cuda.synchronize()
    assert float(crit(outputs, targets, shape)["loss_ce"]) > 0  # the context is healthy


# ---- 9. synchronisation ------------------------------------------------------------------------------------------------------------------------
def test_one_synchronisation_per_criterion_call(gold, cuda):
    c = load_case(gold, "a_pad")
    outputs, targets = _dev(c, cuda)
    crit = _criterion(c)
    _run(crit, outputs, targets, c["input_shape"], c["coef"])
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("warn")
    try:
        with warnings.catch_warnings(record=True) as rec:
            warnings.simplefilter("always")
            _run(crit, outputs, targets, c["input_shape"], c["coef"])
    finally:
        torch.cuda.set_sync_debug_mode("default")
    syncs = [str(w.message) for w in rec if "synchroniz" in str(w.message).lower()]
    assert len(syncs) <= 1, syncs


# ---- 10. decoder output ------------------------------------------------------------------------------------------------------------------------
def test_criterion_on_decoder_output(cuda):
    from yolov7_d2_b200.sparseinst import BaseIAMDecoder

    dec_cfg = ns(MODEL=ns(SPARSE_INST=ns(ENCODER=ns(NUM_CHANNELS=64), DECODER=ns(SCALE_FACTOR=2.0, OUTPUT_IAM=False, NUM_MASKS=20, KERNEL_DIM=32,
                                                                                NUM_CLASSES=10, INST=ns(DIM=64, CONVS=1), MASK=ns(DIM=64, CONVS=1)))))
    torch.manual_seed(0)
    out = BaseIAMDecoder(dec_cfg)(torch.randn(2, 64, 16, 16, device=cuda))
    g = torch.Generator().manual_seed(5)
    targets = [{"labels": torch.randint(0, 10, (n,), generator=g).to(cuda), "masks": sco.BitMasks(_ellipses(g, n, 120, 128).to(cuda))} for n in (3, 5)]
    losses = _criterion(dict(K=10, alpha=0.8, beta=0.2, weights=(2.0, 5.0, 2.0, 1.0), items=("labels", "masks")))(out, targets, (128, 128))
    assert list(losses.keys()) == ["loss_ce", "loss_objectness", "loss_dice", "loss_mask"]
    assert all(math.isfinite(float(v)) for v in losses.values())
