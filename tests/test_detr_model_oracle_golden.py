"""CPU: oracle/detr_model_oracle.py against tests/golden/detr_model.npz, written by oracle/gen_golden_detr_model.py from the unmodified reference
Detr.preprocess_image / prepare_targets / inference, MaskedBackboneTraceFriendly, Joiner and PositionEmbeddingSine.  The normalised batches,
masks, positions, kept sets, labels, scores, boxes and packed targets are bit-identical; the weighted training loss dict has the reference's
keys and order, and its values agree within 1e-5 relative when recomputed from the stored network outputs."""
import os

import numpy as np
import pytest
import torch
from oracle import detr_criterion_oracle as dco
from oracle import detr_model_oracle as dmo
from oracle.gen_golden_detr_model import (IMAGES, INFER, LEVELS, MEAN, NUM_POS_FEATS, STD, TARGETS, THRESH, TRAIN, image_case, infer_case,
                                          targets_case, train_case)

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "detr_model.npz")


def gold():
    return np.load(GOLD, allow_pickle=False)


@pytest.mark.parametrize("name", list(IMAGES))
def test_preprocess_masks_and_positions(name):
    g = gold()
    batch, sizes = dmo.preprocess(image_case(name), MEAN, STD)
    assert np.array_equal(batch.numpy(), g[f"{name}/images"]), "normalised batch differs"
    hp, wp = batch.shape[-2:]
    shapes = [(len(sizes), 16, -(-hp // s) if how == "ceil" else hp // s, -(-wp // s) if how == "ceil" else wp // s) for s, how in LEVELS]
    masks = dmo.mask_out_padding(shapes, [s for s, _ in LEVELS], sizes)
    for l, m in enumerate(masks):
        assert np.array_equal(m.numpy(), g[f"{name}/mask{l}"]), f"mask of level {l}"
        if name == "u8_ragged":
            assert np.array_equal(dmo.position_sine(m, NUM_POS_FEATS).numpy(), g[f"{name}/pos{l}"]), f"positions of level {l}"


def test_inference():
    g = gold()
    logits, boxes = infer_case()
    res = dmo.inference(logits, boxes, INFER["sizes"], INFER["out"], THRESH)
    for b, r in enumerate(res):
        assert np.array_equal(r["labels"].numpy(), g[f"infer/{b}/labels"]), b
        assert np.array_equal(r["scores"].numpy(), g[f"infer/{b}/scores"]), b
        assert np.array_equal(r["boxes"].numpy(), g[f"infer/{b}/boxes"]), b


def test_prepare_targets():
    g = gold()
    tb, tc = targets_case()
    for b, t in enumerate(dmo.prepare_targets(tb, tc, TARGETS["sizes"])):
        assert np.array_equal(t["labels"].numpy(), g[f"targets/{b}/labels"]) and np.array_equal(t["boxes"].numpy(), g[f"targets/{b}/boxes"]), b


def test_training_loss_dict():
    g = gold()
    K = TRAIN["K"]
    wd = dmo.weight_dict(5.0, 2.0, 2, True)
    assert list(wd) == list(g["train/weight_keys"]) and list(wd.values()) == list(g["train/weight_values"])
    _, boxes, classes = train_case()
    targets = dmo.prepare_targets(boxes, classes, TRAIN["sizes"])
    lg, bx = torch.tensor(g["train/logits"]), torch.tensor(g["train/boxes"])
    losses, _ = dco.criterion([(lg[l], bx[l]) for l in range(lg.shape[0])], targets, K, 0.1, (1.0, 5.0, 2.0))
    got = dmo.weighted(losses, wd)
    assert list(got) == list(g["train/keys"])
    np.testing.assert_allclose(np.array([float(v) for v in got.values()], dtype=np.float32), g["train/values"], rtol=1e-5, atol=1e-6)


def test_fixture_covers_the_cases():
    g = gold()
    assert len(g["infer/2/scores"]) == 0  # an image without kept queries
    assert (g["infer/0/labels"][:5] == 1).all()  # exact ties between classes 1 and 3 resolve to 1
    s3 = g["infer/3/scores"][:6].astype(np.float64)  # the kept half of the twelve near-threshold queries
    assert (s3 > THRESH).all() and (s3 - THRESH).max() < 3e-7 and (s3 - THRESH).min() < 1e-7
    logits, boxes = infer_case()
    s, _ = dmo.scores(logits)
    near = s[3, :12]
    assert (near > THRESH).sum() == 6 and (near <= THRESH).sum() == 6  # queries on both sides of the threshold, all within 3e-7 of it
    assert (near.double() - THRESH).abs().max() < 3e-7
    for b in (0, 1):  # kept queries whose boxes clip to empty are dropped by nonempty()
        kept = dmo.inference(logits, boxes, INFER["sizes"], INFER["out"], THRESH)[b]["keep"]
        assert (s[b, 10:13] > THRESH).all() and not any(q in kept for q in (10, 11, 12))
    sizes = [(int(h), int(w)) for h, w in INFER["out"]]
    assert sizes[0][0] > INFER["sizes"][0][0] and sizes[1][0] < INFER["sizes"][1][0]  # originals larger and smaller than the inputs
    assert len(g["targets/1/labels"]) == 0 and g["targets/1/boxes"].shape == (0, 4)
    # ceil(h / stride) reaches past a floor-sized map: image 2 of u8_ragged (33 x 81) at stride 32 on a 2 x 2 map
    assert not g["u8_ragged/mask3"][2].any() and g["u8_ragged/mask0"][2].any()
    keys = list(g["state_dict/keys"])
    assert keys[-1] == "criterion.empty_weight" and sum(k.startswith("detr.transformer.") for k in keys) == 182
    assert "detr.backbone.0.backbone.stem.weight" in keys
