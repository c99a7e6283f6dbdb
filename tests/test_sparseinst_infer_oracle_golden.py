"""CPU: oracle/sparseinst_infer_oracle.py against tests/golden/sparseinst_infer.npz, written by oracle/gen_golden_sparseinst_infer.py from the
unmodified reference SparseInst.preprocess_inputs / inference.  Labels, keep sets, the empty-image structure and the masks are exact; scores
agree within 1e-6 relative; the normalised batch is bit-identical."""
import os

import numpy as np
import pytest
from oracle import sparseinst_infer_oracle as sio
from oracle.gen_golden_sparseinst_infer import CASES, CLS_THRESHOLD, MASK_THRESHOLD, MEAN, STD, case_inputs

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sparseinst_infer.npz")


def gold():
    return np.load(GOLD, allow_pickle=False)


@pytest.mark.parametrize("name", list(CASES))
def test_oracle_reproduces_the_reference(name):
    g = gold()
    images, logits, obj, masks, batched = case_inputs(name)
    batch, sizes = sio.preprocess(images, MEAN, STD)
    assert np.array_equal(batch.numpy(), g[f"{name}/images"]), "normalised batch differs"
    ori = [(x["height"], x["width"]) for x in batched]
    res = sio.inference(logits, obj, masks, batch.shape[2:], sizes, ori, CLS_THRESHOLD, MASK_THRESHOLD)
    for b, r in enumerate(res):
        key = f"{name}/{b}"
        assert np.array_equal(r["labels"].numpy(), g[f"{key}/labels"]), key
        np.testing.assert_allclose(r["scores"].numpy(), g[f"{key}/scores"], rtol=1e-6, atol=0)
        assert bool(g[f"{key}/has_masks"]) == (r["masks"] is not None), key
        if r["masks"] is not None:
            assert tuple(g[f"{key}/mask_shape"]) == tuple(r["masks"].shape) == (len(r["labels"]), *ori[b])
            assert np.array_equal(np.packbits(r["masks"].numpy(), axis=-1), g[f"{key}/masks"]), key


def test_fixture_covers_the_cases():
    g = gold()
    assert not bool(g["b_empty/1/has_masks"]) and g["b_empty/1/scores"].size == 0 and bool(g["b_empty/0/has_masks"])
    assert (g["c_ties/0/labels"] == 2).any()  # the duplicated largest class resolves to its lower index
    _, logits, obj, _, _ = case_inputs("c_ties")
    s, lab = sio.scores(logits, obj)
    assert (lab == 2).sum() > lab.numel() // 2 and not (lab == 5).any()  # class 5 duplicates class 2: never chosen
    sizes = [tuple(g[f"a_mixed/{b}/mask_shape"][1:]) for b in range(3)]
    assert sizes == [(80, 120), (40, 56), (66, 82)]  # originals larger and smaller than the images
    # near-threshold masks: the fp64 composite lies within 1e-2 of MASK_THRESHOLD everywhere, and both sides occur
    _, logits, obj, masks, batched = case_inputs("d_near")
    c = sio.composite(masks[0].double(), (64, 64), (64, 64), (96, 96))
    assert (c - MASK_THRESHOLD).abs().max() < 1e-2 and (c > MASK_THRESHOLD).any() and (c < MASK_THRESHOLD).any()
