"""oracle/sparseinst_criterion_oracle.py against the unmodified reference SparseInstMatcher / SparseInstCriterion
(tests/golden/sparseinst_criterion.npz, oracle/gen_golden_sparseinst_criterion.py), in fp64 on the CPU."""
import os

import numpy as np
import pytest
import torch

from oracle import sparseinst_criterion_oracle as sco

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "sparseinst_criterion.npz")
CASES = ("a_pad", "b_empty_image", "c_ragged", "d_weights", "e_g_eq_n")


@pytest.fixture(scope="module")
def gold():
    return np.load(GOLD, allow_pickle=False)


def load_case(gold, name, dtype=torch.float64):
    """a dict with the case's inputs (logits, masks, scores, mask_list, labels, sizes), shapes, matcher and loss settings"""
    p = name + "/"
    B, N, K, H, W, in_h, in_w = (int(v) for v in gold[p + "dims"])
    sizes = [int(s) for s in gold[p + "sizes"]]
    hw = gold[p + "image_hw"]
    bits = np.unpackbits(gold[p + "mask_bits"])
    mask_list, k = [], 0
    for g, (h, w) in zip(sizes, hw):
        n = g * int(h) * int(w)
        mask_list.append(torch.from_numpy(bits[k:k + n].astype(bool)).reshape(g, int(h), int(w)))
        k += n
    w = [float(v) for v in gold[p + "weights"]]
    return dict(B=B, N=N, K=K, size=(H, W), input_shape=(in_h, in_w), sizes=sizes, mask_list=mask_list,
                logits=torch.tensor(gold[p + "pred_logits"]).to(dtype),
                masks=(torch.tensor(gold[p + "logit_codes"]).double() * float(gold[p + "logit_step"])).to(dtype),  # exact: int8 codes × 2^-4
                scores=torch.tensor(gold[p + "pred_scores"]).to(dtype), labels=torch.tensor(gold[p + "labels"]),
                alpha=float(gold[p + "alpha_beta"][0]), beta=float(gold[p + "alpha_beta"][1]),
                weights=w, weight_dict=dict(zip(("loss_ce", "loss_mask", "loss_dice", "loss_objectness"), w)),
                items=tuple(str(s) for s in gold[p + "items"]), coef=dict(zip(sco.LOSS_KEYS, (float(c) for c in gold[p + "coef"]))))


def golden_indices(gold, name):
    p = name + "/"
    N = int(gold[p + "dims"][1])
    ii, jj = torch.tensor(gold[p + "idx_i"]), torch.tensor(gold[p + "idx_j"])
    out, k = [], 0
    for g in gold[p + "sizes"]:
        n = min(N, int(g))
        out.append((ii[k:k + n], jj[k:k + n]))
        k += n
    return out


def test_fixture_covers_the_cases(gold):
    dims = {n: [int(v) for v in gold[n + "/dims"]] for n in CASES}
    assert dims["a_pad"][:5] == [2, 100, 80, 40, 40] and dims["a_pad"][5:] == [160, 160]
    assert all(int(h) < 160 or int(w) < 160 for h, w in gold["a_pad/image_hw"])  # the padding is exercised
    assert list(gold["a_pad/sizes"]) == [3, 5] and 0 in list(gold["b_empty_image/sizes"])
    assert dims["c_ragged"][5] % dims["c_ragged"][3] and dims["c_ragged"][6] % dims["c_ragged"][4]
    assert list(gold["d_weights/alpha_beta"]) != [0.8, 0.2] and list(gold["d_weights/weights"]) != [2.0, 5.0, 2.0, 1.0]
    assert int(gold["e_g_eq_n/sizes"].max()) == dims["e_g_eq_n"][1]
    assert os.path.getsize(GOLD) < 1_100_000


@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_the_reference(gold, name):
    c = load_case(gold, name)
    p = name + "/"
    lg, mk, sc = (c[k].clone().requires_grad_(True) for k in ("logits", "masks", "scores"))
    losses, indices, blocks = sco.criterion(lg, mk, sc, c["mask_list"], c["labels"], c["input_shape"], c["alpha"], c["beta"], c["weight_dict"],
                                            c["items"])
    cost = torch.cat([b.flatten() for b in blocks])
    ref_cost = torch.tensor(gold[p + "cost"])
    assert torch.allclose(cost, ref_cost, rtol=1e-12, atol=1e-14)
    for (gi, gj), (ri, rj) in zip(indices, golden_indices(gold, name)):
        assert torch.equal(gi, ri) and torch.equal(gj, rj)
    assert list(losses.keys()) == [str(k) for k in gold[p + "keys"]]
    for k, ref in zip(losses, gold[p + "losses"]):
        assert abs(float(losses[k].detach()) - ref) <= 1e-6 * abs(ref) + 1e-12, (k, float(losses[k].detach()), ref)
    dl, dm, ds = sco.loss_gradients(lg, mk, sc, losses, c["coef"])
    B, N, K = c["B"], c["N"], c["K"]
    rows, mrows = torch.tensor(gold[p + "grad_rows"]), torch.tensor(gold[p + "mask_rows"])
    for got, ref in ((dl.reshape(B * N, K)[rows], gold[p + "dlogits"]), (dm.reshape(B * N, -1)[mrows], gold[p + "dmasks"]), (ds, gold[p + "dscores"])):
        ref = torch.tensor(ref)
        assert (got - ref).abs().max() <= 1e-6 * max(ref.abs().max().item(), 1e-30)
    unmatched = torch.ones(B * N, dtype=torch.bool)
    unmatched[mrows] = False
    assert dm.reshape(B * N, -1)[unmatched].abs().max() == 0
