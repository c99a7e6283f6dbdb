"""CPU: autograd through oracle/sparseinst_oracle.py in float64 reproduces the gradients of the unmodified reference decoders
(tests/golden/sparseinst_bwd.npz, oracle/gen_golden_sparseinst_bwd.py): d features and every parameter's gradient, Base and Group, on non-square
maps; and the storage-emulating restatement (oracle/sparseinst_storage_oracle.py) stays within bf16 storage error of them.  The GPU tests judge
the kernels' backward against these two."""
import numpy as np
import pytest
import torch

from oracle import sparseinst_oracle as sio
from oracle import sparseinst_storage_oracle as sso
from oracle.gen_golden_sparseinst_bwd import CASES, OUT, case_upstream, features, state_dict, unpack


def oracle_grads(forward, case):
    """{name: gradient} (and "features") of a decoder forward for the case's upstream gradients, float64"""
    _, groups, _, _, _, _, d = case
    feat = features(case).requires_grad_(True)
    sd = {k: v.double().requires_grad_(True) for k, v in state_dict(case).items()}
    out = forward(feat, sd, num_convs=d["convs"], groups=groups)
    torch.autograd.backward([out["pred_logits"], out["pred_masks"], out["pred_scores"]], list(case_upstream(case)))
    g = {k: v.grad for k, v in sd.items()}
    g["features"] = feat.grad
    return g


def gold_grads(case):
    name = case[0]
    gold = np.load(OUT, allow_pickle=False)
    assert list(gold[f"{name}/meta"]) == list(case[1:6])
    g = {k[len(f"{name}/grad/"):]: unpack(gold, k) for k in gold.files if k.startswith(f"{name}/grad/") and not k.endswith("/scale")}
    g["features"] = unpack(gold, f"{name}/d_features")
    return g


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_oracle_backward_matches_reference(case):
    ref, got = gold_grads(case), oracle_grads(sio.decoder_forward, case)
    assert sorted(ref) == sorted(got)
    for k in ref:
        assert got[k].shape == ref[k].shape, (k, got[k].shape, ref[k].shape)
        err, mx = (got[k] - ref[k]).abs().max().item(), ref[k].abs().max().item()
        assert err <= 2.0 ** -11 * mx, f"{case[0]} {k}: max err {err:.3g} (max |ref| {mx:.3g})"  # the fixture's float16 storage


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_storage_emulating_oracle_is_close_to_reference(case):
    """the bf16 storage points move the gradients, but not grossly: relative L2 < 25 % (the IAM bias gradient, a cancelling sum over the
    probabilities, moves most: ~9 % here)"""
    ref, emu = gold_grads(case), oracle_grads(sso.decoder_forward, case)
    errs = {k: float((emu[k] - ref[k]).norm() / ref[k].norm()) for k in ref}
    assert all(e < 0.25 for e in errs.values()), errs
    assert max(errs.values()) > 2.0 ** -12, errs
