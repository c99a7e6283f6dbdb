"""CPU: oracle/sparseinst_encoder_oracle.py in float64 reproduces the unmodified reference InstanceContextEncoder (tests/golden/sparseinst_encoder.npz,
oracle/gen_golden_sparseinst_encoder.py): the output, d res3 / res4 / res5 and every parameter's gradient on maps whose pyramid pooling hits
MyAdaptiveAvgPool2d's floor quirk; and the storage-emulating forward stays within bf16 storage error of them.  The GPU tests judge the kernels
against these two."""
import numpy as np
import pytest
import torch

from oracle import sparseinst_encoder_oracle as seo
from oracle.gen_golden_sparseinst_bwd import unpack
from oracle.gen_golden_sparseinst_encoder import CASES, OUT, features, state_dict, upstream


def oracle_run(forward, case):
    """(output, {name: gradient}) of an encoder forward for the case's upstream gradient, float64; inputs under "d_res3" etc."""
    feats = {k: v.requires_grad_(True) for k, v in features(case).items()}
    sd = {k: v.double().requires_grad_(True) for k, v in state_dict(case).items()}
    out = forward(feats, sd)
    out.backward(upstream(case))
    g = {k: v.grad for k, v in sd.items()}
    g.update({f"d_{k}": v.grad for k, v in feats.items()})
    return out.detach(), g


def gold(case):
    name = case[0]
    z = np.load(OUT, allow_pickle=False)
    assert list(z[f"{name}/meta"]) == list(case[1:])
    g = {k[len(f"{name}/grad/"):]: unpack(z, k) for k in z.files if k.startswith(f"{name}/grad/") and not k.endswith("/scale")}
    g.update({f"d_{k}": unpack(z, f"{name}/d_{k}") for k in seo.IN_FEATURES})
    return unpack(z, f"{name}/out"), g


def test_ppm_windows_floor_quirk():
    """MyAdaptiveAvgPool2d is avg_pool2d with window ceil(H/s): the pooled maps are not s x s"""
    pooled = lambda h, w: [(h // kh, w // kw) for kh, kw in seo.ppm_windows(h, w)]  # noqa: E731
    assert pooled(20, 20) == [(1, 1), (2, 2), (2, 2), (5, 5)]
    assert pooled(20, 27) == [(1, 1), (2, 1), (2, 3), (5, 5)]
    assert pooled(5, 7) == [(1, 1), (1, 1), (2, 2), (5, 3)]
    assert pooled(4, 6) == [(1, 1), (2, 2), (2, 3), (4, 6)]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_oracle_matches_reference(case):
    ref_out, ref = gold(case)
    out, got = oracle_run(seo.encoder_forward, case)
    assert sorted(ref) == sorted(got)
    assert out.shape == ref_out.shape
    assert (out - ref_out).abs().max() <= 2.0 ** -11 * ref_out.abs().max()  # the fixture's float16 storage
    for k in ref:
        assert got[k].shape == ref[k].shape, (k, got[k].shape, ref[k].shape)
        err, mx = (got[k] - ref[k]).abs().max().item(), ref[k].abs().max().item()
        assert err <= 2.0 ** -11 * mx, f"{case[0]} {k}: max err {err:.3g} (max |ref| {mx:.3g})"


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_storage_emulating_oracle_is_close_to_reference(case):
    """the bf16 storage points move the gradients, but not grossly: relative L2 < 25 % (the PPM stage convolutions' gradients move most, ~15 %
    at the 5x7 top level: a 1x1 or 1x2 prior's gradient is the sum of the bf16 d priors over the whole map, a cancelling sum)"""
    ref_out, ref = gold(case)
    out, emu = oracle_run(seo.encoder_forward_storage, case)
    errs = {k: float((emu[k] - ref[k]).norm() / ref[k].norm()) for k in ref}
    errs["out"] = float((out - ref_out).norm() / ref_out.norm())
    assert all(e < 0.25 for e in errs.values()), errs
    assert max(errs.values()) > 2.0 ** -12, errs
