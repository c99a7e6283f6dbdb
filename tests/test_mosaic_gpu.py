"""Device stages of the mosaic / random_perspective / mixup branch (`yb200_mosaic_warp`, `yb200_mosaic_mixup`, `augment.apply_mosaic`) against
the reference's images (tests/golden/mosaic.npz) and against oracle/mosaic_oracle.py (cv2) at the default mosaic sizes, and the YOLOX training
step on a recipe batch against the same images handed over as plain CUDA tensors.

Pixel bound: max |diff| <= 1 and at least 99.9 % identical bytes per image.  The resize and the warp restate cv2's integer arithmetic and
are expected to be exact; the one known source of a difference is the mixup's float64 resize, whose last bits differ from cv2's (about 1e-12)
and can move a value that sits on an integer across the uint8 truncation (csrc/augment.cu)."""
import copy

import numpy as np
import pytest
import torch

cv2 = pytest.importorskip("cv2")

from oracle import mosaic_oracle as orc  # noqa: E402
from yolov7_d2_b200 import capi  # noqa: E402
from yolov7_d2_b200.augment import MosaicMixupMapper, Yb200Error, apply_mosaic  # noqa: E402

pytestmark = pytest.mark.gpu


def _check_image(got, ref, what):
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    d = np.abs(got.astype(np.int16) - ref.astype(np.int16))
    same = float((d == 0).mean())
    assert d.max() <= 1 and same >= 0.999, (what, int(d.max()), same)
    return same


@pytest.fixture(scope="module")
def golden(cuda):
    return orc.replay_golden(MosaicMixupMapper)


def test_golden_images_boxes_and_sizes(golden):
    batch = [x for _, x, _, _ in golden]
    apply_mosaic(batch)
    torch.cuda.synchronize()
    worst, exact = 1.0, 0
    for n, ((rec, _, _, _), x) in enumerate(zip(golden, batch)):
        img = x["image"]
        assert img.is_cuda and img.dtype == torch.uint8 and "mosaic" not in x
        same = _check_image(img.cpu().numpy(), rec["img"], n)
        worst, exact = min(worst, same), exact + (same == 1.0)
        assert tuple(img.shape[1:]) == rec["img"].shape[1:]  # odd h / w give h - 1 / w - 1 like the reference
        inst = x["instances"]
        assert inst.gt_boxes.tensor.is_cuda and np.array_equal(inst.gt_boxes.tensor.cpu().numpy(), rec["boxes"])
        assert np.array_equal(inst.gt_classes.cpu().numpy(), rec["classes"])
    print(f"golden: {exact}/{len(batch)} images bit-exact, worst identical fraction {worst:.6f}")


def _recipe_batch(n, seed, mixup):
    return orc.synthetic_recipes(MosaicMixupMapper, n, seed, mixup=mixup)


@pytest.mark.parametrize("mixup", [True, False])
def test_default_ranges_against_the_cv2_oracle(cuda, mixup):
    """64 samples at MOSAIC_*_RANGE (512, 800) from 420..640 px sources, rendered in one call; the oracle runs in the test"""
    batch = _recipe_batch(64, 3 if mixup else 4, mixup)
    expect = [orc.render([s.numpy() for s in x["mosaic"]["sources"]], x["mosaic"]["draws"],
                         bool(x["mosaic"].get("mixup", {}).get("blend", False))) for x in batch]
    assert not mixup or sum(bool(x["mosaic"].get("mixup", {}).get("blend")) for x in batch) > 8
    apply_mosaic(batch)
    torch.cuda.synchronize()
    worst, exact = 1.0, 0
    for n, (x, ref) in enumerate(zip(batch, expect)):
        same = _check_image(x["image"].cpu().numpy(), ref, n)
        worst, exact = min(worst, same), exact + (same == 1.0)
    print(f"default ranges, mixup={mixup}: {exact}/64 bit-exact, worst identical fraction {worst:.6f}")


def test_two_runs_give_identical_bytes(cuda):
    batch = _recipe_batch(16, 5, True)
    a, b = copy.deepcopy(batch), copy.deepcopy(batch)
    apply_mosaic(a)
    apply_mosaic(b)
    torch.cuda.synchronize()
    for x, y in zip(a, b):
        assert torch.equal(x["image"], y["image"])


def test_argument_rejection(cuda):
    L = capi.lib()
    t = torch.zeros(1024, dtype=torch.uint8, device=cuda)
    p = capi.ptr(t)
    st = capi.stream_ptr()
    assert L.yb200_mosaic_warp(None, 1, p, p, 8, 8, st) == capi.ERR_INVALID
    assert L.yb200_mosaic_warp(p, 0, p, p, 8, 8, st) == capi.ERR_INVALID
    assert L.yb200_mosaic_mixup(p, 1, None, p, 8, 8, st) == capi.ERR_INVALID
    assert L.yb200_mosaic_mixup(p, 1, p, p, 0, 8, st) == capi.ERR_INVALID
    assert b"mosaic_mixup" in L.yb200_last_error()
    x = _recipe_batch(1, 6, False)[0]
    bad = copy.deepcopy(x)
    bad["mosaic"]["sources"][2] = bad["mosaic"]["sources"][2][..., :2].contiguous()
    with pytest.raises(Yb200Error, match="3-channel uint8"):
        apply_mosaic([bad])
    bad = copy.deepcopy(x)
    bad["mosaic"]["sources"][1] = bad["mosaic"]["sources"][1].float()
    with pytest.raises(Yb200Error, match="3-channel uint8"):
        apply_mosaic([bad])


@pytest.fixture(scope="module")
def model(cuda):
    import bench
    from oracle import yolox_oracle as yo
    from yolov7_d2_b200.modeling import YOLOX

    m = YOLOX(bench.yolox_s_cfg("cuda"))
    m.load_state_dict(yo.yolox_state_dict(4), strict=True)
    m.train()
    return m


def _small_batch(seed):
    return orc.synthetic_recipes(MosaicMixupMapper, 4, seed, size_range=(120, 160), src_range=(90, 200))


def _plain(recipes):
    """the same batch with the rendered images as plain CUDA tensors (a copy, so nothing is shared with the recipe batch)"""
    b = copy.deepcopy(recipes)
    apply_mosaic(b)
    for x in b:
        x["image"] = x["image"].clone()
    return b


def _step(m, batch, prefetch=False):
    m.zero_grad(set_to_none=True)
    if prefetch:
        m.prefetch(batch)
    out = m(batch)
    sum(out.values()).backward()
    torch.cuda.synchronize()
    return [float(v.detach()) for v in out.values()], m.engine.flat_grad.clone()


@pytest.mark.parametrize("prefetch", [False, True])
def test_training_step_on_recipes_matches_plain_images(model, prefetch):
    recipes = _small_batch(7 + int(prefetch))
    plain = _plain(recipes)
    loss_p, grad_p = _step(model, plain)
    loss_r, grad_r = _step(model, recipes, prefetch)
    assert all("image" in x and "mosaic" not in x for x in recipes)
    assert loss_r == loss_p, (loss_r, loss_p)
    assert torch.equal(grad_r, grad_p)
