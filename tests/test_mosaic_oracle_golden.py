"""CPU checks of the mosaic / random_perspective / mixup branch against tests/golden/mosaic.npz (the unmodified reference
`MyDatasetMapper2`, see oracle/gen_golden_mosaic.py):
  * oracle/mosaic_oracle.py reproduces every golden image from the sources and the draws;
  * `MosaicMixupMapper`, seeded like the reference, makes the same draws and computes the same `labels4`, boxes and classes bit for bit,
    and its recipes describe the golden images;
  * the fixture covers the branches the device kernels must get right."""
import copy
import random

import numpy as np
import pytest
import torch

cv2 = pytest.importorskip("cv2")

from oracle import gen_golden_mosaic as gen  # noqa: E402
from oracle import mosaic_oracle as orc  # noqa: E402
from yolov7_d2_b200.augment import MosaicMixupMapper, Yb200Error  # noqa: E402


class _MemMapper(MosaicMixupMapper):
    def _load_image_with_annos(self, dataset_dict):
        return gen.load_in_memory(dataset_dict)


@pytest.fixture(scope="module")
def replay():
    return orc.replay_golden(MosaicMixupMapper)


def _sources(x):
    return [s.numpy() for s in x["mosaic"]["sources"]]


def test_mapper_reproduces_draws_labels_and_boxes(replay):
    for n, (rec, x, e, _) in enumerate(replay):
        d = x["mosaic"]["draws"]
        for key in ("flag", "picks", "w", "h", "yc", "xc", "angle", "scale", "shear_x", "shear_y", "tx", "ty", "jit", "flip", "mix_picks",
                    "y_off", "x_off"):
            assert (key in e) == (key in d), (n, key)
            if key in e:
                assert e[key] == d[key], (n, key, e[key], d[key])
        b, c = x["instances"].gt_boxes.tensor.numpy(), x["instances"].gt_classes.numpy()
        assert b.dtype == np.float32 and np.array_equal(b, rec["boxes"]) and np.array_equal(c, rec["classes"]), n
        if x["mosaic"]["mode"] == 1:  # labels4 before annotations_to_instances, float64, bit for bit
            lab4 = np.concatenate([b.astype(np.float64), c[:, None].astype(np.float64)], 1)
            assert rec["labels4"].shape[0] >= lab4.shape[0]
            kept = ((rec["labels4"][:, 2] - rec["labels4"][:, 0]).astype(np.float32) > 1e-5)
            assert np.array_equal(rec["labels4"][:, :4].astype(np.float32)[kept], b)
        assert tuple(x["mosaic"]["size"]) == rec["img"].shape[1:], n


def test_oracle_and_recipes_reproduce_the_golden_images(replay):
    for n, (rec, x, e, _) in enumerate(replay):
        r = x["mosaic"]
        blend = bool(r.get("mixup", {}).get("blend", False))
        img = orc.render(_sources(x), r["draws"], blend)
        assert img.shape == rec["img"].shape and np.array_equal(img, rec["img"]), n


def test_fixture_covers_every_branch(replay):
    seen = set()
    for rec, x, e, name in replay:
        r = x["mosaic"]
        if r["mode"] == 0:
            seen.add("pass_through" if e.get("drawn") else "pass_through_warmup")
            continue
        h, w = r["input_dim"]
        seen.add(f"h_{'odd' if h % 2 else 'even'}")
        seen.add(f"w_{'odd' if w % 2 else 'even'}")
        if e.get("ratio_clamped"):
            seen.add("ratio_clamp")
        for (th, tw, xa1, ya1, xa2, ya2, _, _), s in zip(r["tiles"], r["sources"]):
            if (xa2 - xa1, ya2 - ya1) != (tw, th):
                seen.add("tile_clipped")
            sh, sw = s.shape[:2]
            seen.add("upscale" if th > sh else "downscale")
            if 2 * th == sh and 2 * tw == sw:
                seen.add("exact_2x")
        mix = r.get("mixup")
        if mix is not None:
            seen.add("mixup_blend" if mix["blend"] else "mixup_skipped")
            seen.add(f"flip_{bool(mix['flip'])}")
        if rec["img"].shape[1:] != (h, w):
            seen.add("odd_output_crop")
    need = {"pass_through_warmup", "pass_through", "h_odd", "h_even", "w_odd", "w_even", "ratio_clamp", "tile_clipped", "upscale", "downscale",
            "exact_2x", "mixup_blend", "mixup_skipped", "flip_True", "flip_False", "odd_output_crop"}
    assert need <= seen, need - seen
    # a tile without boxes: some mosaic uses a source whose dataset entry has no annotations
    g = gen.dataset(**gen.RUNS[0][1])
    empty = {d["image_id"] for d in g if not d["annotations"]}
    assert any(set(e.get("picks", [])) & empty for _, _, e, name in replay if name == "general")


def test_mapper_rejects_what_the_device_path_does_not_implement():
    cfg = dict(w=(20, 24), h=(20, 24), mixup=True)
    mt = gen.cfg_of(cfg)
    mt.PERSPECTIVE = 0.001
    with pytest.raises(Yb200Error, match="PERSPECTIVE"):
        _MemMapper(True, augmentations=[], image_format="BGR", mosaic_trans=mt)
    mt = gen.cfg_of(cfg)
    mt.NUM_IMAGES = 9
    with pytest.raises(Yb200Error, match="NUM_IMAGES"):
        _MemMapper(True, augmentations=[], image_format="BGR", mosaic_trans=mt)
    m = _MemMapper(True, augmentations=[], image_format="BGR", mosaic_trans=gen.cfg_of(cfg))
    d = gen.dataset(seed=5, n=1, sizes=(10, 12))[0]
    d["_img"] = d["_img"][..., :1].copy()
    with pytest.raises(Yb200Error, match="3-channel uint8"):
        m(d)


def test_mosaic_without_any_box_fails_like_the_reference():
    """dataset_mapper.py:459 calls `.shape` on the empty list `labels4` when no tile had a box: the mirror raises the same AttributeError"""
    cfg = dict(w=(20, 24), h=(20, 24), mixup=False)
    m = _MemMapper(True, augmentations=[], image_format="BGR", mosaic_trans=gen.cfg_of(cfg))
    data = gen.dataset(seed=6, n=6, sizes=(10, 20))
    for d in data:
        d["annotations"] = []
    random.seed(0)
    np.random.seed(1)
    with pytest.raises(AttributeError):
        for _ in range(40):
            m(copy.deepcopy(data[0]))


def test_mapper_recipes_hold_torch_uint8_sources(replay):
    for _, x, _, _ in replay[:20]:
        for s in x["mosaic"]["sources"]:
            assert isinstance(s, torch.Tensor) and s.dtype == torch.uint8 and s.dim() == 3 and s.shape[2] == 3 and not s.is_cuda
