"""TEST INFRASTRUCTURE -- the pixels of the YOLOX mosaic branch (MyDatasetMapper2, yolov7/data/dataset_mapper.py:504-611 and mixup :686-767,
random_perspective data_augment.py:31-74) restated with numpy and cv2 as a pure function of the sources and the random draws.

`render(sources, draws, blend)` -> CHW uint8.  `sources` are the HWC uint8 images in the mapper's order (the current image, the three pool
samples, the mixup source), `draws` the values the mapper drew (`MosaicMixupMapper` records them in `recipe["draws"]`), `blend` whether the
mixup kept a box (the host's decision).  No draw is made here.
"""
import math
import os

import cv2
import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "mosaic.npz")


def mosaic_canvas(sources, h, w, yc, xc):
    img4 = np.full((2 * h, 2 * w, 3), 114, dtype=np.uint8)
    for i, src in enumerate(sources[:4]):
        h0, w0 = src.shape[:2]
        s = min(1.0 * h / h0, 1.0 * w / w0)
        t = cv2.resize(src, (int(w0 * s), int(h0 * s)), interpolation=cv2.INTER_LINEAR)
        th, tw = t.shape[:2]
        if i == 0:
            xa, ya, xb, yb = max(xc - tw, 0), max(yc - th, 0), xc, yc
            img4[ya:yb, xa:xb] = t[th - (yb - ya):th, tw - (xb - xa):tw]
        elif i == 1:
            xa, ya, xb, yb = xc, max(yc - th, 0), min(xc + tw, 2 * w), yc
            img4[ya:yb, xa:xb] = t[th - (yb - ya):th, 0:min(tw, xb - xa)]
        elif i == 2:
            xa, ya, xb, yb = max(xc - tw, 0), yc, xc, min(2 * h, yc + th)
            img4[ya:yb, xa:xb] = t[0:min(yb - ya, th), tw - (xb - xa):tw]
        else:
            xa, ya, xb, yb = xc, yc, min(xc + tw, 2 * w), min(2 * h, yc + th)
            img4[ya:yb, xa:xb] = t[0:min(yb - ya, th), 0:min(tw, xb - xa)]
    return img4


def affine(h, w, d):
    """M = T S R C of random_perspective for the 2h x 2w canvas, and the output size"""
    height, width = 2 * h + 2 * (-h // 2), 2 * w + 2 * (-w // 2)
    C = np.eye(3)
    C[0, 2], C[1, 2] = -w, -h
    R = np.eye(3)
    R[:2] = cv2.getRotationMatrix2D(angle=d["angle"], center=(0, 0), scale=d["scale"])
    S = np.eye(3)
    S[0, 1], S[1, 0] = d["shear_x"], d["shear_y"]
    T = np.eye(3)
    T[0, 2], T[1, 2] = d["tx"], d["ty"]
    return T @ S @ R @ C, (height, width)


def mixup_image(src, h, w, out_hw, d):
    """the padded, cropped mixup image (uint8 HWC) the blend adds"""
    cp = np.ones((h, w, 3)) * 114.0
    r = min(h / src.shape[0], w / src.shape[1])
    rh, rw = int(src.shape[0] * r), int(src.shape[1] * r)
    cp[:rh, :rw] = cv2.resize(src, (rw, rh), interpolation=cv2.INTER_LINEAR).astype(np.float32)
    cp = cv2.resize(cp, (int(w * d["jit"]), int(h * d["jit"])))
    if d["flip"]:
        cp = cp[:, ::-1, :]
    oh, ow = cp.shape[:2]
    th, tw = out_hw
    padded = np.zeros((max(oh, th), max(ow, tw), 3)).astype(np.uint8)
    padded[:oh, :ow] = cp
    return padded[d["y_off"]:d["y_off"] + th, d["x_off"]:d["x_off"] + tw]


def render(sources, draws, blend=False):
    if draws.get("flag", 0) != 1:
        return np.ascontiguousarray(sources[0].transpose(2, 0, 1))
    h, w = draws["h"], draws["w"]
    img4 = mosaic_canvas(sources, h, w, draws["yc"], draws["xc"])
    M, (height, width) = affine(h, w, draws)
    img = cv2.warpAffine(img4, M[:2], dsize=(width, height), borderValue=(114, 114, 114))
    if blend:
        mix = mixup_image(sources[4], h, w, (height, width), draws)
        img = (0.5 * img.astype(np.float32) + 0.5 * mix.astype(np.float32)).astype(np.uint8)
    return np.ascontiguousarray(img.transpose(2, 0, 1))


def synthetic_recipes(mapper_cls, n, seed, size_range=(512, 800), src_range=(420, 641), mixup=True):
    """`n` mapper calls at the default mosaic ranges on random uint8 sources with random boxes (every call after the pool warm-up is a
    mosaic; mixup on or off): returns the `n` mosaic samples the mapper produced"""
    import random
    import types

    rng = np.random.default_rng(seed)
    data = []
    for k in range(max(8, n // 4)):
        hh, ww = (int(v) for v in rng.integers(*src_range, 2))
        img = rng.integers(0, 256, (hh, ww, 3), dtype=np.uint8)
        img[: hh // 3] = rng.integers(0, 256, 3, dtype=np.uint8)
        boxes = []
        for _ in range(int(rng.integers(1, 6))):
            x1, y1 = rng.uniform(0, ww * 0.7), rng.uniform(0, hh * 0.7)
            boxes.append({"bbox": [x1, y1, min(ww, x1 + rng.uniform(8, ww * 0.5)), min(hh, y1 + rng.uniform(8, hh * 0.5))],
                          "category_id": int(rng.integers(0, 80)), "bbox_mode": 0})
        data.append({"image_id": k, "annotations": boxes, "_img": img})
    mt = types.SimpleNamespace(ENABLED=True, POOL_CAPACITY=1000, NUM_IMAGES=4, DEGREES=10.0, TRANSLATE=0.1, SCALE=[0.5, 1.5],
                               MSCALE=[0.5, 1.5], SHEAR=2.0, PERSPECTIVE=0.0, ENABLE_MIXUP=mixup, MOSAIC_WIDTH_RANGE=size_range,
                               MOSAIC_HEIGHT_RANGE=size_range)

    class M(mapper_cls):
        def _load_image_with_annos(self, d):
            return d["_img"], [{"bbox": np.asarray(a["bbox"], dtype=np.float64), "category_id": a["category_id"]} for a in d.pop("annotations")]

    m = M(True, augmentations=[], image_format="BGR", mosaic_trans=mt)
    random.seed(seed)
    np.random.seed(seed)
    for d in data[:5]:  # fill the pool
        m(d)
    out = []
    while len(out) < n:
        x = m(data[int(rng.integers(0, len(data)))])
        if x["mosaic"]["mode"] == 1:
            out.append(x)
    return out


def expected_draws(log, j, pool_before):
    """the reference's draws of call j, read from its recorded log in the order dataset_mapper.py makes them"""
    it = iter(log)
    e = {"flag": 0}
    if pool_before > 4:
        e["drawn"] = True
        e["flag"] = int(next(it)[1])
        if e["flag"]:
            e["picks"] = next(it)[1]
    if not e["flag"]:
        return e
    w, h = int(next(it)[1]), int(next(it)[1])
    if max(w / h, h / w) > 1.2:
        e["ratio_clamped"] = True
        h = min(h, w)
        w = int(1.2 * h)
    e.update(w=w, h=h, yc=int(next(it)[1]), xc=int(next(it)[1]), angle=next(it)[1], scale=next(it)[1])
    e["shear_x"] = math.tan(next(it)[1] * math.pi / 180)
    e["shear_y"] = math.tan(next(it)[1] * math.pi / 180)
    height, width = 2 * h + 2 * (-h // 2), 2 * w + 2 * (-w // 2)
    e["tx"], e["ty"] = next(it)[1] * width, next(it)[1] * height
    rest = list(it)
    if rest:
        e["jit"], e["flip"] = rest[0][1], rest[1][1] > 0.5
        e["mix_picks"] = [v[0] for name, v in rest[2:] if name == "np.choice"]
        offs = [v for name, v in rest[2:] if name == "random.randint"]
        jh, jw = int(h * e["jit"]), int(w * e["jit"])
        e["y_off"] = offs.pop(0) if max(jh, height) > height else 0
        e["x_off"] = offs.pop(0) if max(jw, width) > width else 0
        assert not offs
    return e


def replay_golden(mapper_cls, path=GOLDEN):
    """Replays tests/golden/mosaic.npz through `mapper_cls` (seeded like the reference, loading in memory): a list of (golden record,
    mapper output, the draws the reference made, run name) per recorded call"""
    import copy
    import random

    from oracle import gen_golden_mosaic as gen

    class _MemMapper(mapper_cls):
        def _load_image_with_annos(self, dataset_dict):
            return gen.load_in_memory(dataset_dict)

    g = np.load(path)
    cases = [c.split(":") for c in g["cases"]]
    runs = {name: (d, c) for name, d, c, _, _ in gen.RUNS}
    out, i = [], 0
    for name in dict.fromkeys(c[0] for c in cases):
        mine = [c for c in cases if c[0] == name]
        seed = int(mine[0][1])
        dargs, cfg = runs[name]
        data = gen.dataset(**dargs)
        m = _MemMapper(True, augmentations=[], image_format="BGR", mosaic_trans=gen.cfg_of(cfg), input_size=[640, 640])
        random.seed(seed)
        np.random.seed(seed)
        for j, (_, _, jj, k) in enumerate(mine):
            assert int(jj) == j
            pool_before = len(m.mosaic_pool)
            x = m(copy.deepcopy(data[int(k)]))
            log = eval(str(g[f"draws_{i}"]), {"np": np})  # noqa: S307 -- the fixture's own repr of the draws
            rec = {f: g[f"{f}_{i}"] for f in ("img", "boxes", "classes", "labels4")}
            out.append((rec, x, expected_draws(log, j, pool_before), name))
            i += 1
    assert i == len(cases)
    return out
