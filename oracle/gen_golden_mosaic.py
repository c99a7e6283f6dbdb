"""TEST INFRASTRUCTURE -- tests/golden/mosaic.npz: the UNMODIFIED reference `MyDatasetMapper2.__call__` (yolov7/data/dataset_mapper.py:339-767,
with `random_perspective` / `box_candidates` from yolov7/data/transforms/data_augment.py:16-102, imported through oracle/ref_shim.py) on small
in-memory images.  Run in the build container only:  python -m oracle.gen_golden_mosaic

The detectron2 pieces the mapper touches are stubbed here with detectron2's semantics: `annotations_to_instances` (fp32 `Boxes`, int64 classes)
and `filter_empty_instances` (keep w > 1e-5 and h > 1e-5).  `_load_image_with_annos` is overridden to load from memory, `augmentations=[]`.

Per call the fixture records every draw the reference made (the module-level `random` / `np.random` functions it calls are wrapped, not
changed), the output image (CHW uint8), `labels4` as handed to `_labels_to_annos`, and the final boxes / classes.
"""
import copy
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_shim  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "mosaic.npz")


class _Instances:
    def __init__(self, image_size):
        self.image_size = image_size


class _Boxes:
    def __init__(self, t):
        self.tensor = torch.as_tensor(t, dtype=torch.float32).reshape(-1, 4)


def _annotations_to_instances(annos, image_size, mask_format="polygon"):
    inst = _Instances(image_size)
    boxes = [np.asarray(a["bbox"], dtype=np.float64) for a in annos]
    inst.gt_boxes = _Boxes(np.stack(boxes) if boxes else np.zeros((0, 4)))
    inst.gt_classes = torch.tensor([int(a["category_id"]) for a in annos], dtype=torch.int64)
    return inst


def _filter_empty_instances(inst, by_box=True, by_mask=True, box_threshold=1e-5):
    b = inst.gt_boxes.tensor
    keep = ((b[:, 2] - b[:, 0]) > box_threshold) & ((b[:, 3] - b[:, 1]) > box_threshold)
    out = _Instances(inst.image_size)
    out.gt_boxes = _Boxes(b[keep])
    out.gt_classes = inst.gt_classes[keep]
    return out


def _install_data_stubs():
    ref_shim.install()

    def _mod(name, **attrs):
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        sys.modules[name] = m
        return m

    class _CfgNode(dict):
        pass

    class _AugmentationList:
        def __init__(self, augs):
            self.augs = list(augs)

        def __call__(self, aug_input):
            return []

    class _BoxMode:
        XYXY_ABS, XYWH_ABS = 0, 1

    class _DatasetMapper:
        pass

    t = _mod("detectron2.data.transforms", AugmentationList=_AugmentationList, Augmentation=object, Transform=object,
             AugInput=object, RandomFlip=object, RandomBrightness=object, RandomLighting=object, RandomSaturation=object)
    utils = _mod("detectron2.data.detection_utils", annotations_to_instances=_annotations_to_instances,
                 filter_empty_instances=_filter_empty_instances)
    data = _mod("detectron2.data", transforms=t, detection_utils=utils)
    data.__path__ = []
    _mod("detectron2.data.dataset_mapper", DatasetMapper=_DatasetMapper)
    _mod("detectron2.config", configurable=lambda f: f, CfgNode=_CfgNode)
    _mod("detectron2.structures", BoxMode=_BoxMode)
    _mod("yolov7.data.detection_utils", build_augmentation=None, transform_instance_annotations=None, vis_annos=None)
    alfred = sys.modules["alfred"]
    alfred.__path__ = []
    _mod("alfred.utils").__path__ = []
    _mod("alfred.utils.log", logger=alfred.logger)
    for sub in (".data", ".data.transforms"):
        ref_shim._pkg("yolov7" + sub, os.path.join(ref_shim.REF, "yolov7", *sub.strip(".").split(".")))


class _Recorder:
    """forwards attribute access to a module (`random` or `np.random`) and logs every draw of the named functions"""

    def __init__(self, target, names, log, tag):
        self._t, self._names, self._log, self._tag = target, names, log, tag

    def __getattr__(self, name):
        f = getattr(self._t, name)
        if name not in self._names:
            return f

        def wrapped(*a, **k):
            r = f(*a, **k)
            if name == "choice":
                self._log.append((self._tag + "." + name, [d["image_id"] for d in np.atleast_1d(r)]))
            else:
                self._log.append((self._tag + "." + name, r))
            return r

        return wrapped


def dataset(seed, n, sizes, two_x=None):
    """in-memory dataset dicts: images HWC uint8 BGR, XYXY_ABS boxes with fractional corners; every 5th image has no boxes"""
    rng = np.random.default_rng(seed)
    out = []
    for k in range(n):
        if two_x is not None and k % 3 == 0:
            h, w = two_x
        else:
            h, w = int(rng.integers(*sizes)), int(rng.integers(*sizes))
        img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        img[: h // 4] = rng.integers(0, 256, 3, dtype=np.uint8)  # a flat band: exact interpolation results
        annos = []
        for _ in range(0 if k % 5 == 4 else int(rng.integers(1, 5))):
            x1, y1 = rng.uniform(-2, w - 3), rng.uniform(-2, h - 3)
            x2, y2 = x1 + rng.uniform(0.5, w / 1.5), y1 + rng.uniform(0.5, h / 1.5)
            annos.append({"bbox": [float(max(x1, 0)), float(max(y1, 0)), float(min(x2, w)), float(min(y2, h))],
                          "bbox_mode": 0, "category_id": int(rng.integers(0, 80))})
        out.append({"image_id": k, "file_name": f"mem://{k}", "height": h, "width": w, "annotations": annos, "_img": img})
    return out


# (name, dataset args, mosaic config, seed, calls)
RUNS = [
    ("general", dict(seed=1, n=24, sizes=(9, 41)), dict(w=(20, 33), h=(17, 31), mixup=True), 11, 60),
    ("nomix", dict(seed=2, n=16, sizes=(12, 30)), dict(w=(21, 27), h=(21, 27), mixup=False), 12, 24),
    ("two_x", dict(seed=3, n=12, sizes=(10, 30), two_x=(48, 44)), dict(w=(22, 22), h=(24, 24), mixup=True), 13, 30),
]


def cfg_of(c):
    return types.SimpleNamespace(ENABLED=True, POOL_CAPACITY=8, NUM_IMAGES=4, DEGREES=10.0, TRANSLATE=0.1, SCALE=[0.5, 1.5],
                                 MSCALE=[0.5, 1.5], SHEAR=2.0, PERSPECTIVE=0.0, ENABLE_MIXUP=c["mixup"],
                                 MOSAIC_WIDTH_RANGE=c["w"], MOSAIC_HEIGHT_RANGE=c["h"], DEBUG_VIS=False)


def load_in_memory(dataset_dict):
    """what `_load_image_with_annos` returns for a training image without augmentations: the image and XYXY_ABS annotations"""
    annos = [{"bbox": np.asarray(a["bbox"], dtype=np.float64), "category_id": a["category_id"], "bbox_mode": 0}
             for a in dataset_dict.pop("annotations") if a.get("iscrowd", 0) == 0]
    return dataset_dict["_img"].copy(), annos


def run(Mapper, data, c, seed, calls, log):
    """`calls` calls of a fresh mapper after seeding both generators; None if the reference raised"""
    import random

    m = Mapper(True, augmentations=[], image_format="BGR", mosaic_trans=cfg_of(c), input_size=[640, 640])
    random.seed(seed)
    np.random.seed(seed)
    order = np.random.default_rng(seed).integers(0, len(data), calls)
    outs = []
    for k in order:
        del log[:]
        m._labels4 = None
        try:
            out = m(copy.deepcopy(data[int(k)]))
        except (AttributeError, IndexError):  # no tile had a box (dataset_mapper.py:459) / a mixup source without boxes (:741)
            return None
        outs.append({"img": out["image"].numpy(), "boxes": out["instances"].gt_boxes.tensor.numpy(),
                     "classes": out["instances"].gt_classes.numpy(),
                     "labels4": m._labels4 if m._labels4 is not None else np.zeros((0, 5)), "draws": np.array(repr(log))})
    return order, outs


def main():
    import importlib
    import random

    _install_data_stubs()
    dm = importlib.import_module("yolov7.data.dataset_mapper")
    da = importlib.import_module("yolov7.data.transforms.data_augment")

    class Mapper(dm.MyDatasetMapper2):
        def _load_image_with_annos(self, dataset_dict):
            return load_in_memory(dataset_dict)

        def _labels_to_annos(self, labels):
            self._labels4 = np.array(labels, dtype=np.float64).reshape(-1, 5)
            return super()._labels_to_annos(labels)

    log = []
    dm.random = da.random = _Recorder(random, ("uniform", "randint"), log, "random")
    dm.np = types.SimpleNamespace(**{k: getattr(np, k) for k in dir(np) if not k.startswith("__")})
    dm.np.random = _Recorder(np.random, ("randint", "choice"), log, "np")
    rec = {}
    cases = []
    for name, dargs, c, seed0, calls in RUNS:
        data = dataset(**dargs)
        for seed in range(seed0, seed0 + 1000):  # the first seed whose calls all complete
            got = run(Mapper, data, c, seed, calls, log)
            if got is not None:
                break
        for j, (k, out) in enumerate(zip(*got)):
            i = len(cases)
            rec.update({f"{f}_{i}": v for f, v in out.items()})
            cases.append((name, seed, j, int(k)))
    rec["cases"] = np.array([f"{n}:{sd}:{j}:{k}" for n, sd, j, k in cases])
    np.savez_compressed(OUT, **rec)
    print(f"wrote {OUT}: {len(cases)} calls, {os.path.getsize(OUT)} bytes")


if __name__ == "__main__":
    main()
