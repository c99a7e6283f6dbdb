"""Mosaic, `random_perspective` and mixup of the YOLOX training mapper (`MyDatasetMapper2`, yolov7/data/dataset_mapper.py:339-767) with the
pixels on the GPU.

`MosaicMixupMapper` is a drop-in for `MyDatasetMapper2`.  It runs in the dataloader workers and never touches CUDA: it keeps the mosaic pool,
makes every random draw of the reference in the reference's order (`np.random` for the pool, the mosaic size and the mixup source, `random` for
the centre, the affine warp and the mixup), computes the final boxes on the host in float64 exactly like the reference, and returns instead of
`"image"` a `"mosaic"` recipe: the source images as uint8 HWC tensors (so detectron2's dataloader moves them through shared memory) and the
scalars the two device stages need.  `apply_mosaic(batched_inputs)` then renders every recipe of a batch with two launches
(`yb200_mosaic_warp`, `yb200_mosaic_mixup`) and replaces `"mosaic"` by `"image"`: a CUDA uint8 CHW tensor of the reference's output size.
`YOLOX.forward` and `YOLOX.prefetch` call it for batches that carry recipes.

Unsupported settings raise `Yb200Error`: PERSPECTIVE != 0 (warpPerspective), NUM_IMAGES != 4, sources that are not 3-channel uint8.
"""
import copy
import math
import random
from collections import deque

import numpy as np
import torch

from . import capi
from .capi import MosaicDesc, Yb200Error
from .modeling import Boxes, Instances

try:  # the per-image loading of the reference (dataset_mapper.py:641-684); tests replace `_load_image_with_annos`
    from detectron2.data import detection_utils as d2_utils
    from detectron2.data import transforms as d2_T
except Exception:  # noqa: BLE001
    d2_utils = d2_T = None

MAX_SOURCES = capi.MOSAIC_MAX_SOURCES


def box_candidates(box1, box2, wh_thr=2, ar_thr=20, area_thr=0.2):
    """data_augment.py:16-28: keep boxes wider and taller than wh_thr, with aspect ratio below ar_thr and area ratio above area_thr"""
    w1, h1 = box1[2] - box1[0], box1[3] - box1[1]
    w2, h2 = box2[2] - box2[0], box2[3] - box2[1]
    ar = np.maximum(w2 / (h2 + 1e-16), h2 / (w2 + 1e-16))
    return (w2 > wh_thr) & (h2 > wh_thr) & (w2 * h2 / (w1 * h1 + 1e-16) > area_thr) & (ar < ar_thr)


def _rotation(angle_deg, scale):
    """cv2.getRotationMatrix2D(angle, center=(0, 0), scale)[:2]"""
    t = angle_deg * (math.pi / 180)
    a, b = math.cos(t) * scale, math.sin(t) * scale
    return np.array([[a, b, 0.0], [-b, a, 0.0]])


def invert_affine(m):
    """the inverse cv2.warpAffine samples with (imgwarp.cpp, invertAffineTransform order of operations)"""
    m = [float(v) for v in np.asarray(m).reshape(-1)[:6]]
    d = m[0] * m[4] - m[1] * m[3]
    d = 1.0 / d if d != 0 else 0.0
    a11, a22, a12, a21 = m[4] * d, m[0] * d, m[1] * -d, m[3] * -d
    return (a11, a12, -a11 * m[2] - a12 * m[5], a21, a22, -a21 * m[2] - a22 * m[5])


def _instances(labels, image_size):
    """annotations_to_instances + filter_empty_instances: fp32 XYXY boxes, int64 classes, keep w > 1e-5 and h > 1e-5"""
    inst = Instances(image_size)
    b = torch.as_tensor(np.asarray(labels[:, :4], dtype=np.float64), dtype=torch.float32).reshape(-1, 4)
    c = torch.tensor([int(v) for v in labels[:, 4]], dtype=torch.int64)
    keep = ((b[:, 2] - b[:, 0]) > 1e-5) & ((b[:, 3] - b[:, 1]) > 1e-5)
    inst.gt_boxes = Boxes(b[keep])
    inst.gt_classes = c[keep]
    return inst


def _check_source(img):
    if not (isinstance(img, np.ndarray) and img.dtype == np.uint8 and img.ndim == 3 and img.shape[2] == 3):
        raise Yb200Error(f"mosaic sources must be HWC 3-channel uint8 images, got {getattr(img, 'dtype', type(img))} "
                         f"{getattr(img, 'shape', '')}")
    return img


def _cfg_get(node, key, default=None):
    return getattr(node, key, default) if not isinstance(node, dict) else node.get(key, default)


class MosaicMixupMapper:
    """Drop-in for `MyDatasetMapper2` (dataset_mapper.py:339-767): `MosaicMixupMapper(cfg, True)` or the reference's keyword form."""

    def __init__(self, *args, **kwargs):
        if args and not isinstance(args[0], bool) and hasattr(args[0], "INPUT"):
            kwargs = {**self.from_config(*args, **kwargs)}
            args = ()
        self._init(*args, **kwargs)

    def _init(self, is_train, *, augmentations, image_format, mosaic_trans, use_instance_mask=False, use_keypoint=False,
              instance_mask_format="polygon", recompute_boxes=False, add_meta_infos=False, input_size=(640, 640)):
        self.is_train = is_train
        self.augmentations = d2_T.AugmentationList(augmentations) if d2_T is not None else list(augmentations)
        self.image_format = image_format
        self.use_instance_mask, self.use_keypoint = use_instance_mask, use_keypoint
        self.instance_mask_format, self.recompute_boxes, self.add_meta_infos = instance_mask_format, recompute_boxes, add_meta_infos
        self.input_size = input_size
        self.mosaic_trans = mt = mosaic_trans
        self.enable_aug = True
        if _cfg_get(mt, "ENABLED"):
            if float(_cfg_get(mt, "PERSPECTIVE", 0.0)) != 0.0:
                raise Yb200Error("MosaicMixupMapper: PERSPECTIVE != 0 needs warpPerspective, which the device path does not implement")
            if int(_cfg_get(mt, "NUM_IMAGES", 4)) != 4:
                raise Yb200Error(f"MosaicMixupMapper: NUM_IMAGES must be 4, got {_cfg_get(mt, 'NUM_IMAGES')}")
            self.mosaic_pool = deque(maxlen=mt.POOL_CAPACITY)
            self.degrees, self.translate, self.scale = mt.DEGREES, mt.TRANSLATE, mt.SCALE
            self.mixup_scale, self.shear, self.perspective, self.enable_mixup = mt.MSCALE, mt.SHEAR, mt.PERSPECTIVE, mt.ENABLE_MIXUP

    @classmethod
    def from_config(cls, cfg, is_train=True):
        """dataset_mapper.py:418-441"""
        try:
            from yolov7.data.detection_utils import build_augmentation
            augs = build_augmentation(cfg, is_train)
        except ImportError:
            augs = []
        recompute = False
        if cfg.INPUT.CROP.ENABLED and is_train:
            augs.insert(0, d2_T.RandomCrop(cfg.INPUT.CROP.TYPE, cfg.INPUT.CROP.SIZE))
            recompute = cfg.MODEL.MASK_ON
        return {"is_train": is_train, "augmentations": augs, "image_format": cfg.INPUT.FORMAT, "mosaic_trans": cfg.INPUT.MOSAIC_AND_MIXUP,
                "use_instance_mask": cfg.MODEL.MASK_ON, "instance_mask_format": cfg.INPUT.MASK_FORMAT,
                "use_keypoint": cfg.MODEL.KEYPOINT_ON, "recompute_boxes": recompute, "add_meta_infos": cfg.INPUT.JITTER_CROP.ENABLED,
                "input_size": cfg.INPUT.INPUT_SIZE}

    def disable_aug(self):
        self.enable_aug = False

    # -- per-image loading (dataset_mapper.py:641-684) ------------------------------------------------------------------------------
    def _load_image_with_annos(self, dataset_dict):
        if d2_utils is None:
            raise Yb200Error("MosaicMixupMapper: loading images from files needs detectron2; override _load_image_with_annos otherwise")
        from yolov7.data.detection_utils import transform_instance_annotations

        image = d2_utils.read_image(dataset_dict["file_name"], format=self.image_format)
        d2_utils.check_image_size(dataset_dict, image)
        aug_input = d2_T.AugInput(image)
        transforms = self.augmentations(aug_input)
        image = aug_input.image
        if not self.is_train:
            dataset_dict.pop("annotations", None)
            dataset_dict.pop("sem_seg_file_name", None)
            return image, None
        if "annotations" not in dataset_dict:
            return image, None
        for anno in dataset_dict["annotations"]:
            if not self.use_instance_mask:
                anno.pop("segmentation", None)
            if not self.use_keypoint:
                anno.pop("keypoints", None)
        annos = [transform_instance_annotations(obj, transforms, image.shape[:2], add_meta_infos=self.add_meta_infos)
                 for obj in dataset_dict.pop("annotations") if obj.get("iscrowd", 0) == 0]
        return image, annos

    @staticmethod
    def _anno_to_labels(annos):
        """rows [x1, y1, x2, y2, cls] in float64 (an empty array without columns when there is no box)"""
        return np.array([np.append(a["bbox"], a["category_id"]) for a in annos] if annos is not None else [])

    # -- the mapper ----------------------------------------------------------------------------------------------------------------
    def __call__(self, dataset_dict):
        dataset_dict = copy.deepcopy(dataset_dict)
        mt = self.mosaic_trans
        flag, picks, draws = 0, None, {}
        if _cfg_get(mt, "ENABLED") and self.is_train and self.enable_aug:
            if len(self.mosaic_pool) > mt.NUM_IMAGES:
                flag = int(np.random.randint(2))  # dataset_mapper.py:492; choice below draws like np.random.choice(pool, 3)
                if flag == 1:
                    picks = [self.mosaic_pool[i] for i in np.random.choice(len(self.mosaic_pool), mt.NUM_IMAGES - 1)]
            self.mosaic_pool.append(copy.deepcopy(dataset_dict))
        draws["flag"] = flag
        img, annos = self._load_image_with_annos(dataset_dict)
        _check_source(img)
        if self.is_train and flag == 1 and picks is not None and self.enable_aug:
            draws["picks"] = [p.get("image_id") for p in picks]
            return self._mosaic(dataset_dict, img, annos, picks, draws)
        h, w = img.shape[:2]
        if annos is not None:
            lab = self._anno_to_labels(annos).reshape(-1, 5)
            dataset_dict["instances"] = _instances(lab, (h, w))
        dataset_dict["mosaic"] = {"mode": 0, "sources": [torch.from_numpy(np.ascontiguousarray(img))], "size": (h, w), "draws": draws}
        return dataset_dict

    def _mosaic(self, dataset_dict, img, annos, picks, draws):
        mt = self.mosaic_trans
        w = int(np.random.randint(mt.MOSAIC_WIDTH_RANGE[0], mt.MOSAIC_WIDTH_RANGE[1] + 1))
        h = int(np.random.randint(mt.MOSAIC_HEIGHT_RANGE[0], mt.MOSAIC_HEIGHT_RANGE[1] + 1))
        if max(w / h, h / w) > 1.2:
            h = min(h, w)
            w = int(1.2 * h)
        yc = int(random.uniform(0.5 * h, 1.5 * h))
        xc = int(random.uniform(0.5 * w, 1.5 * w))
        draws.update(w=w, h=h, yc=yc, xc=xc)
        sources, tiles, labels4 = [], [], []
        for i in range(4):
            if i:
                img, annos = self._load_image_with_annos(copy.deepcopy(picks[i - 1]))
                _check_source(img)
            lab = self._anno_to_labels(annos)
            h0, w0 = img.shape[:2]
            s = min(1.0 * h / h0, 1.0 * w / w0)
            th, tw = int(h0 * s), int(w0 * s)
            if i == 0:    # top left
                xa1, ya1, xa2, ya2 = max(xc - tw, 0), max(yc - th, 0), xc, yc
                xb1, yb1 = tw - (xa2 - xa1), th - (ya2 - ya1)
            elif i == 1:  # top right
                xa1, ya1, xa2, ya2 = xc, max(yc - th, 0), min(xc + tw, 2 * w), yc
                xb1, yb1 = 0, th - (ya2 - ya1)
            elif i == 2:  # bottom left
                xa1, ya1, xa2, ya2 = max(xc - tw, 0), yc, xc, min(2 * h, yc + th)
                xb1, yb1 = tw - (xa2 - xa1), 0
            else:         # bottom right
                xa1, ya1, xa2, ya2 = xc, yc, min(xc + tw, 2 * w), min(2 * h, yc + th)
                xb1, yb1 = 0, 0
            padw, padh = xa1 - xb1, ya1 - yb1
            sources.append(torch.from_numpy(np.ascontiguousarray(img)))
            tiles.append((th, tw, xa1, ya1, xa2, ya2, padw, padh))
            if lab.size > 0:
                lab = lab.copy()
                lab[:, 0] = s * lab[:, 0] + padw
                lab[:, 1] = s * lab[:, 1] + padh
                lab[:, 2] = s * lab[:, 2] + padw
                lab[:, 3] = s * lab[:, 3] + padh
                labels4.append(lab)
        if labels4:
            labels4 = np.concatenate(labels4, 0)
            for c, hi in ((0, 2 * w), (1, 2 * h), (2, 2 * w), (3, 2 * h)):
                np.clip(labels4[:, c], 0, hi, out=labels4[:, c])
        labels4, m, out_hw = self._perspective(labels4, h, w, draws)
        recipe = {"mode": 1, "sources": sources, "tiles": tiles, "input_dim": (h, w), "size": out_hw, "matrix": m, "draws": draws}
        if self.enable_mixup and len(labels4) != 0:
            labels4 = self._mixup(labels4, (h, w), out_hw, recipe, draws)
        if isinstance(labels4, list):  # no tile had a box: the reference fails in `_labels_to_annos` (dataset_mapper.py:459)
            raise AttributeError("'list' object has no attribute 'shape'")
        dataset_dict["instances"] = _instances(labels4.reshape(-1, 5), out_hw)
        dataset_dict["mosaic"] = recipe
        return dataset_dict

    def _perspective(self, targets, h, w, draws):
        """random_perspective (data_augment.py:31-102) on the 2h x 2w canvas with border (-h // 2, -w // 2)"""
        height, width = 2 * h + 2 * (-h // 2), 2 * w + 2 * (-w // 2)
        C = np.eye(3)
        C[0, 2], C[1, 2] = -(2 * w) / 2, -(2 * h) / 2
        R = np.eye(3)
        a = random.uniform(-self.degrees, self.degrees)
        s = random.uniform(self.scale[0], self.scale[1])
        R[:2] = _rotation(a, s)
        S = np.eye(3)
        S[0, 1] = math.tan(random.uniform(-self.shear, self.shear) * math.pi / 180)
        S[1, 0] = math.tan(random.uniform(-self.shear, self.shear) * math.pi / 180)
        T = np.eye(3)
        T[0, 2] = random.uniform(0.5 - self.translate, 0.5 + self.translate) * width
        T[1, 2] = random.uniform(0.5 - self.translate, 0.5 + self.translate) * height
        draws.update(angle=a, scale=s, shear_x=S[0, 1], shear_y=S[1, 0], tx=T[0, 2], ty=T[1, 2])
        M = T @ S @ R @ C
        n = len(targets)
        if n:
            xy = np.ones((n * 4, 3))
            xy[:, :2] = targets[:, [0, 1, 2, 3, 0, 3, 2, 1]].reshape(n * 4, 2)
            xy = (xy @ M.T)[:, :2].reshape(n, 8)
            x, y = xy[:, [0, 2, 4, 6]], xy[:, [1, 3, 5, 7]]
            xy = np.concatenate((x.min(1), y.min(1), x.max(1), y.max(1))).reshape(4, n).T
            xy[:, [0, 2]] = xy[:, [0, 2]].clip(0, width)
            xy[:, [1, 3]] = xy[:, [1, 3]].clip(0, height)
            keep = box_candidates(box1=targets[:, :4].T * s, box2=xy.T)
            targets = targets[keep]
            targets[:, :4] = xy[keep]
        return targets, M[:2].copy(), (height, width)

    def _mixup(self, labels, input_dim, out_hw, recipe, draws):
        """mixup (dataset_mapper.py:686-767): draws, boxes and the blend decision; the pixels are stage B's"""
        jit = random.uniform(*self.mixup_scale)
        flip = random.uniform(0, 1) > 0.5
        annos = None
        picks = []
        while annos is None:  # the reference loops on `annos == None`: a source with an empty box list ends the loop
            d = copy.deepcopy(self.mosaic_pool[int(np.random.choice(len(self.mosaic_pool), 1)[0])])
            picks.append(d.get("image_id"))
            img, annos = self._load_image_with_annos(d)
        _check_source(img)
        cp_labels = self._anno_to_labels(annos)
        h, w = input_dim
        r = min(h / img.shape[0], w / img.shape[1])
        mix_h, mix_w = int(img.shape[0] * r), int(img.shape[1] * r)
        jit_h, jit_w = int(h * jit), int(w * jit)
        r *= jit
        th, tw = out_hw
        ph, pw = max(jit_h, th), max(jit_w, tw)
        y_off = random.randint(0, ph - th - 1) if ph > th else 0
        x_off = random.randint(0, pw - tw - 1) if pw > tw else 0
        draws.update(jit=jit, flip=flip, mix_picks=picks, y_off=y_off, x_off=x_off)
        bb = cp_labels[:, :4]  # IndexError for a source without boxes, as in the reference (dataset_mapper.py:741)
        bb[:, 0::2] = np.clip(bb[:, 0::2] * r + 0, 0, jit_w)
        bb[:, 1::2] = np.clip(bb[:, 1::2] * r + 0, 0, jit_h)
        if flip:
            bb[:, 0::2] = jit_w - bb[:, 0::2][:, ::-1]
        tr = bb.copy()
        tr[:, 0::2] = np.clip(tr[:, 0::2] - x_off, 0, tw)
        tr[:, 1::2] = np.clip(tr[:, 1::2] - y_off, 0, th)
        keep = box_candidates(bb.T, tr.T, 5)
        blend = bool(keep.sum() >= 1.0)
        if blend:
            labels = np.vstack((labels, np.hstack((tr[keep], cp_labels[keep, 4:5]))))
        recipe["sources"].append(torch.from_numpy(np.ascontiguousarray(img)))
        recipe["mixup"] = {"blend": blend, "mix_hw": (mix_h, mix_w), "jit_hw": (jit_h, jit_w), "flip": flip, "offset": (y_off, x_off)}
        return labels


def has_recipes(batched_inputs):
    return any("mosaic" in x for x in batched_inputs)


def build_table(recipes):
    """host side of `apply_mosaic`: (table as a uint8 tensor, byte offset of every source, total source bytes, output offsets, sizes)"""
    n = len(recipes)
    table = (MosaicDesc * n)()
    src_total, out_total, sizes = 0, 0, []
    for d, r in zip(table, recipes):
        srcs = r["sources"]
        if not 1 <= len(srcs) <= MAX_SOURCES:
            raise Yb200Error(f"apply_mosaic: a recipe has {len(srcs)} sources")
        for k, s in enumerate(srcs):
            if s.dtype != torch.uint8 or s.dim() != 3 or s.shape[2] != 3:
                raise Yb200Error(f"apply_mosaic: sources must be HWC 3-channel uint8, got {s.dtype} {tuple(s.shape)}")
            d.src_off[k], d.src_h[k], d.src_w[k] = src_total, s.shape[0], s.shape[1]
            src_total += s.numel()
        oh, ow = (int(v) for v in r["size"])
        d.out_off, d.out_h, d.out_w = out_total, oh, ow
        out_total += 3 * oh * ow
        sizes.append((oh, ow))
        d.mode = int(r["mode"])
        if d.mode == 1:
            if len(srcs) < 4:
                raise Yb200Error("apply_mosaic: a mosaic recipe needs four tile sources")
            d.in_h, d.in_w = r["input_dim"]
            for k, (th, tw, xa1, ya1, xa2, ya2, padw, padh) in enumerate(r["tiles"]):
                d.tile_h[k], d.tile_w[k] = th, tw
                d.rect[4 * k:4 * k + 4] = (xa1, ya1, xa2, ya2)
                d.pad[2 * k:2 * k + 2] = (padw, padh)
            d.minv[:] = invert_affine(r["matrix"])
            mix = r.get("mixup")
            if mix is not None and mix["blend"]:
                if len(srcs) != 5:
                    raise Yb200Error("apply_mosaic: a blended mixup needs its source")
                d.mix = 1
                d.mix_h, d.mix_w = mix["mix_hw"]
                d.jit_h, d.jit_w = mix["jit_hw"]
                d.flip = int(bool(mix["flip"]))
                d.y_off, d.x_off = mix["offset"]
        elif (oh, ow) != tuple(srcs[0].shape[:2]):
            raise Yb200Error("apply_mosaic: a pass-through recipe must keep its source size")
    raw = torch.frombuffer(bytearray(bytes(table)), dtype=torch.uint8)
    return raw, src_total, out_total, sizes


def apply_mosaic(batched_inputs):
    """Render every `"mosaic"` recipe of the batch on the current CUDA stream and replace it by `"image"` (uint8 CHW on the device); the
    recipes' `instances` move to the device.  Returns the device tensors it made (images, boxes, classes).  Dicts without a recipe are left
    as they are."""
    idx = [k for k, x in enumerate(batched_inputs) if "mosaic" in x]
    if not idx:
        return []
    recipes = [batched_inputs[k]["mosaic"] for k in idx]
    raw, src_total, out_total, sizes = build_table(recipes)
    dev = torch.device("cuda", torch.cuda.current_device())
    src = torch.empty(src_total, dtype=torch.uint8, device=dev)
    off = 0
    for r in recipes:  # one asynchronous copy per source into the packed buffer
        for s in r["sources"]:
            n = s.numel()
            src[off:off + n].copy_(s.reshape(-1), non_blocking=True)
            off += n
    table = raw.to(dev, non_blocking=True)
    out = torch.empty(out_total, dtype=torch.uint8, device=dev)
    max_h = max(h for h, _ in sizes)
    max_w = max(w for _, w in sizes)
    L, st = capi.lib(), capi.stream_ptr()
    capi.check(L.yb200_mosaic_warp(capi.ptr(table), len(recipes), capi.ptr(src), capi.ptr(out), max_h, max_w, st), "yb200_mosaic_warp")
    if any(r.get("mixup") is not None and r["mixup"]["blend"] for r in recipes):
        capi.check(L.yb200_mosaic_mixup(capi.ptr(table), len(recipes), capi.ptr(src), capi.ptr(out), max_h, max_w, st), "yb200_mosaic_mixup")
    made, o = [], 0
    for k, (h, w) in zip(idx, sizes):
        x = batched_inputs[k]
        img = out[o:o + 3 * h * w].view(3, h, w)
        o += 3 * h * w
        x["image"] = img
        del x["mosaic"]
        made.append(img)
        inst = x.get("instances")
        if inst is not None:
            dinst = Instances(inst.image_size)
            dinst.gt_boxes = Boxes(inst.gt_boxes.tensor.to(dev, non_blocking=True))
            dinst.gt_classes = inst.gt_classes.to(dev, non_blocking=True)
            x["instances"] = dinst
            made += [dinst.gt_boxes.tensor, dinst.gt_classes]
    return made
