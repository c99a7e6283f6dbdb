"""The DETR meta-architecture on one GPU: this package's kernels against the reference's torch arithmetic on the same GPU and tensors.

Workload (seeded; config 4's shapes, DETR-R50 at 800 x 1333 with 16 images): uint8 images 16 x 800 x 1333, or a ragged batch with heights in
640..800 and widths in 1000..1333; the stand-in backbone returns one fixed [16, 2048, 25, 42] feature map that requires grad.
  (a) input: this package's normalisation (one yb200_normalize_pad) plus masks and positions (one yb200_detr_mask_pos), against the reference's
      per-image normalisation, ImageList padding, mask_out_padding and PositionEmbeddingSine in torch (oracle/detr_model_oracle.py); for the
      res5 level alone, and for four levels at strides 4 / 8 / 16 / 32 as a res2..res5 backbone would give (Joiner computes every level);
  (b) eval: Detr.inference (yb200_detr_infer, one copy of the counts, one synchronisation) against the reference's `inference` plus a
      per-image detector_postprocess in torch, on fixed outputs pred_logits [16, 100, 81] and pred_boxes [16, 100, 4];
  (c) a whole Detr training step after the backbone (the torchvision DETR config: 256 wide, 8 heads, 6 + 6 layers, FFN 2048, 100 queries,
      80 classes, dropout 0.1, deep supervision): input, transformer, heads, criterion, backward;
  (d) bytes and FLOPs computed from the shapes (floors, not measurements).
Times are CUDA events over --iters repetitions after --warmup, and every measurement is repeated --repeats times to show the spread.  The card
name, power limit and max SM clock are read in the same run.
usage: python tools/bench_detr_model.py [--iters N] [--warmup N] [--repeats N] [--out results.json]
"""
import argparse
import json
import os
import subprocess
import sys
import types

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import detr_model_oracle as dmo  # noqa: E402
from oracle.gen_golden_detr_model import cfg_of  # noqa: E402
from yolov7_d2_b200 import modeling  # noqa: E402
from yolov7_d2_b200.batch_input import normalize_pad  # noqa: E402
from yolov7_d2_b200.detr_model import Detr, PositionEmbeddingSine  # noqa: E402

B, Q, K1, C, HF, WF, D, FFN = 16, 100, 81, 2048, 25, 42, 256, 2048
H, W = 800, 1333
MEAN, STD = (123.675, 116.280, 103.530), (58.395, 57.120, 57.375)
HBM_BPS, BF16_FLOPS = 3.35e12, 989e12  # H100 SXM data sheet


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        power = q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"
    except Exception:  # noqa: BLE001
        power = "unknown"
    return name, power


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def level_shapes(strides):
    return [(B, C, -(-H // s), -(-W // s)) for s in strides]


def pos_bytes(strides):
    return sum(4 * 2 * 128 * B * h * w + B * h * w for _, _, h, w in level_shapes(strides))


def transformer_flops():
    """forward multiply-adds x 2 of input_proj, 6 encoder and 6 decoder layers and the heads; the step's floor is 3x (forward + backward)"""
    T = HF * WF
    enc = 2 * T * (4 * D * D + 2 * D * FFN) + 4 * T * T * D
    dec = 2 * Q * (4 * D * D + 2 * D * D + 2 * D * FFN) + 2 * T * 2 * D * D + 4 * Q * Q * D + 4 * Q * T * D
    heads = 2 * 6 * Q * (D * K1 + 2 * D * D + D * 4)
    return B * (2 * T * C * D + 6 * enc + 6 * dec + heads)


class FixedBackbone(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.feat = torch.nn.Parameter(torch.randn(B, C, HF, WF, generator=torch.Generator().manual_seed(1)).cuda())

    def output_shape(self):
        return {"res5": types.SimpleNamespace(channels=C, stride=32)}

    def forward(self, x):
        return {"res5": self.feat}


def batch(ragged, targets=False):
    g = torch.Generator().manual_seed(2 + ragged)
    out = []
    for b in range(B):
        h, w = (int(torch.randint(640, 801, (1,), generator=g)), int(torch.randint(1000, 1334, (1,), generator=g))) if ragged else (H, W)
        x = {"image": torch.randint(0, 256, (3, h, w), generator=g, dtype=torch.uint8), "height": 480, "width": 640}
        if targets:
            n = int(torch.randint(1, 20, (1,), generator=g))
            xy = torch.rand(n, 2, generator=g) * torch.tensor([w * 0.7, h * 0.7])
            bx = torch.cat([xy, xy + torch.rand(n, 2, generator=g) * torch.tensor([w * 0.3, h * 0.3]) + 4], 1)
            x["instances"] = modeling.Instances((h, w), gt_boxes=modeling.Boxes(bx), gt_classes=torch.randint(0, 80, (n,), generator=g))
        out.append(x)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_detr_model needs a CUDA device")
    dev = torch.device("cuda")
    name, power = card()
    print(f"card: {name}; power limit, max SM clock: {power}")
    if "build_detr_fixed_backbone" not in modeling.BACKBONE_REGISTRY:
        def build_detr_fixed_backbone(cfg, input_shape=None):
            return FixedBackbone()

        modeling.BACKBONE_REGISTRY.register(build_detr_fixed_backbone)
    torch.manual_seed(0)
    model = Detr(cfg_of(device="cuda", backbone="build_detr_fixed_backbone"))
    res = {"card": name, "power_limit_max_sm_clock": power, "runs": []}
    mean, std = model.pixel_mean, model.pixel_std
    pe = PositionEmbeddingSine(128, normalize=True)
    g = torch.Generator().manual_seed(5)
    logits = (torch.randn(B, Q, K1, generator=g) * 3).to(dev)
    boxes = torch.sigmoid(torch.randn(B, Q, 4, generator=g)).to(dev)
    train_batch = {r: batch(r, targets=True) for r in (False, True)}
    for rep in range(args.repeats):
        run = {}
        for ragged in (False, True):
            tag = "ragged" if ragged else "full"
            imgs = [x["image"] for x in batch(ragged)]
            sizes = [(int(i.shape[1]), int(i.shape[2])) for i in imgs]
            imgs_d = [i.to(dev) for i in imgs]
            for lv, strides in (("res5", [32]), ("res2-res5", [4, 8, 16, 32])):
                shapes = level_shapes(strides)

                def ours():
                    normalize_pad(model.L, imgs_d, mean, std, 0, "bench")
                    pe(shapes, strides, sizes, dev)

                def ref():
                    dmo.preprocess(imgs_d, MEAN, STD)
                    for m in dmo.mask_out_padding(shapes, strides, sizes, device=dev):
                        dmo.position_sine(m, 128)

                run[f"a_input_{lv}_{tag}_ms"] = timed(ours, args.iters, args.warmup)
                run[f"a_input_{lv}_{tag}_reference_ms"] = timed(ref, max(2, args.iters // 4), 2)
        outs = [(480, 640)] * B
        sizes = [(H, W)] * B
        run["b_eval_ms"] = timed(lambda: model.inference(logits, boxes, sizes, outs), args.iters, args.warmup)
        run["b_eval_reference_ms"] = timed(lambda: dmo.inference(logits, boxes.clone(), sizes, outs, model.ignore_thresh), args.iters, args.warmup)
        model.train()
        for ragged in (False, True):
            tb = train_batch[ragged]

            def step():
                model.zero_grad(set_to_none=True)
                losses = model(tb)
                sum(v for k, v in losses.items() if k.startswith("loss_")).backward()

            run[f"c_train_step_{'ragged' if ragged else 'full'}_ms"] = timed(step, max(3, args.iters // 4), 2)
        res["runs"].append(run)
        print(json.dumps({"repeat": rep, **{k: round(v, 3) for k, v in run.items()}}))
    img_bytes = B * 3 * H * W * (1 + 4)
    floors = {"a_bytes_res5": img_bytes + pos_bytes([32]), "a_bytes_res2_res5": img_bytes + pos_bytes([4, 8, 16, 32]),
              "a_unused_level_bytes_res2_res4": pos_bytes([4, 8, 16]), "b_bytes": 4 * B * Q * (K1 + 4),
              "c_flops_fwd_bwd": 3 * transformer_flops()}
    floors["a_floor_ms_res5"] = floors["a_bytes_res5"] / HBM_BPS * 1e3
    floors["a_floor_ms_res2_res5"] = floors["a_bytes_res2_res5"] / HBM_BPS * 1e3
    floors["c_floor_ms_bf16"] = floors["c_flops_fwd_bwd"] / BF16_FLOPS * 1e3
    res["floors_from_shapes"] = floors
    print(json.dumps({"floors_from_shapes": floors}))
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
