"""SparseInst inference on one GPU: this package's kernels against the reference's `inference` arithmetic in torch on the same GPU and tensors.

Workload (seeded): 16 images at the shipped test size (MIN_SIZE_TEST 640, MAX_SIZE_TEST 853): each COCO-like image is 480 x 640, resized to
640 x 853, padded to 640 x 864; the decoder's outputs are pred_logits [16, 100, 80], pred_scores [16, 100, 1] and pred_masks
[16, 100, 160, 216]; CONF_THRESHOLD 0.01 keeps nearly all 100 queries.
  (a) device inference: yb200_sparseinst_infer_scores, one copy of the 16 keep counts, yb200_sparseinst_paste_masks (SparseInst.inference);
  (b) the reference's inference (sparseinst.py:179-232) in torch, restated by oracle/sparseinst_infer_oracle.py: the per-image loop with two
      fp32 F.interpolate calls per kept mask;
  (c) InstanceContextEncoder + GroupIAMDecoder + (a) from given ResNet-50-shaped res3 / res4 / res5 [16, 512 | 1024 | 2048, 80 x 108 | 40 x 54 |
      20 x 27].
Times are CUDA events over --iters repetitions after --warmup.  Also printed: the card name, power limit and max SM clock read in the same run,
the number of mask pixels where (a) and (b) disagree, and byte counts computed from the shapes (not measurements): the least traffic of (a)
and the traffic of (b)'s chain, each with its time at the data sheet's HBM bandwidth.
usage: python tools/bench_sparseinst_infer.py [--iters N] [--warmup N] [--out results.json]
"""
import argparse
import json
import os
import subprocess
import sys
import types

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import sparseinst_infer_oracle as sio  # noqa: E402
from yolov7_d2_b200 import capi  # noqa: E402
from yolov7_d2_b200.sparseinst import GroupIAMDecoder  # noqa: E402
from yolov7_d2_b200.sparseinst_encoder import InstanceContextEncoder  # noqa: E402
from yolov7_d2_b200.sparseinst_model import SparseInst  # noqa: E402

B, N, K = 16, 100, 80
IMG, PAD, ORI = (640, 853), (640, 864), (480, 640)
HM, WM = PAD[0] // 4, PAD[1] // 4
CLS_THRESHOLD, MASK_THRESHOLD = 0.01, 0.45
HBM_BPS = 3.35e12  # H100 SXM HBM3, data sheet


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        power = q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"
    except Exception:  # noqa: BLE001
        power = "unknown"
    return name, power


def floor_bytes(kept):
    """(a): read the logits, objectness and every mask once, write the kept bool masks"""
    return 4 * (B * N * K + B * N + B * N * HM * WM) + kept * ORI[0] * ORI[1]


def reference_bytes(kept):
    """(b)'s chain from the shapes: sigmoid of all masks (read + write), the kept masks gathered, resize A (read, write fp32 at the padded size),
    the strided crop read by resize B, resize B written in fp32, read again by the threshold, the bool masks written"""
    f = 4
    return (2 * f * B * N * HM * WM + 2 * f * kept * HM * WM + f * kept * PAD[0] * PAD[1] + f * kept * IMG[0] * IMG[1]
            + 2 * f * kept * ORI[0] * ORI[1] + kept * ORI[0] * ORI[1])


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(iters):
        fn()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_sparseinst_infer needs a CUDA device")
    dev = torch.device("cuda:0")
    name, power = card()
    g = torch.Generator().manual_seed(0)
    out = {"pred_logits": (torch.randn(B, N, K, generator=g) * 2 - 3).to(dev), "pred_scores": torch.randn(B, N, 1, generator=g).to(dev),
           "pred_masks": (torch.randn(B, N, HM, WM, generator=g) * 2).to(dev)}
    batched = [{"height": ORI[0], "width": ORI[1]} for _ in range(B)]
    stub = types.SimpleNamespace(L=capi.lib(), device=dev, cls_threshold=CLS_THRESHOLD, mask_threshold=MASK_THRESHOLD)
    device_inference = lambda o: SparseInst.inference(stub, o, batched, PAD, [IMG] * B)  # noqa: E731
    reference = lambda: sio.inference(out["pred_logits"], out["pred_scores"], out["pred_masks"], PAD, [IMG] * B, [ORI] * B, CLS_THRESHOLD,  # noqa: E731
                                      MASK_THRESHOLD)
    res_a, res_b = device_inference(out), reference()
    kept = sum(len(r["labels"]) for r in res_b)
    differ = sum(int((a.pred_masks != r["masks"]).sum()) for a, r in zip(res_a, res_b) if r["masks"] is not None)
    del res_a, res_b
    t_a = timed(lambda: device_inference(out), args.iters, args.warmup)
    t_b = timed(reference, args.iters, args.warmup)
    ns = types.SimpleNamespace
    cfg = ns(MODEL=ns(SPARSE_INST=ns(ENCODER=ns(NAME="InstanceContextEncoder", NUM_CHANNELS=256, IN_FEATURES=["res3", "res4", "res5"]),
                                     DECODER=ns(NAME="GroupIAMDecoder", SCALE_FACTOR=2.0, OUTPUT_IAM=False, NUM_MASKS=N, KERNEL_DIM=128, NUM_CLASSES=K,
                                                GROUPS=4, INST=ns(DIM=256, CONVS=4), MASK=ns(DIM=256, CONVS=4)))))
    enc = InstanceContextEncoder(cfg, {k: ns(channels=c) for k, c in zip(("res3", "res4", "res5"), (512, 1024, 2048))}, device=dev)
    dec = GroupIAMDecoder(cfg, device=dev)
    feats = {k: torch.randn(B, c, PAD[0] // s, PAD[1] // s, generator=g).to(dev) for k, c, s in zip(("res3", "res4", "res5"), (512, 1024, 2048),
                                                                                                   (8, 16, 32))}

    def full():
        with torch.no_grad():
            return device_inference(dec(enc(feats)))

    t_c = timed(full, max(1, args.iters // 2), args.warmup)
    fb, rb = floor_bytes(kept), reference_bytes(kept)
    res = {"bench": "sparseinst_infer", "gpu": name, "power_limit_and_max_sm_clock": power, "images": B, "queries": N, "kept": kept,
           "mask_pixels_differing_from_reference": differ, "device_inference_ms": round(t_a, 4), "reference_inference_ms": round(t_b, 4),
           "encoder_decoder_inference_ms": round(t_c, 4), "floor_bytes": fb, "floor_ms_at_datasheet_hbm": round(fb / HBM_BPS * 1e3, 4),
           "reference_chain_bytes": rb, "reference_chain_ms_at_datasheet_hbm": round(rb / HBM_BPS * 1e3, 4), "iters": args.iters}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
