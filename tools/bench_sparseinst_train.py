"""SparseInst decoder training step on one GPU: this package's kernels against the reference's arithmetic in torch on the same GPU.

Workload (seeded): 16 images of 256 encoder channels at 80 x 80 (258 decoder input channels with the coordinates; the per-GPU share of
BASELINE.json configs[4]), 100 masks, dim 256, kernel dim 128, 80 classes, Base (BaseIAMDecoder) and Group (GroupIAMDecoder, 4 groups).
  (a) decoder forward + backward (seeded upstream gradients of the three outputs);
  (b) decoder + SparseInstCriterion forward + backward (1-20 random ellipses per image on a 320 x 320 input);
  (c) the reference's arithmetic: oracle/sparseinst_oracle.py under bf16 autocast, channels_last, forward + backward of (a).
Times are CUDA events over --iters repetitions after --warmup.  Also printed: the card name and power limit read in the same run, the algorithmic
FLOPs of the backward convolutions (dgrad + wgrad of the eight 3x3 layers: 2 x 7.55 GFLOP each per image, ~121 GFLOP per image) and of the whole
step, and their time at the data sheet's dense BF16 rate (a floor, not a measurement).
usage: python tools/bench_sparseinst_train.py [--iters N] [--warmup N] [--out results.json]
"""
import argparse
import json
import os
import subprocess
import sys
import types

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import sparseinst_criterion_oracle as sco  # noqa: E402
from oracle import sparseinst_oracle as sio  # noqa: E402
from yolov7_d2_b200.sparseinst import BaseIAMDecoder, GroupIAMDecoder  # noqa: E402
from yolov7_d2_b200.sparseinst_criterion import build_sparse_inst_criterion  # noqa: E402

B, C, H, W, NM, DIM, KD, NC, CONVS, IN = 16, 256, 80, 80, 100, 256, 128, 80, 4, 320
BF16_FLOPS = 989e12  # H100 SXM dense BF16, data sheet (700 W)


def ns(**kw):
    return types.SimpleNamespace(**kw)


def decoder(kind, dev):
    cfg = ns(MODEL=ns(SPARSE_INST=ns(ENCODER=ns(NUM_CHANNELS=C), DECODER=ns(SCALE_FACTOR=2.0, OUTPUT_IAM=False, NUM_MASKS=NM, KERNEL_DIM=KD, NUM_CLASSES=NC,
                                                                          GROUPS=4, INST=ns(DIM=DIM, CONVS=CONVS), MASK=ns(DIM=DIM, CONVS=CONVS)))))
    dec = (GroupIAMDecoder if kind == "Group" else BaseIAMDecoder)(cfg, device=dev)
    sd = sio.decoder_state_dict(1, groups=4 if kind == "Group" else 0)
    dec.load_state_dict({k: v.to(dev) for k, v in sd.items()}, strict=True)
    return dec, sd


def criterion():
    return build_sparse_inst_criterion(ns(MODEL=ns(SPARSE_INST=ns(
        LOSS=ns(NAME="SparseInstCriterion", ITEMS=("labels", "masks"), CLASS_WEIGHT=2.0, MASK_PIXEL_WEIGHT=5.0, MASK_DICE_WEIGHT=2.0, OBJECTNESS_WEIGHT=1.0),
        MATCHER=ns(NAME="SparseInstMatcher", ALPHA=0.8, BETA=0.2), DECODER=ns(NUM_CLASSES=NC)))))


def targets(dev, g):
    out = []
    yy, xx = torch.meshgrid(torch.arange(IN, dtype=torch.float32), torch.arange(IN, dtype=torch.float32), indexing="ij")
    for _ in range(B):
        n = int(torch.randint(1, 21, (1,), generator=g))
        c = torch.rand(n, 4, generator=g)
        m = ((yy - c[:, 0, None, None] * IN) / (8 + c[:, 2, None, None] * IN / 4)) ** 2 + ((xx - c[:, 1, None, None] * IN) / (8 + c[:, 3, None, None] * IN / 4)) ** 2 <= 1
        out.append({"labels": torch.randint(0, NC, (n,), generator=g).to(dev), "masks": sco.BitMasks(m.to(dev))})
    return out


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


def flops(kind):
    """multiply-adds x 2 of every GEMM of one training step (forward, data and weight gradients), per image; and the backward 3x3 convolutions"""
    px = H * W
    conv3 = 2 * px * 9 * DIM * DIM                            # one 3x3 256 -> 256 layer (the first reads 258 channels)
    first = 2 * px * 9 * (C + 2) * DIM
    layers = 2 * (first + 3 * conv3)                          # both branches
    iam = 2 * px * 9 * DIM * NM                               # grouped: G groups of dim / G inputs x N maps, the same count
    agg = 2 * px * DIM * NM * (4 if kind == "Group" else 1)
    proj, bmm = 2 * px * DIM * KD, 2 * px * KD * NM
    fwd = layers + iam + agg + proj + bmm
    bwd_conv3 = 2 * (2 * first + 6 * conv3)                   # dgrad + wgrad of the eight 3x3 layers
    return fwd * 3, bwd_conv3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_sparseinst_train.py needs a GPU (no CPU timing is reported)")
    dev = torch.device("cuda:0")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    g = torch.Generator().manual_seed(0)
    feat = torch.randn(B, C, H, W, generator=g).to(dev)
    ups = [torch.randn(B, NM, NC, generator=g).to(dev), (torch.randn(B, NM, 2 * H, 2 * W, generator=g) * 0.1).to(dev), torch.randn(B, NM, 1, generator=g).to(dev)]
    tg = targets(dev, g)
    crit = criterion()
    res = {"card": q, "workload": f"{B}x{C + 2}x{H}x{W}, {NM} masks"}
    for kind in ("Base", "Group"):
        dec, sd = decoder(kind, dev)
        fin = feat.clone().requires_grad_(True)

        def dec_step():
            out = dec(fin)
            torch.autograd.backward([out["pred_logits"], out["pred_masks"], out["pred_scores"]], ups)

        def crit_step():
            out = dec(fin)
            losses = crit(out, tg, (IN, IN))
            sum(losses.values()).backward()

        sdd = {k: v.to(dev).requires_grad_(True) for k, v in sd.items()}
        fcl = feat.contiguous(memory_format=torch.channels_last).requires_grad_(True)

        def ref_step():
            with torch.autocast("cuda", dtype=torch.bfloat16):
                out = sio.decoder_forward(fcl, sdd, groups=4 if kind == "Group" else 0)
            torch.autograd.backward([out["pred_logits"].float(), out["pred_masks"].float(), out["pred_scores"].float()], ups)

        t_dec = timed(dec_step, args.iters, args.warmup)
        t_crit = timed(crit_step, args.iters, args.warmup)
        t_ref = timed(ref_step, args.iters, args.warmup)
        step, bwd3 = flops(kind)
        res[kind] = {"decoder_fwd_bwd_ms": round(t_dec, 3), "decoder_criterion_fwd_bwd_ms": round(t_crit, 3), "reference_torch_bf16_fwd_bwd_ms": round(t_ref, 3),
                     "step_gflop": round(B * step / 1e9, 1), "bwd_conv3x3_gflop_per_image": round(bwd3 / 1e9, 1),
                     "floor_ms_at_989_tflops": round(B * step / BF16_FLOPS * 1e3, 3), "decoder_tflops": round(B * step / t_dec / 1e9, 1)}
        del dec, sdd
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
