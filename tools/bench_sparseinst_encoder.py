"""SparseInst InstanceContextEncoder on one GPU: this package's kernels against the reference's arithmetic in torch on the same GPU.

Workload (seeded): 16 images at 640 x 640 through a ResNet-50's shapes: res3 [16, 512, 80, 80], res4 [16, 1024, 40, 40], res5 [16, 2048, 20, 20],
fp32 NCHW, NUM_CHANNELS 256.
  (a) encoder forward;
  (b) encoder forward + backward (seeded upstream gradient), including d res3 / res4 / res5;
  (c) encoder + GroupIAMDecoder + SparseInstCriterion forward + backward (1-20 random ellipses per image);
  (d) the reference's arithmetic: oracle/sparseinst_encoder_oracle.py under bf16 autocast, channels_last, forward + backward of (b).
Times are CUDA events over --iters repetitions after --warmup.  Also printed: the card name and power limit read in the same run, and floors
computed from the shapes (not measurements): the GEMM FLOPs of the forward and of a training step (forward, data and weight gradients) at the
data sheet's dense BF16 rate, and the fp32 input bytes at the data sheet's HBM bandwidth.
usage: python tools/bench_sparseinst_encoder.py [--iters N] [--warmup N] [--out results.json]
"""
import argparse
import json
import os
import subprocess
import sys
import types

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import sparseinst_encoder_oracle as seo  # noqa: E402
from yolov7_d2_b200.sparseinst_encoder import InstanceContextEncoder  # noqa: E402

B, C, SIZE = 16, 256, 640
IN_CH = (512, 1024, 2048)
BF16_FLOPS = 989e12  # H100 SXM dense BF16, data sheet (700 W)
HBM_BPS = 3.35e12    # H100 SXM HBM3, data sheet


def ns(**kw):
    return types.SimpleNamespace(**kw)


def maps():
    return [(SIZE // s, SIZE // s) for s in (8, 16, 32)]  # res3, res4, res5


def forward_macs_per_image():
    """multiply-accumulates of the encoder's convolutions for one image"""
    (h3, w3), (h4, w4), (h5, w5) = maps()
    p3, p4, p5 = h3 * w3, h4 * w4, h5 * w5
    pooled = sum((h5 // kh) * (w5 // kw) for kh, kw in seo.ppm_windows(h5, w5))
    return (p5 * IN_CH[2] * C + p4 * IN_CH[1] * C + p3 * IN_CH[0] * C     # laterals
            + pooled * C * (C // 4) + p5 * 2 * C * C                        # PPM stages, bottleneck
            + (p5 + p4 + p3) * 9 * C * C                                    # output convolutions
            + p3 * 3 * C * C)                                               # fusion


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
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_sparseinst_encoder: no GPU (this benchmark does not fall back to the CPU)")
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(0)
    cfg = ns(MODEL=ns(SPARSE_INST=ns(ENCODER=ns(NAME="InstanceContextEncoder", NUM_CHANNELS=C, IN_FEATURES=list(seo.IN_FEATURES)))))
    enc = InstanceContextEncoder(cfg, {k: ns(channels=c) for k, c in zip(seo.IN_FEATURES, IN_CH)}, device=dev)
    sd = seo.encoder_state_dict(1, IN_CH, C)
    enc.load_state_dict({k: v.to(dev) for k, v in sd.items()}, strict=True)
    feats = {k: torch.randn(B, c, h, w, generator=g).to(dev).requires_grad_(True) for k, c, (h, w) in zip(seo.IN_FEATURES, IN_CH, maps())}
    h3, w3 = maps()[0]
    up = torch.randn(B, C, h3, w3, generator=g).to(dev)
    res = {}

    def fwd():
        with torch.no_grad():
            enc(feats)

    def fwd_bwd():
        for v in feats.values():
            v.grad = None
        enc(feats).backward(up)

    res["a_encoder_fwd_ms"] = timed(fwd, args.iters, args.warmup)
    res["b_encoder_fwd_bwd_ms"] = timed(fwd_bwd, args.iters, args.warmup)

    # (c) encoder + GroupIAMDecoder + SparseInstCriterion
    from bench_sparseinst_train import criterion, decoder, targets

    import bench_sparseinst_train as bst

    bst.IN = SIZE
    dec, _ = decoder("Group", dev)
    crit = criterion()
    tg = targets(dev, g)

    def step():
        for v in feats.values():
            v.grad = None
        losses = crit(dec(enc(feats)), tg, (SIZE, SIZE))
        sum(losses.values()).backward()

    res["c_encoder_decoder_criterion_fwd_bwd_ms"] = timed(step, max(1, args.iters // 2), max(1, args.warmup // 2))
    del dec

    # (d) the reference's arithmetic in torch: bf16 autocast, channels_last
    fl = {k: v.detach().contiguous(memory_format=torch.channels_last).requires_grad_(True) for k, v in feats.items()}
    sdt = {k: v.to(dev).contiguous(memory_format=torch.channels_last if v.dim() == 4 else torch.contiguous_format).requires_grad_(True)
           for k, v in sd.items()}

    def torch_step():
        for v in list(fl.values()) + list(sdt.values()):
            v.grad = None
        with torch.autocast("cuda", dtype=torch.bfloat16):
            out = seo.encoder_forward(fl, sdt)
        out.float().backward(up)

    res["d_torch_reference_fwd_bwd_ms"] = timed(torch_step, args.iters, args.warmup)
    name, power = card()
    macs = forward_macs_per_image() * B
    fwd_flop, step_flop = 2 * macs, 6 * macs
    in_bytes = sum(B * c * h * w * 4 for c, (h, w) in zip(IN_CH, maps()))
    out = dict(card=name, power_limit_and_max_sm_clock=power, batch=B, size=SIZE, **{k: round(v, 3) for k, v in res.items()},
               floor_fwd_gflop=round(fwd_flop / 1e9, 1), floor_fwd_ms_at_bf16_peak=round(fwd_flop / BF16_FLOPS * 1e3, 3),
               floor_step_gflop=round(step_flop / 1e9, 1), floor_step_ms_at_bf16_peak=round(step_flop / BF16_FLOPS * 1e3, 3),
               floor_input_mb=round(in_bytes / 1e6, 1), floor_input_read_ms_at_hbm_peak=round(in_bytes / HBM_BPS * 1e3, 3))
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    main()
