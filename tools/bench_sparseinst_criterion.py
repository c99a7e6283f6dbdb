"""SparseInst matcher + criterion at the shipped shape: this package's kernels against the reference's arithmetic in torch on the same GPU.

Workload (seeded): B = 16 images, N = 100 queries, K = 80 classes, 160 x 160 mask logits from a 640 x 640 input, G ~ U{1..20} random filled
ellipses per image on images of 400-640 pixels a side.
  (a) the four entry points alone (target masks, matching cost, losses, gradients), launched back to back;
  (b) SparseInstCriterion forward + backward, including the cost copy, the synchronisation and scipy;
  (c) the reference's algorithm as plain torch ops on the GPU (oracle/sparseinst_criterion_oracle.py's functions plus the reference matcher's
      full [B*N, G] cost and its .cpu()): pad + interpolate twice, the full dice matrix, the losses through autograd.
Times are CUDA events over --iters repetitions after warm-up (host wall time too for (b) and (c), which synchronise).  Also printed: the card
name and power limit read in the same run, and the algorithmic bytes and their time at the data sheet's 3.35 TB/s (a floor, not a measurement).
usage: python tools/bench_sparseinst_criterion.py [--iters N] [--out results.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import sparseinst_criterion_oracle as sco  # noqa: E402
from yolov7_d2_b200 import capi  # noqa: E402
from yolov7_d2_b200.sparseinst_criterion import SparseInstCriterion, SparseInstMatcher, _Targets  # noqa: E402

B, N, K, S, IN = 16, 100, 80, 160, 640
ALPHA, BETA = 0.8, 0.2
WEIGHTS = (2.0, 5.0, 2.0, 1.0)  # CLASS, MASK_PIXEL, MASK_DICE, OBJECTNESS
WEIGHT_DICT = dict(zip(("loss_ce", "loss_mask", "loss_dice", "loss_objectness"), WEIGHTS))
HBM_BYTES_PER_S = 3.35e12


def _cfg():
    ns = __import__("types").SimpleNamespace
    return ns(MODEL=ns(SPARSE_INST=ns(LOSS=ns(NAME="SparseInstCriterion", ITEMS=("labels", "masks"), CLASS_WEIGHT=WEIGHTS[0], MASK_PIXEL_WEIGHT=WEIGHTS[1],
                                              MASK_DICE_WEIGHT=WEIGHTS[2], OBJECTNESS_WEIGHT=WEIGHTS[3]),
                                      MATCHER=ns(NAME="SparseInstMatcher", ALPHA=ALPHA, BETA=BETA), DECODER=ns(NUM_CLASSES=K))))


def workload(dev, seed=0):
    g = torch.Generator().manual_seed(seed)
    sizes = torch.randint(1, 21, (B,), generator=g).tolist()
    targets = []
    for n in sizes:
        h, w = (int(v) for v in torch.randint(400, IN + 1, (2,), generator=g))
        yy, xx = torch.meshgrid(torch.arange(h, dtype=torch.float32), torch.arange(w, dtype=torch.float32), indexing="ij")
        c = torch.rand(n, 4, generator=g)
        m = ((yy - c[:, 0, None, None] * h) / (8 + c[:, 2, None, None] * h / 4)) ** 2 + ((xx - c[:, 1, None, None] * w) / (8 + c[:, 3, None, None] * w / 4)) ** 2 <= 1
        targets.append({"labels": torch.randint(0, K, (n,), generator=g).to(dev), "masks": sco.BitMasks(m.to(dev))})
    outputs = {"pred_logits": (torch.randn(B, N, K, generator=g) * 2 - 2).to(dev).requires_grad_(True),
               "pred_masks": (torch.randn(B, N, S, S, generator=g) * 2.5).to(dev).requires_grad_(True),
               "pred_scores": torch.randn(B, N, 1, generator=g).to(dev).requires_grad_(True)}
    return outputs, targets, sizes


def reference_step(outputs, targets):
    """sparseinst_loss.py's arithmetic in torch: the matcher's full cost matrix and .cpu(), then the losses (a second interpolation)"""
    lg, mk, sc = outputs["pred_logits"], outputs["pred_masks"], outputs["pred_scores"]
    mask_list = [t["masks"].tensor for t in targets]
    labels = torch.cat([t["labels"] for t in targets])
    sizes = [len(t["masks"]) for t in targets]
    with torch.no_grad():
        tm = sco.target_masks(mask_list, (IN, IN), (S, S), mk.dtype)
        s = mk.detach().view(B * N, -1).sigmoid()
        t = tm.flatten(1)
        dice = 2 * (s @ t.T) / ((s * s).sum(-1)[:, None] + (t * t).sum(-1) + 1e-4)
        C = (dice ** ALPHA * lg.detach().sigmoid().view(B * N, -1)[:, labels] ** BETA).view(B, N, -1).cpu()
        blocks = [c[i] for i, c in enumerate(C.split(sizes, -1))]
    indices = sco.assign(blocks)
    num = torch.clamp(torch.as_tensor([float(sum(sizes))], device=lg.device), min=1).item()
    tm2 = sco.target_masks(mask_list, (IN, IN), (S, S), mk.dtype)
    losses = sco.losses(lg, mk, sc, tm2, sizes, labels, indices, WEIGHT_DICT, num)
    sum(losses.values()).backward()


def package_step(crit, outputs, targets):
    losses = crit(outputs, targets, (IN, IN))
    sum(losses.values()).backward()


def time_events(fn, iters, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0 = time.perf_counter()
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    wall = (time.perf_counter() - t0) / iters * 1e3
    return a.elapsed_time(b) / iters, wall


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()[0]
        return q
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark measures the GPU only")
    dev = torch.device("cuda")
    outputs, targets, sizes = workload(dev)
    G = sum(sizes)
    crit = SparseInstCriterion(_cfg(), SparseInstMatcher(_cfg()))

    # (a) the four entry points alone, on the operands of one criterion call
    logits, masks = outputs["pred_logits"].detach(), outputs["pred_masks"].detach()
    scores = outputs["pred_scores"].detach().reshape(B, N).contiguous()
    tg = _Targets(targets, (IN, IN), masks.shape, dev, "bench")
    _, match_host = crit.matcher.match(logits, masks, tg)
    match = match_host.to(dev)
    packed = torch.cat([t["masks"].tensor.view(torch.uint8).reshape(-1) for t in targets])
    table, off = [], 0
    for t in targets:
        g, h, w = t["masks"].tensor.shape
        table += [(off + j * h * w, h, w) for j in range(g)]
        off += g * h * w
    table = torch.tensor(table, dtype=torch.int64, device=dev)
    cost = torch.empty(N * G + 1, device=dev)
    out, save, grad = torch.empty(4, device=dev), torch.empty(B, N, 8, device=dev), torch.ones(4, device=dev)
    dl, dm, ds = torch.empty_like(logits), torch.empty_like(masks), torch.empty_like(scores)
    w4 = (WEIGHTS[0], WEIGHTS[3], WEIGHTS[2], WEIGHTS[1])  # (ce, objectness, dice, mask): the kernels' order

    def kernels():
        capi.sparseinst_target_masks(packed, table, G, (IN, IN), (S, S), tg.masks, tg.tsq)
        capi.sparseinst_match_cost(logits, masks, tg.labels, tg.offsets, tg.masks, tg.tsq, G, ALPHA, BETA, cost)
        capi.sparseinst_set_loss(logits, masks, scores, match, tg.labels, tg.offsets, tg.masks, tg.tsq, G, w4, float(G), save, out)
        capi.sparseinst_set_loss_bwd(logits, masks, scores, match, tg.labels, tg.offsets, tg.masks, tg.tsq, save, G, w4, float(G), grad, dl, dm, ds)

    per_kernel = {}
    for name, fn in (("target_masks", lambda: capi.sparseinst_target_masks(packed, table, G, (IN, IN), (S, S), tg.masks, tg.tsq)),
                     ("match_cost", lambda: capi.sparseinst_match_cost(logits, masks, tg.labels, tg.offsets, tg.masks, tg.tsq, G, ALPHA, BETA, cost)),
                     ("set_loss", lambda: capi.sparseinst_set_loss(logits, masks, scores, match, tg.labels, tg.offsets, tg.masks, tg.tsq, G, w4, float(G),
                                                                   save, out)),
                     ("set_loss_bwd", lambda: capi.sparseinst_set_loss_bwd(logits, masks, scores, match, tg.labels, tg.offsets, tg.masks, tg.tsq, save,
                                                                           G, w4, float(G), grad, dl, dm, ds))):
        per_kernel[name] = round(time_events(fn, args.iters * 4)[0], 4)
    a_ms, _ = time_events(kernels, args.iters * 4)

    def zero_grads():
        for v in outputs.values():
            v.grad = None

    b_ms, b_wall = time_events(lambda: (zero_grads(), package_step(crit, outputs, targets)), args.iters)
    c_ms, c_wall = time_events(lambda: (zero_grads(), reference_step(outputs, targets)), max(3, args.iters // 5))

    HW = S * S
    gt_bytes = sum(t["masks"].tensor.numel() for t in targets)
    algo = {"mask_logits_read_once": B * N * HW * 4, "gt_masks_uint8": gt_bytes, "matched_rows_fwd_bwd": 2 * 2 * G * HW * 4,
            "d_pred_masks_written": B * N * HW * 4}
    total = sum(algo.values())
    res = {"card": card(), "workload": {"B": B, "N": N, "K": K, "mask": [S, S], "input": [IN, IN], "G": G},
           "a_kernels_ms": round(a_ms, 4), "a_per_kernel_ms": per_kernel,
           "b_criterion_fwd_bwd_ms": round(b_ms, 3), "b_wall_ms": round(b_wall, 3),
           "c_reference_torch_fwd_bwd_ms": round(c_ms, 3), "c_wall_ms": round(c_wall, 3),
           "algorithmic_bytes": algo, "algorithmic_total_MB": round(total / 1e6, 1),
           "floor_ms_at_3.35TBps": round(total / HBM_BYTES_PER_S * 1e3, 4), "a_over_floor": round(a_ms / (total / HBM_BYTES_PER_S * 1e3), 2)}
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
