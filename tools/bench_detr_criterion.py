"""DETR criterion and heads: the reference's algorithm in torch on the GPU (arm a) against this package (arm b).

Workload: B = 16 images, Q = 100 and 300 queries, L = 6 decoder layers (deep supervision), K1 = 81, G ~ U{1..20} targets per image, seeded.
  arm a: oracle/detr_criterion_oracle.py on the GPU, one cost matrix per layer copied to the host (`.cpu()`, one sync each) and solved with
         scipy, the losses in torch autograd; heads as fp32 nn.Linear / MLP in torch.
  arm b: SetCriterion / HungarianMatcher (one cost launch, one copy, one sync, two loss kernels); heads on the bf16 GEMM kernels.
Reports per arm and Q: criterion forward + backward and heads forward + backward, each as CUDA-event time and host wall time around
synchronised calls after warm-up; the device-to-host copies of one criterion call, counted from a torch.profiler trace in a separate run; and
the card name and power limit.  usage: python tools/bench_detr_criterion.py [--iters N] [--out results.json]
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
from oracle import detr_criterion_oracle as dco  # noqa: E402
from yolov7_d2_b200.detr import MLP, _Kernels, _linear_stack  # noqa: E402
from yolov7_d2_b200.detr_criterion import HungarianMatcher, SetCriterion  # noqa: E402

L, B, K1, D = 6, 16, 81, 256
COSTS, EOS = (1.0, 5.0, 2.0), 0.1
WEIGHTS = {"loss_ce": 1.0, "loss_bbox": 5.0, "loss_giou": 2.0}


def workload(q, dev, seed=0):
    g = torch.Generator().manual_seed(seed)
    logits = (torch.randn(L, B, q, K1, generator=g) * 2).to(dev)
    boxes = torch.sigmoid(torch.randn(L, B, q, 4, generator=g)).to(dev)
    targets = []
    for n in torch.randint(1, 21, (B,), generator=g).tolist():
        targets.append({"labels": torch.randint(0, K1 - 1, (n,), generator=g).to(dev),
                        "boxes": torch.cat([torch.rand(n, 2, generator=g) * 0.8 + 0.1, torch.rand(n, 2, generator=g) * 0.4 + 0.05], 1).to(dev)})
    hs = torch.randn(L, B, q, D, generator=g).to(dev)
    return logits, boxes, targets, hs


def weighted(losses):
    return sum(v * w for k, v in losses.items() for n, w in WEIGHTS.items() if k == n or k.startswith(n + "_"))


def reference_matcher(lg, bx, targets):
    """detr_utils.py:65-91: the full [B*Q, G] cost on the device, one .cpu() per layer, scipy per image"""
    from scipy.optimize import linear_sum_assignment

    bs, nq = lg.shape[:2]
    prob = lg.flatten(0, 1).softmax(-1)
    ob = bx.flatten(0, 1)
    ids = torch.cat([t["labels"] for t in targets])
    tb = torch.cat([t["boxes"] for t in targets])
    c = COSTS[1] * torch.cdist(ob, tb, p=1) + COSTS[0] * -prob[:, ids] + \
        COSTS[2] * -dco.generalized_box_iou(dco.box_cxcywh_to_xyxy(ob), dco.box_cxcywh_to_xyxy(tb))
    c = c.view(bs, nq, -1).cpu()
    sizes = [len(t["boxes"]) for t in targets]
    return [tuple(torch.as_tensor(a, dtype=torch.int64) for a in linear_sum_assignment(m[i])) for i, m in enumerate(c.split(sizes, -1))]


def crit_a(logits, boxes, targets):
    layers = [(logits[l].clone().requires_grad_(True), boxes[l].clone().requires_grad_(True)) for l in range(L)]
    indices = [reference_matcher(lg.detach(), bx.detach(), targets) for lg, bx in layers]
    nb = torch.clamp(torch.as_tensor([float(sum(len(t["labels"]) for t in targets))], device=logits.device), min=1).item()
    last = L - 1
    losses = dict(dco.set_losses(*layers[last], targets, indices[last], K1 - 1, EOS, nb))
    for i in range(last):
        losses.update({k + f"_{i}": v for k, v in dco.set_losses(*layers[i], targets, indices[i], K1 - 1, EOS, nb, log=False).items()})
    weighted(losses).backward()


def crit_b(crit, logits, boxes, targets):
    layers = [(logits[l].clone().requires_grad_(True), boxes[l].clone().requires_grad_(True)) for l in range(L)]
    out = {"pred_logits": layers[-1][0], "pred_boxes": layers[-1][1], "aux_outputs": [{"pred_logits": a, "pred_boxes": b} for a, b in layers[:-1]]}
    weighted(crit(out, targets)).backward()


def heads_a(mods, hs):
    cls, mlp = mods
    x = hs.clone().requires_grad_(True)
    lg = F.linear(x, cls.weight, cls.bias)
    h = x
    for i, lin in enumerate(mlp):
        h = F.linear(h, lin.weight, lin.bias)
        h = F.relu(h) if i < 2 else h
    (lg.square().mean() + torch.sigmoid(h).mean()).backward()


def heads_b(mods, hs):
    cls, mlp, kn = mods
    x = hs.clone().requires_grad_(True)
    lg = _linear_stack(kn, x, [cls])
    (lg.square().mean() + torch.sigmoid(mlp(x)).mean()).backward()


def timed(fn, iters, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0 = time.perf_counter()
    ev0.record()
    for _ in range(iters):
        fn()
    ev1.record()
    torch.cuda.synchronize()
    wall = (time.perf_counter() - t0) / iters * 1e3
    return {"event_ms": ev0.elapsed_time(ev1) / iters, "wall_ms": wall}


def count_d2h(fn):
    from torch.profiler import ProfilerActivity, profile

    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if "Memcpy DtoH" in e.name)


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_detr_criterion needs a CUDA device")
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    cls = torch.nn.Linear(D, K1).to(dev)
    mlp = MLP(D, D, 4, 3).to(dev)
    crit = SetCriterion(K1 - 1, HungarianMatcher(*COSTS), WEIGHTS, EOS, ["labels", "boxes", "cardinality"])
    res = {"card": card(), "L": L, "B": B, "K1": K1, "results": {}}
    for q in (100, 300):
        logits, boxes, targets, hs = workload(q, dev)
        r = {
            "criterion_a": timed(lambda: crit_a(logits, boxes, targets), args.iters),
            "criterion_b": timed(lambda: crit_b(crit, logits, boxes, targets), args.iters),
            "heads_a": timed(lambda: heads_a((cls, mlp.layers), hs), args.iters),
            "heads_b": timed(lambda: heads_b((cls, mlp, _Kernels()), hs), args.iters),
            "d2h_copies_a": count_d2h(lambda: crit_a(logits, boxes, targets)),
            "d2h_copies_b": count_d2h(lambda: crit_b(crit, logits, boxes, targets)),
            "targets": int(sum(len(t["labels"]) for t in targets)),
        }
        res["results"][f"Q{q}"] = r
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
