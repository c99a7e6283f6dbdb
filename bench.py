#!/usr/bin/env python
"""Headline benchmark: YOLOX-s 640x640 forward+backward images/s on N H100s (BASELINE.json metric), one JSON line.

    python bench.py --gpus N --steps K --warmup W            # this repo (libyb200.so kernels)
    python bench.py --impl reference --gpus N --steps K ...  # the reference's CPU path (oracle port) on the host cores
    python bench.py ... --dump-outputs DIR                    # also write what the last timed step computed, DIR/<name>.npy

A "step" = one pass of the hot path over one synthetic COCO-shaped batch per GPU: uint8->Focus preprocessing, CSPDarknet,
YOLOPAFPN, YOLOX head, SimOTA assignment, IoU/BCE losses and the full backward (data + weight + BN gradients); for N > 1
followed by ONE NCCL all-reduce of the flat gradient buffer.  No optimizer step (the metric is fwd+bwd).
`value`  : inputs resident in HBM, engine called directly, CUDA-event time, max over ranks.
`e2e`    : the public API a detectron2 trainer calls -- YOLOX.forward(batched_inputs) on pinned HOST uint8 images +
           sum(losses).backward() + loss.item() -- with the H2D / D2H copies inside the timed region.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import threading
import time
import types

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

METRIC = "images/sec (640x640) YOLOX-s fwd+bwd"
WORKLOAD = "YOLOX-s 640x640 bs=64 per GPU, fwd+bwd, synthetic COCO-shaped input (BASELINE.json configs[1])"
FLOP_PER_IMAGE = 79.35e9  # SURVEY.md par.8d: 26.69 fwd + 52.66 bwd GFLOP


def peaks():
    """roofline denominators: MEASURED_PEAKS.json when present, else NVIDIA's H100 SXM data sheet (3.35 TB/s HBM3, 989 TFLOP/s dense bf16 at
    700 W) -- a ceiling, not a rate this code has been measured to reach"""
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        with open(p) as fh:
            d = json.load(fh)
        return dict(hbm=d.get("hbm_gbs", 3350.0), tf_burst=d.get("bf16_tflops", 989.0), tf_sust=d.get("bf16_tflops_sustained", 989.0),
                    source="measured")
    return dict(hbm=3350.0, tf_burst=989.0, tf_sust=989.0, source="H100 SXM data sheet")


class ClockSampler:
    """nvidia-smi clocks / throttle reasons sampled DURING the timed region"""

    Q = ("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
         "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, index):
        self.rows, self.proc = [], None
        try:
            self.proc = subprocess.Popen(["nvidia-smi", f"--id={index}", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits", "-lms", "50"],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.t = threading.Thread(target=self._read, daemon=True)
            self.t.start()
        except Exception:  # noqa: BLE001
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append([c.strip() for c in line.split(",")])

    def stop(self):
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        self.proc.terminate()
        sm = [float(r[0]) for r in self.rows if len(r) >= 7 and r[0].replace(".", "").isdigit()]
        mx = [float(r[1]) for r in self.rows if len(r) >= 7 and r[1].replace(".", "").isdigit()]
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        reasons = sorted({names[i] for r in self.rows if len(r) >= 7 for i in range(4) if r[3 + i].lower().startswith("active")})
        return {"sm_mhz": statistics.median(sm) if sm else None, "sm_max_mhz": max(mx) if mx else None, "reasons": reasons,
                "samples": len(sm)}


# the optimizer step is part of the timed step; a tiny learning rate keeps 1000s of steps on one synthetic batch from diverging
BENCH_LR = 1e-5


def ns(**kw):
    return types.SimpleNamespace(**kw)


def yolox_s_cfg(device="cuda"):
    """the attributes YOLOX.__init__ reads from configs/coco/yolox_s.yaml + yolov7/config.py defaults (yolox.py:38-58)"""
    return ns(MODEL=ns(DEVICE=device, NMS_TYPE="normal", PADDED_VALUE=114.0, PIXEL_MEAN=[0.485, 0.456, 0.406], PIXEL_STD=[0.229, 0.224, 0.225],
                       BACKBONE=ns(NAME="build_cspdarknetx_backbone"), DARKNET=ns(DEPTH_WISE=False, OUT_FEATURES=["dark3", "dark4", "dark5"]),
                       YOLO=ns(CLASSES=80, CONF_THRESHOLD=0.001, NMS_THRESHOLD=0.65, WIDTH_MUL=0.50, DEPTH_MUL=0.33, LOSS_TYPE="v7",
                               MAX_BOXES_NUM=100, IN_FEATURES=["dark3", "dark4", "dark5"])),
              SOLVER=ns(MAX_ITER=230000, OPTIMIZER="SGD", BASE_LR=BENCH_LR, MOMENTUM=0.9, NESTEROV=False, WEIGHT_DECAY=5e-4, WEIGHT_DECAY_NORM=0.0),
              INPUT=ns(MOSAIC_AND_MIXUP=ns(DISABLE_AT_ITER=120000)))


class _GtBoxes:
    def __init__(self, t):
        self.tensor = t


def batched_inputs_from(images_u8, labels):
    """list[dict] in detectron2's format: uint8 CHW host image + Instances-like (gt_boxes XYXY, gt_classes)"""
    out = []
    for b in range(images_u8.shape[0]):
        lab = labels[b]
        lab = lab[lab.sum(1) > 0]
        xyxy = __import__("torch").stack([lab[:, 1] - lab[:, 3] / 2, lab[:, 2] - lab[:, 4] / 2, lab[:, 1] + lab[:, 3] / 2, lab[:, 2] + lab[:, 4] / 2], 1)
        out.append({"image": images_u8[b], "instances": ns(gt_boxes=_GtBoxes(xyxy), gt_classes=lab[:, 0].long()), "height": 640, "width": 640})
    return out


def pick_cpu_threads(step_fn, torch, candidates=(8, 16, 32, 64, 128, 256)):
    """The oracle is torch CPU fp32: more threads than physical cores (or than the cgroup grants) make it slower, not
    faster.  Try a few thread counts for one step each and keep the fastest -- 'all the host threads it can use'."""
    avail = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)
    best_t, best_n = None, 1
    for n in [c for c in candidates if c <= avail] or [avail]:
        torch.set_num_threads(n)
        t0 = time.perf_counter()
        step_fn()
        dt = time.perf_counter() - t0
        if best_t is None or dt < best_t:
            best_t, best_n = dt, n
        if dt > 60:  # do not keep climbing when a step already takes a minute
            break
    torch.set_num_threads(best_n)
    return best_n, avail


def run_reference(args, rank, world):
    """the reference's own CPU implementation of the path (oracle port: plain torch fp32, all host threads)"""
    import torch
    from oracle import yolox_oracle as orc

    if rank != 0:
        return
    bs = args.ref_batch
    sd = orc.yolox_state_dict(0)
    for k, v in sd.items():
        if v.dtype == torch.float32 and "running" not in k:
            v.requires_grad_(True)
    images, labels = orc.synthetic_batch(bs, 640, 0)
    x = images.float()

    ropt = None if args.no_optimizer else torch.optim.SGD([v for v in sd.values() if v.requires_grad], lr=BENCH_LR, momentum=0.9, weight_decay=5e-4)

    def step():
        for v in sd.values():
            if v.requires_grad and v.grad is not None:
                v.grad = None
        out = orc.yolox_forward_train(x, labels, sd)
        out[0].backward()
        if ropt is not None:
            ropt.step()
        return float(out[0])

    threads, avail = pick_cpu_threads(step, torch)  # doubles as the warm-up
    t0 = time.perf_counter()
    for _ in range(args.steps):
        step()
    dt = time.perf_counter() - t0
    val = bs * args.steps / dt
    line = {"metric": METRIC, "value": val, "unit": "images/s", "impl": "reference", "n_gpus": args.gpus, "steps": args.steps, "warmup": args.warmup,
            "ms_per_step": 1e3 * dt / args.steps, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f32",
            "data": "synthetic", "config": {"workload": WORKLOAD, "sample": f"bs={bs} per step on the host CPU"},
            "cpu_baseline": {"value": val, "unit": "images/s", "cores": threads, "cores_available": avail, "kind": "port",
                             "sample": f"{args.steps} steps of bs={bs} YOLOX-s 640x640 fwd+bwd (oracle/yolox_oracle.py, torch CPU fp32)"},
            "e2e": {"value": val, "unit": "images/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}
    print(json.dumps(line), flush=True)


def library_bar(torch, dev, batch, with_optimizer, steps=5, warmup=3):
    """Stock PyTorch on the same GPU: the oracle port (plain torch ops: F.conv2d / F.batch_norm / SiLU -> cuDNN, cuBLAS, ATen kernels)
    under autocast(fp16) with channels_last tensors, the same synthetic batch, forward + SimOTA + losses + backward (+ torch.optim.SGD).
    A reported baseline, like cpu_baseline: nothing of this repo's kernels runs here, and this repo's path never calls it."""
    from oracle import yolox_oracle as orc  # baseline being timed (not the product path)
    torch.backends.cudnn.benchmark = True
    sd = {k: v.to(dev) for k, v in orc.yolox_state_dict(0).items()}
    for k, v in sd.items():
        if v.dtype == torch.float32 and "running" not in k:
            if v.dim() == 4:
                sd[k] = v = v.contiguous(memory_format=torch.channels_last)
            v.requires_grad_(True)
    images, labels = orc.synthetic_batch(batch, 640, 100)
    x = images.to(dev).float().contiguous(memory_format=torch.channels_last)
    labels = labels.to(dev)
    params = [v for v in sd.values() if v.requires_grad]
    sgd = torch.optim.SGD(params, lr=BENCH_LR, momentum=0.9, weight_decay=5e-4) if with_optimizer else None

    def step():
        for v in params:
            v.grad = None
        with torch.autocast("cuda", dtype=torch.float16):
            raw = orc.head_raw(orc.pafpn(orc.csp_darknet(x, sd, True), sd, True), sd, True)
        outputs = orc.decode_train([r.float() for r in raw])
        xs, ys, ss = orc.anchor_grid([o.shape[-2:] for o in raw], device=dev)
        loss = orc.yolox_losses(outputs, labels, xs, ys, ss)[0]
        loss.backward()
        if sgd is not None:
            sgd.step()
        return loss

    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        loss = step()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    # network only (no SimOTA / loss Python loop): forward + backward of a scalar functional of the head outputs
    def net_step():
        for v in params:
            v.grad = None
        with torch.autocast("cuda", dtype=torch.float16):
            raw = orc.head_raw(orc.pafpn(orc.csp_darknet(x, sd, True), sd, True), sd, True)
        sum(r.float().square().mean() for r in raw).backward()

    for _ in range(2):
        net_step()
    torch.cuda.synchronize()
    e0.record()
    for _ in range(steps):
        net_step()
    e1.record()
    torch.cuda.synchronize()
    ms_net = e0.elapsed_time(e1) / steps
    out = {"value": batch / ms * 1e3, "unit": "images/s", "ms_per_step": ms, "network_only_images_per_s": batch / ms_net * 1e3, "network_only_ms": ms_net,
           "what": "oracle port (plain torch ops) on cuda:0, torch %s / cuDNN %s, autocast fp16 + channels_last, bs=%d 640x640, fwd + SimOTA/loss (per-image "
                   "Python loop, as the reference) + bwd%s; network_only = conv/BN/SiLU forward+backward without the loss" % (
                       torch.__version__, torch.backends.cudnn.version(), batch, " + torch.optim.SGD" if with_optimizer else ""),
           "loss": float(loss)}
    del sd, params, x
    torch.cuda.empty_cache()
    return out


def yolox_convnext_step(torch, dist, dev, rank, world, batch, steps, warmup, with_optimizer, use_graph):
    """BASELINE.json configs[2]: YOLOX on a ConvNeXt-T backbone (corrected wiring, yolov7_d2_b200/yolox_convnext.py), `batch` images of 640x640 per
    GPU: forward, SimOTA + losses, backward, (N > 1: all-reduce of the two flat gradient buffers), fused SGD step.  Returns the result dict."""
    from yolov7_d2_b200 import optim as yopt, synth
    from yolov7_d2_b200.yolox_convnext import YoloxConvNeXtEngine

    eng = YoloxConvNeXtEngine(batch, 640, 640, device=dev)
    eng.init_weights(0)
    for pname in eng.cn.param_names:  # a trained-like layer scale instead of the 1e-6 initial value, so the residual branches carry signal
        if pname.endswith("gamma"):
            eng.cn.params[pname].fill_(0.1)
    images, labels = synth.synthetic_batch(batch, 640, seed=200 + rank)
    eng.images_u8.copy_(images.to(dev))
    eng.labels.copy_(labels.to(dev))
    cfg = yolox_s_cfg("cuda")
    opt = yopt.build_optimizer_mapper(cfg, eng) if with_optimizer else None
    if opt is not None:
        opt.grad_scale = 1.0 / world
    grads = [g for _, g, _, _ in eng.flat_buffers()]

    def fb():
        eng.train_step()
        if opt is not None and world == 1:
            opt.step()

    def eager():
        eng.train_step()
        if world > 1:
            for g in grads:
                dist.all_reduce(g)
        if opt is not None:
            opt.step()

    for _ in range(max(warmup, 3)):
        eager()
    torch.cuda.synchronize()
    launches = eng.kernel_launches // max(warmup, 3)
    graph = None
    if use_graph:
        try:
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, capture_error_mode="thread_local"):
                fb()
            graph = g
            graph.replay()
            torch.cuda.synchronize()
        except Exception as e:  # noqa: BLE001
            sys.stderr.write(f"[bench] yolox_convnext graph capture failed ({e}); eager launches\n")
            graph = None
            torch.cuda.synchronize()

    def step():
        if graph is None:
            return eager()
        graph.replay()
        if world > 1:
            for g in grads:
                dist.all_reduce(g)
            if opt is not None:
                opt.step()

    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    if world > 1:
        dist.barrier()
    torch.cuda.synchronize()
    e0.record()
    for _ in range(steps):
        step()
    e1.record()
    if world > 1:
        dist.barrier()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1)
    if world > 1:
        t = torch.tensor([ms], device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        ms = float(t)
    ips = world * batch * steps / (ms / 1e3)
    out = {"workload": "YOLOX-ConvNeXt-T (ConvNeXt-T stages 1-3 -> PAFPN / head width 0.75), %d x 640x640 per GPU, fwd + SimOTA/loss + bwd%s%s" % (
               batch, " + all-reduce" if world > 1 else "", " + fused SGD" if opt is not None else ""),
           "images_per_s": ips, "ms_per_step": ms / steps, "n_gpus": world, "global_batch": world * batch, "cuda_graph": graph is not None,
           "launches_per_step": launches, "loss": float(eng.losses[0])}
    del eng
    torch.cuda.empty_cache()
    return out


def dump_outputs(out_dir, eng, torch):
    """What the timed step handed its caller in the last timed step, as DIR/<name>.npy: the six loss values (float64), the decoded head
    outputs, the flat gradient and the flat parameters after the optimizer step (float32).  Arrays above 4 M entries are replaced by a fixed,
    seeded sample of 4 M entries (the same positions in every run), so the files stay under 64 MB in all and two builds can be compared."""
    import numpy as np

    os.makedirs(out_dir, exist_ok=True)
    cap = 1 << 22

    def sample(t, seed):
        flat = t.detach().reshape(-1)
        if flat.numel() <= cap:
            return flat
        idx = torch.randperm(flat.numel(), generator=torch.Generator().manual_seed(seed))[:cap].sort().values
        return flat[idx.to(flat.device)]

    arrays = {"losses": eng.losses.detach().double(), "head_outputs": sample(eng.outputs, 1), "flat_grad": sample(eng.flat_grad, 2),
              "flat_param": sample(eng.flat_param, 3)}
    for name, t in arrays.items():
        a = t.cpu().numpy()
        np.save(os.path.join(out_dir, name + ".npy"), a if a.dtype == np.float64 else a.astype(np.float32))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="yb200", choices=["yb200", "reference"])
    ap.add_argument("--batch", type=int, default=64, help="images per GPU (BASELINE.json configs[1]: 64)")
    ap.add_argument("--ref-batch", type=int, default=16, help="images per CPU step of the reference arm / cpu_baseline: enough work per step to use every host core (bs=2 left most of a 128-thread host idle)")
    ap.add_argument("--no-graph", action="store_true", help="launch kernels eagerly instead of replaying a CUDA graph")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-e2e", action="store_true")
    ap.add_argument("--no-convnext", action="store_true")
    ap.add_argument("--no-library-bar", action="store_true")
    ap.add_argument("--workload", default="yolox_s", choices=["yolox_s", "yolox_convnext"],
                    help="yolox_s = the headline metric (BASELINE.json configs[1]); yolox_convnext = configs[2] (32 images per GPU; `--gpus 8` = bs 256)")
    ap.add_argument("--no-prefetch", action="store_true", help="e2e leg: copy each batch inside forward() (serial), as the reference does")
    ap.add_argument("--no-optimizer", action="store_true", help="time forward+backward(+all-reduce) only, without the fused SGD step")
    ap.add_argument("--dump-outputs", metavar="DIR", help="after the timed steps, write what the last timed step computed to DIR/<name>.npy (yolox_s)")
    args = ap.parse_args()
    if args.dump_outputs and args.workload != "yolox_s":
        ap.error("--dump-outputs writes the outputs of the yolox_s step; it is not implemented for --workload %s" % args.workload)
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if args.impl == "reference":
        return run_reference(args, rank, world)

    import torch
    import torch.distributed as dist
    from yolov7_d2_b200 import capi, synth  # the GPU arm never imports oracle/: inputs come from yolov7_d2_b200.synth
    from yolov7_d2_b200.engine import YoloxEngine
    from yolov7_d2_b200.modeling import YOLOX, postprocess

    if not torch.cuda.is_available():
        raise SystemExit("bench.py needs a CUDA device: the hot path has no CPU fallback")
    capi.lib()
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
    if args.workload == "yolox_convnext":
        res = yolox_convnext_step(torch, dist, dev, rank, world, 32, args.steps, args.warmup, not args.no_optimizer, not args.no_graph)
        if rank == 0:
            print(json.dumps({"metric": "images/sec (640x640) YOLOX-ConvNeXt-T fwd+bwd", "value": res["images_per_s"], "unit": "images/s", "n_gpus": world,
                              "steps": args.steps, "warmup": max(args.warmup, 3), "ms_per_step": res["ms_per_step"], "higher_is_better": True,
                              "scaling": "weak", "vs_baseline": None, "dtype": "bf16", "data": "synthetic",
                              "config": {"workload": res["workload"] + " (BASELINE.json configs[2])", "global_batch": res["global_batch"],
                                         "parallelism": f"dp{world}", "cuda_graph": res["cuda_graph"]},
                              "gpu_launches": res["launches_per_step"] * args.steps, "loss": res["loss"]}), flush=True)
        if world > 1:
            dist.destroy_process_group()
        return
    B = args.batch

    cfg = yolox_s_cfg("cuda")
    model = YOLOX(cfg)  # random initialisation of the reference architecture (seeded; wrappers.py / yolox_head.py defaults)
    model.train()
    eng = model._plan(B, 640, 640)
    images, labels = synth.synthetic_batch(B, 640, seed=100 + rank)
    eng.images_u8.copy_(images.to(dev))
    eng.labels.copy_(labels.to(dev))
    flat_grad = eng.flat_grad
    opt = None
    if not args.no_optimizer:
        from yolov7_d2_b200 import optim as yopt
        opt = yopt.build_optimizer_mapper(cfg, model)  # one fused SGD launch over the flat buffers (optimizer/build.py:234-245)
        opt.grad_scale = 1.0 / world                    # the mean of DDP, folded into the update

    # N = 1: the whole step (forward, backward, optimizer) is ONE CUDA graph.
    # N > 1: the step is three graphs -- [forward + loss + head backward], [neck backward], [backbone backward] -- and the gradient bucket of
    # each finished range is all-reduced (NCCL, communication stream) while the next graph runs (yolov7_d2_b200.dist.GradientBuckets);
    # the optimizer step follows the last reduction.
    from yolov7_d2_b200.dist import GradientBuckets
    gb = GradientBuckets(eng) if world > 1 else None
    n_seg = 3 if world > 1 else 1

    def segment(i):
        if world == 1:
            eng.train_step()
            if opt is not None:
                opt.step()
            return
        if i == 0:
            eng.pack_weights()
            eng.preprocess()
            eng.forward_features(True)
            eng.assign_and_loss(True)
        eng.backward(False, eng.ranges[gb.PARTS[i]], fresh=(i == 0))

    graphs = None

    def step():
        for i in range(n_seg):
            if graphs is not None:
                graphs[i].replay()
            else:
                segment(i)
            if gb is not None:
                gb.reduce_part(i)
        if gb is not None:
            gb.wait()
            if opt is not None:
                opt.step()

    for _ in range(max(args.warmup, 3)):
        step()
    torch.cuda.synchronize()
    launches_per_step = eng.kernel_launches // max(args.warmup, 3)

    if not args.no_graph:
        try:
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                for i in range(n_seg):
                    segment(i)
            torch.cuda.current_stream().wait_stream(s)
            torch.cuda.synchronize()
            gs = []
            for i in range(n_seg):
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g, capture_error_mode="thread_local"):
                    segment(i)
                gs.append(g)
            graphs = gs
            for _ in range(2):
                step()
            torch.cuda.synchronize()
        except Exception as e:  # noqa: BLE001
            sys.stderr.write(f"[bench] CUDA graph capture failed ({e}); timing eager launches\n")
            graphs = None
            torch.cuda.synchronize()
    graph = graphs

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    sampler = ClockSampler(local) if rank == 0 else None
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    barrier()
    e0.record()
    for _ in range(args.steps):
        step()
    e1.record()
    barrier()
    ms = e0.elapsed_time(e1)
    if world > 1:
        t = torch.tensor([ms], device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        ms = float(t)
    clocks = sampler.stop() if sampler else None
    value = world * B * args.steps / (ms / 1e3)
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, eng, torch)

    # ---- roofline: every C-ABI call of the step timed live with CUDA events on the launch stream (eager launches, weight gradients serialised
    # on the same stream), grouped into kernel classes; the class with the LARGEST summed time is the one reported ----
    pk = peaks()
    roof, classes, top_calls = None, None, None
    if rank == 0:
        calls = eng.profile_step(reps=3)
        agg = {}
        for c in calls:
            a = agg.setdefault(c["cls"], dict(ms=0.0, bytes=0.0, flops=0.0, launches=0, roof_ms=0.0))
            a["ms"] += c["ms"]; a["bytes"] += c["bytes"]; a["flops"] += c["flops"]; a["launches"] += c["launches"]
            a["roof_ms"] += max(c["bytes"] / (pk["hbm"] * 1e9), c["flops"] / (pk["tf_sust"] * 1e12)) * 1e3  # per call: max(memory, compute) floor
        serial_ms = sum(a["ms"] for a in agg.values())
        floor_ms = sum(a["roof_ms"] for a in agg.values())
        classes = []
        for name, a in sorted(agg.items(), key=lambda kv: -kv[1]["ms"]):
            gbs, tfs = a["bytes"] / a["ms"] / 1e6, a["flops"] / a["ms"] / 1e9
            classes.append({"class": name, "launches_per_step": a["launches"], "ms_per_step": round(a["ms"], 4), "share": round(a["ms"] / serial_ms, 4),
                            "algorithmic_GB": round(a["bytes"] / 1e9, 4), "GB_per_s": round(gbs, 1), "TFLOP_per_s": round(tfs, 1),
                            "frac_of_roofline": round(a["roof_ms"] / a["ms"], 4)})
        top_calls = []
        for c in sorted(calls, key=lambda c: -c["ms"])[:14]:
            fl = max(c["bytes"] / (pk["hbm"] * 1e9), c["flops"] / (pk["tf_sust"] * 1e12)) * 1e3
            top_calls.append({"call": c["label"], "ms": round(c["ms"], 4), "floor_ms": round(fl, 4), "frac_of_roofline": round(fl / c["ms"], 3) if c["ms"] > 0 else None})
        if os.environ.get("YB200_DUMP_CALLS"):  # every call of the step (label, class, ms, floor) for profiles/
            with open(os.environ["YB200_DUMP_CALLS"], "w") as f:
                for c in calls:
                    fl = max(c["bytes"] / (pk["hbm"] * 1e9), c["flops"] / (pk["tf_sust"] * 1e12)) * 1e3
                    f.write(json.dumps({"call": c["label"], "cls": c["cls"], "launches": c["launches"], "ms": round(c["ms"], 4), "floor_ms": round(fl, 4)}) + "\n")
        top_name, top = max(agg.items(), key=lambda kv: kv[1]["ms"])
        hbm_bound = top["bytes"] / (pk["hbm"] * 1e9) >= top["flops"] / (pk["tf_sust"] * 1e12)
        traffic = None
        tp = os.path.join(ROOT, "profiles", "roofline_traffic.json")
        if os.path.exists(tp):
            with open(tp) as fh:
                traffic = json.load(fh).get(top_name)
        step_ms = ms / args.steps
        if hbm_bound:
            ach, peak, unit = top["bytes"] / top["ms"] / 1e6, pk["hbm"], "GB/s"
        else:
            ach, peak, unit = top["flops"] / top["ms"] / 1e9, pk["tf_sust"], "TFLOP/s"
        roof = {"bound": "hbm" if hbm_bound else "tensor",
                "kernel": "%s: the kernel class with the largest summed time in the step (%d launches per step, %.1f %% of the serialised step)" % (
                    top_name, top["launches"], 100 * top["ms"] / serial_ms),
                "achieved": ach, "peak": peak, "unit": unit, "frac": ach / peak, "traffic": traffic,
                "traffic_note": "dram__bytes read+write of this class summed over one step (ncu --set full, profiles/), null when not captured",
                "peak_source": pk["source"] + (" hbm_gbs" if hbm_bound else " bf16_tflops_sustained (kernels timed inside a long step)"),
                "ms_per_step": top["ms"], "algorithmic_bytes_per_step": top["bytes"], "algorithmic_flops_per_step": top["flops"],
                "how": "sum over the class of (algorithmic bytes or FLOPs of the call: each tensor moved once in 16 bits) / sum of CUDA-event durations, "
                       "median of 3 eager steps; per-call numbers in `kernel_classes`",
                "step_serialised_ms": serial_ms,
                "step_frac_of_layer_roofline": floor_ms / step_ms,
                "step_frac_of_layer_roofline_note": "sum over calls of max(bytes/HBM peak, FLOPs/sustained bf16 peak) = %.3f ms, divided by the timed step (%.3f ms)" % (floor_ms, step_ms),
                "step_frac_of_sustained_peak": value / world * FLOP_PER_IMAGE / 1e12 / pk["tf_sust"],
                "step_frac_of_hbm_peak_on_algorithmic_bytes": value / world * 444e6 / 1e9 / pk["hbm"]}

    # ---- end to end through the public API: pinned host uint8 images -> loss.item() ----
    e2e = None
    if not args.no_e2e:
        # two pinned host batches used alternately; the next step's batch is handed to model.prefetch() right after this step's forward
        # was launched, so its host->device copy (inside the timed region, every step) overlaps this step's backward
        # as a detectron2 dataloader delivers them: every image its own pageable host tensor (no collated / pinned batch tensor): the model
        # gathers them into its pinned staging buffer and issues one DMA per batch
        def as_list(imgs, labs):
            b = batched_inputs_from(imgs, labs)
            for x in b:
                x["image"] = x["image"].clone()
            return b
        batches = [as_list(images, labels), as_list(images.flip(0), labels.flip(0).contiguous())]
        h2d = world * (images.numel() + labels.numel() * 4 + B * 8)
        api_i, api_cpu = [0], [0.0]
        def api_step():
            if opt is not None:
                opt.zero_grad()
            cur, nxt = batches[api_i[0] & 1], batches[(api_i[0] + 1) & 1]
            api_i[0] += 1
            losses = model(cur)
            sum(losses.values()).backward()
            if world > 1:
                dist.all_reduce(flat_grad)
            if opt is not None:
                opt.step()
            if not args.no_prefetch:
                t0 = time.perf_counter()
                model.prefetch(nxt)  # host gather + DMA of the next batch while this step's graphs run on the device
                api_cpu[0] += time.perf_counter() - t0
            return float(losses["total_loss"].detach())  # device -> host read of the step's result

        for _ in range(max(3, args.warmup)):  # call 1 eager, call 2 captures the forward / backward graphs, then replays
            api_step()
        barrier()
        api_cpu[0] = 0.0
        e0.record()
        for _ in range(args.steps):
            api_step()
        e1.record()
        barrier()
        ms2 = e0.elapsed_time(e1)
        if world > 1:
            t = torch.tensor([ms2], device=dev)
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
            ms2 = float(t)
        e2e = {"value": world * B * args.steps / (ms2 / 1e3), "unit": "images/s", "h2d_bytes_per_step": int(h2d), "d2h_bytes_per_step": 4 * world,
               "prefetch_host_ms_per_step": round(api_cpu[0] / args.steps * 1e3, 3),
               "api": ("optimizer.zero_grad() + " if opt is not None else "") + "YOLOX.forward(batched_inputs) + sum(loss_dict.values()).backward()"
                      + (" + optimizer.step()" if opt is not None else "") + " + loss.item()"
                      + ("" if args.no_prefetch else "; inputs = a list of separately allocated pageable uint8 images (as a detectron2 dataloader delivers them); model.prefetch(next batch) after the step's launches: the host gather into pinned memory and the host -> device copy overlap this step's device work")}

    # ---- NMS boxes/s (second half of the BASELINE metric) ----
    nms = None
    if rank == 0:
        pred = synth.clustered_predictions(4, 8400, 80, 7).repeat(B // 4, 1, 1).to(dev)
        cand = int(((pred[..., 4] * pred[..., 5:].max(-1).values) >= 0.001).sum())
        for _ in range(3):
            postprocess(pred.clone(), 80, 0.001, 0.65)
        clones = [pred.clone() for _ in range(5)]
        torch.cuda.synchronize()
        e0.record()
        for c in clones:
            postprocess(c, 80, 0.001, 0.65)
        e1.record()
        torch.cuda.synchronize()
        nms = {"value": cand * len(clones) / (e0.elapsed_time(e1) / 1e3), "unit": "boxes/s", "candidates_per_call": cand,
               "workload": "postprocess on [%d,8400,85] clustered stress set, conf 0.001, IoU 0.65" % B}

    final_loss = float(eng.losses[0])
    # ---- secondary workload (BASELINE.json configs[2], per-GPU share): YOLOX-ConvNeXt-T training step, 32 x 640x640 ----
    cnx_line = None
    if rank == 0 and world == 1 and not args.no_convnext:
        try:
            cnx_line = yolox_convnext_step(torch, None, dev, 0, 1, 32, 5, 3, not args.no_optimizer, not args.no_graph)
        except Exception as e:  # noqa: BLE001
            cnx_line = {"error": str(e)[:200]}

    # ---- CPU baseline: the oracle port on this box's host cores, bounded sample ----
    cpu = None
    if rank == 0 and world == 1 and not args.no_cpu_baseline:
        from oracle import yolox_oracle as orc  # the only place the GPU arm's process touches oracle/: the CPU baseline being timed
        csd = orc.yolox_state_dict(0)
        for k, v in csd.items():
            if v.dtype == torch.float32 and "running" not in k:
                v.requires_grad_(True)
        cb = args.ref_batch
        ci, cl = orc.synthetic_batch(cb, 640, 0)
        cx = ci.float()

        copt = None if opt is None else torch.optim.SGD([v for v in csd.values() if v.requires_grad], lr=BENCH_LR, momentum=0.9, weight_decay=5e-4)

        def cstep():
            for v in csd.values():
                if v.requires_grad:
                    v.grad = None
            orc.yolox_forward_train(cx, cl, csd)[0].backward()
            if copt is not None:
                copt.step()

        threads, avail = pick_cpu_threads(cstep, torch)
        t0 = time.perf_counter()
        iters = 0
        while iters < 2 or (time.perf_counter() - t0 < 15 and iters < 20):
            cstep()
            iters += 1
        cdt = time.perf_counter() - t0
        cpu = {"value": cb * iters / cdt, "unit": "images/s", "cores": threads, "cores_available": avail, "kind": "port",
               "sample": f"{iters} iterations of bs={cb} YOLOX-s 640x640 fwd+bwd(+SGD) with oracle/yolox_oracle.py, torch CPU fp32, thread count picked "
                         f"as the fastest of 8..{avail}"}

    # ---- library bar: the same step through stock PyTorch / cuDNN on this GPU (oracle port on cuda, autocast fp16 + channels_last, the
    # reference's shipped AMP setting configs/coco/yolox_s.yaml:66-68; SimOTA / losses in fp32 as yolox_head.py:350-379 does) ----
    lib_bar = None
    if rank == 0 and world == 1 and not args.no_library_bar:
        try:
            lib_bar = library_bar(torch, dev, B, opt is not None)
        except Exception as e:  # noqa: BLE001
            lib_bar = {"error": str(e)[:300]}

    if rank == 0:
        line = {"metric": METRIC, "value": value, "unit": "images/s", "n_gpus": world, "steps": args.steps, "warmup": max(args.warmup, 3),
                "ms_per_step": ms / args.steps, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "bf16",
                "data": "synthetic",
                "config": {"workload": WORKLOAD, "global_batch": world * B, "parallelism": f"dp{world}", "cuda_graph": graph is not None,
                           "optimizer": None if opt is None else "fused SGD step inside the timed step (momentum 0.9, wd 5e-4, lr %g)" % BENCH_LR,
                           "allreduce": None if world == 1 else "3 gradient buckets (head / neck / backbone+BN), NCCL all-reduce of each overlapped with the backward of the next range",
                           "l2": "per-step working set (~%.0f GB of activations and gradients) exceeds the 50 MB L2; no explicit flush" % (0.245 * B)},
                "clocks": clocks, "e2e": e2e, "gpu_launches": (launches_per_step + (1 if opt is not None else 0)) * args.steps, "roofline": roof, "kernel_classes": classes, "slowest_calls": top_calls if rank == 0 else None, "cpu_baseline": cpu, "library_bar": lib_bar, "nms": nms, "convnext": cnx_line,
                "loss": final_loss}
        print(json.dumps(line), flush=True)
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
