"""Throughput of the mosaic / random_perspective / mixup branch (yolov7_d2_b200/augment.py) for one batch of samples at the default mosaic
ranges (512..800), mixup on and off:
  (a) device-resident sources and table, the two kernels only (CUDA events);
  (b) `apply_mosaic` from pageable host sources: packing table, one H2D copy per source, the kernels (host clock around a synchronised run);
  (c) oracle/mosaic_oracle.py (cv2) on the host, one process with one cv2 thread, and one process per core.
Also the bytes the kernels must move (every source byte read once, the output written once, blended outputs read and written again) against
the H100 SXM's 3.35 TB/s, as a floor, and the H2D volume per batch.  Prints one JSON line; with --out also writes it there.

    python tools/bench_mosaic.py --n 64 --iters 20 --warmup 3 --out /tmp/bench_mosaic.json
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from oracle import mosaic_oracle as orc  # noqa: E402
from yolov7_d2_b200 import augment, capi  # noqa: E402

_BATCH = None


def _render_one(i):
    r = _BATCH[i]["mosaic"]
    return orc.render([s.numpy() for s in r["sources"]], r["draws"], bool(r.get("mixup", {}).get("blend", False))).nbytes


def _oracle_rate(batch, procs):
    import cv2

    global _BATCH
    _BATCH = batch
    cv2.setNumThreads(1)
    t0 = time.perf_counter()
    if procs == 1:
        for i in range(len(batch)):
            _render_one(i)
    else:
        import multiprocessing as mp

        with mp.get_context("fork").Pool(procs) as pool:
            t0 = time.perf_counter()  # pool start-up excluded
            pool.map(_render_one, range(len(batch)), chunksize=1)
    return len(batch) / (time.perf_counter() - t0)


def _card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        pl = pl.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        pl = f"unknown ({type(e).__name__})"
    return name, pl


def measure(n, iters, warmup, mixup, seed):
    batch = orc.synthetic_recipes(augment.MosaicMixupMapper, n, seed, mixup=mixup)
    recipes = [x["mosaic"] for x in batch]
    raw, src_total, out_total, sizes = augment.build_table(recipes)
    dev = torch.device("cuda:0")
    src = torch.cat([s.reshape(-1) for r in recipes for s in r["sources"]]).to(dev)
    table = raw.to(dev)
    out = torch.empty(out_total, dtype=torch.uint8, device=dev)
    mh, mw = max(h for h, _ in sizes), max(w for _, w in sizes)
    blended = [bool(r.get("mixup", {}).get("blend", False)) for r in recipes]
    L, st = capi.lib(), capi.stream_ptr()

    def kernels():
        capi.check(L.yb200_mosaic_warp(capi.ptr(table), n, capi.ptr(src), capi.ptr(out), mh, mw, st), "yb200_mosaic_warp")
        if any(blended):
            capi.check(L.yb200_mosaic_mixup(capi.ptr(table), n, capi.ptr(src), capi.ptr(out), mh, mw, st), "yb200_mosaic_mixup")

    for _ in range(warmup):
        kernels()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        kernels()
    e1.record()
    torch.cuda.synchronize()
    t_kern = e0.elapsed_time(e1) / 1e3 / iters

    def host_run():
        apply = [{"mosaic": x["mosaic"]} for x in batch]
        augment.apply_mosaic(apply)
        return apply

    for _ in range(warmup):
        host_run()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(iters):
        host_run()
    torch.cuda.synchronize()
    t_host = (time.perf_counter() - t0) / iters

    out_bytes = sum(3 * h * w for h, w in sizes)
    mix_bytes = sum(2 * 3 * h * w + r["sources"][4].numel() for (h, w), r, b in zip(sizes, recipes, blended) if b)
    moved = src_total + out_bytes + mix_bytes
    res = {
        "mixup": mixup, "samples": n, "blended": int(sum(blended)),
        "a_kernels_samples_per_s": n / t_kern, "a_kernels_ms": t_kern * 1e3,
        "b_from_pageable_host_samples_per_s": n / t_host, "b_ms": t_host * 1e3,
        "kernel_bytes_floor": moved, "floor_ms_at_3.35TBps": moved / 3.35e12 * 1e3,
        "floor_share_of_kernel_time": (moved / 3.35e12) / t_kern,
        "h2d_bytes_per_batch": src_total, "output_bytes_per_batch": out_bytes, "h2d_over_output": src_total / out_bytes,
    }
    res["c_oracle_1_thread_samples_per_s"] = _oracle_rate(batch, 1)
    procs = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else os.cpu_count()
    res["c_oracle_all_cores_samples_per_s"] = _oracle_rate(batch, procs)
    res["c_oracle_processes"] = procs
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=64)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_mosaic needs a CUDA device: there is no CPU fallback to time")
    name, pl = _card()
    res = {"card": name, "power_limit": pl, "cpu_count": os.cpu_count(),
           "runs": [measure(a.n, a.iters, a.warmup, mix, a.seed + mix) for mix in (True, False)]}
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
