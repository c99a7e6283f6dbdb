"""Per-layer forward convolution vs its mirror data gradient, at the exact views of the YOLOX-s training plan (bs 64, 640x640).

The forward convolution of a layer and its data gradient are mirror-image implicit GEMMs with the same FLOPs (N and K swapped) and run
the same kernel, so the difference of their times is a cost only one direction pays.  For every convolution of the plan this script
times, each as a CUDA graph of --reps launches (so host launch overhead is not part of the number):

  (a) yb200_conv2d_fwd (or _fwd_fold for the stem) with BatchNorm statistics, exactly as the training step calls it
  (b) the same call without statistics (stat_sum = NULL: the EPI_F16 epilogue)
  (c) the layer's yb200_conv2d_dgrad, with the addend the training step passes
  (d) (a) on dense copies of its input and output (no channel slice, no channel pitch)

and prints the launch parameters of (a) and (c) (column tile BN, k-block BK, CTAs per SM, k-blocks per ring slot, ring stages, pixel
tile, grid), one table of fwd / dgrad per layer and the sums over the plan.

    python tools/conv_pairs.py [--reps 50] [--json out.json]
"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from yolov7_d2_b200 import capi, synth  # noqa: E402
from yolov7_d2_b200.engine import ConvOp, YoloxEngine  # noqa: E402


# ---- launch parameters: a restatement of the host-side choices in csrc/conv_api.cu (pick_block_k / pick_block_n, choose_tile in
# csrc/host_common.cu, launch_conv_inst) and csrc/conv_gemm.cuh (conv_min_ctas, ConvEpiCfg, kMaxStagesP) for the YOLOX modes ----
def pick_block_k(c):
    return 64 if c % 64 == 0 else 32 if c % 32 == 0 else 16 if c % 16 == 0 else 0


def pick_block_n(c):
    return 128 if c > 64 else 64 if c > 32 else 32 if c > 16 else 16


def choose_tile(n, h, w, npix=128):
    lp = npix.bit_length() - 1
    best, bw, bh = -1, 0, 0
    for lw in range(lp, -1, -1):
        for lh in range(lp - lw, -1, -1):
            tw, th, tn = 1 << lw, 1 << lh, npix >> (lw + lh)
            cost = -(-w // tw) * tw * -(-h // th) * th * -(-n // tn) * tn
            if best < 0 or cost < best:
                best, bw, bh = cost, lw, lh
    return bw, bh


def launch_params(bn, bk, n, h, w, num_kb, cols, phases, sms):
    lw, lh = choose_tile(n, h, w)
    tw, th, tn = 1 << lw, 1 << lh, 128 >> (lw + lh)
    tiles = -(-w // tw) * -(-h // th) * -(-n // tn)
    occ = 1 if (bn >= 128 or bk == 16) else 2
    kcols = (bn if bn < 32 else 32) if bn <= 64 else 64
    fixed = 2 * 64 * (kcols + 4) * 4
    stage = 128 * bk * 2 + bn * bk * 2
    slots_kb = ((212 if occ == 1 else 104) * 1024 - 1024 - fixed) // stage
    kbs = 1
    if bk <= 32:
        for t in range(1, num_kb + 1):
            if num_kb % t == 0 and t * bk <= 144 and 2 * t <= slots_kb:
                kbs = t
    pst = max(2, min(slots_kb // kbs, 8))
    n_tiles = -(-cols // bn)
    m_tiles = tiles * phases
    groups = min(max((occ * sms) // n_tiles, 1), m_tiles)
    if phases == 4 and groups > 1 and groups % 2 == 0:
        groups -= 1
    return dict(BN=bn, BK=bk, ctas_per_sm=occ, kb_per_slot=kbs, stages=pst, tile="%dx%dx%d" % (tw, th, tn),
                grid=groups * n_tiles, work_items=m_tiles * n_tiles)


def act_of(arg):
    """the yb200_act a recorded ctypes.byref() argument points at (None for NULL)"""
    return None if arg is None else arg._obj


class Recorder:
    """stands in for the library during one training step and records the convolution calls with their arguments"""

    def __init__(self, lib):
        self._lib, self.fwd, self.dgrad = lib, [], []

    def __getattr__(self, name):
        fn = getattr(self._lib, name)
        if name in ("yb200_conv2d_fwd", "yb200_conv2d_fwd_fold"):
            def rec(*a):
                self.fwd.append((name, a))
                return fn(*a)
            return rec
        if name == "yb200_conv2d_dgrad":
            def rec(*a):
                self.dgrad.append(a)
                return fn(*a)
            return rec
        return fn


def graph_ms(call, reps, rounds=3):
    """device time of one call: `reps` launches captured in one CUDA graph, median over `rounds` replays"""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):
            call()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(reps):
            call()
    g.replay()
    torch.cuda.synchronize()
    out = []
    for _ in range(rounds):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        g.replay()
        e1.record()
        torch.cuda.synchronize()
        out.append(e0.elapsed_time(e1) / reps)
    return statistics.median(out)


def gpu_info():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        q = "nvidia-smi unavailable (%s)" % e
    return name, q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--size", type=int, default=640)
    ap.add_argument("--reps", type=int, default=50, help="launches per timed CUDA graph (>= 50)")
    ap.add_argument("--json", help="also write the per-layer rows to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("conv_pairs.py needs a CUDA device")
    dev = torch.device("cuda:0")
    name, q = gpu_info()
    print("GPU: %s | power.limit, clocks.max.sm: %s" % (name, q), flush=True)
    sms = torch.cuda.get_device_properties(0).multi_processor_count

    eng = YoloxEngine(args.batch, args.size, args.size, device=dev)
    eng.init_weights(0)
    images, labels = synth.synthetic_batch(args.batch, args.size, seed=100)
    eng.images_u8.copy_(images.to(dev))
    eng.labels.copy_(labels.to(dev))
    eng.train_step()
    rec = Recorder(eng.L)
    eng.L = rec
    eng.train_step()  # record every convolution call of one step with the views it passes
    eng.L = rec._lib
    torch.cuda.synchronize()

    L = capi.lib()
    convs = [op for op in eng.ops if isinstance(op, ConvOp)]
    assert len(rec.fwd) == len(convs), (len(rec.fwd), len(convs))
    dgrad_of = {int(a[1].value): a for a in rec.dgrad}
    s_sum = torch.zeros(4096, dtype=torch.float64, device=dev)
    s_sq = torch.zeros_like(s_sum)
    rows = []
    for op, (fname, a) in zip(convs, rec.fwd):
        x, z = act_of(a[0]), act_of(a[2])
        k, s = a[3], a[4]
        fold = (a[7],) if fname == "yb200_conv2d_fwd_fold" else ()
        fwd = getattr(L, fname)
        call_a = lambda x=x, z=z: capi.check(fwd(ctypes.byref(x), a[1], ctypes.byref(z), k, s, capi.ptr(s_sum), capi.ptr(s_sq), *fold,
                                                 capi.stream_ptr()), "fwd")
        call_b = lambda: capi.check(fwd(ctypes.byref(x), a[1], ctypes.byref(z), k, s, None, None, *fold, capi.stream_ptr()), "fwd (no stats)")
        # dense copies: the same values without slice or pitch (the stem's views are the pixel-grouped ones it is called with)
        xt = op.x.buf.t.view(x.n, x.h, x.w, x.c_pitch)[..., x.c_off:x.c_off + x.c].contiguous()
        zt = torch.empty(z.n, z.h, z.w, z.c, dtype=torch.float16, device=dev)
        xd, zd = capi.act(xt), capi.act(zt)
        ta = graph_ms(call_a, args.reps)
        tb = graph_ms(call_b, args.reps)
        td = graph_ms(lambda: call_a(xd, zd), args.reps)
        row = dict(layer=op.prefixes[0], shape=YoloxEngine._desc(op), x_view="c%d/pitch%d+%d" % (x.c, x.c_pitch, x.c_off),
                   fwd_ms=ta, fwd_nostats_ms=tb, fwd_dense_ms=td)
        bk, bn = pick_block_k(x.c), pick_block_n(z.c)
        row["fwd_launch"] = launch_params(bn, bk, z.n, z.h, z.w, k * k * (x.c // bk), z.c, 1, sms)
        d = dgrad_of.get(op.w_dgrad.data_ptr()) if op.w_dgrad is not None else None
        if d is not None:
            dz, dx, add = act_of(d[0]), act_of(d[2]), act_of(d[3])
            call_c = lambda: capi.check(L.yb200_conv2d_dgrad(ctypes.byref(dz), d[1], ctypes.byref(dx), ctypes.byref(add) if add is not None else None,
                                                             k, s, capi.stream_ptr()), "dgrad")
            row["dgrad_ms"] = graph_ms(call_c, args.reps)
            row["dgrad_addend"] = add is not None
            bk, bn = pick_block_k(dz.c), pick_block_n(dx.c)
            row["dgrad_launch"] = launch_params(bn, bk, dz.n, dz.h, dz.w, (dz.c // bk) * (1 if s == 2 else k * k), dx.c, 4 if s == 2 else 1, sms)
        rows.append(row)
        del xt, zt

    lp = lambda p: "%3d %2d %d %2d %d %-8s %5d" % (p["BN"], p["BK"], p["ctas_per_sm"], p["kb_per_slot"], p["stages"], p["tile"], p["grid"])
    print("\n%-28s %-24s %-18s %8s %8s %8s %8s %6s  %-36s %-36s" % ("layer", "x -> cout k s", "x view", "(a)fwd", "(b)nostat", "(d)dense", "(c)dgrad",
                                                                "a/c", "fwd: BN BK cta kbs st tile grid", "dgrad: BN BK cta kbs st tile grid"))
    for r in rows:
        c = r.get("dgrad_ms")
        print("%-28s %-24s %-18s %8.4f %8.4f %8.4f %8s %6s  %-36s %-36s" % (
            r["layer"], r["shape"], r["x_view"], r["fwd_ms"], r["fwd_nostats_ms"], r["fwd_dense_ms"], "%.4f" % c if c is not None else "-",
            "%.2f" % (r["fwd_ms"] / c) if c else "-", lp(r["fwd_launch"]), lp(r["dgrad_launch"]) if "dgrad_launch" in r else "-"))
    paired = [r for r in rows if "dgrad_ms" in r]
    sa = sum(r["fwd_ms"] for r in rows)
    sb = sum(r["fwd_nostats_ms"] for r in rows)
    sd = sum(r["fwd_dense_ms"] for r in rows)
    pa = sum(r["fwd_ms"] for r in paired)
    pc = sum(r["dgrad_ms"] for r in paired)
    only = [r for r in rows if "dgrad_ms" not in r]
    print("\nsum over the plan, ms: (a) fwd %.3f | (b) fwd without statistics %.3f | (d) fwd on dense copies %.3f" % (sa, sb, sd))
    print("layers with a data gradient: fwd %.3f vs dgrad %.3f -> fwd / dgrad %.3f, forward-only cost %.3f ms" % (pa, pc, pa / pc, pa - pc))
    print("forward-only layers (no data gradient): %s = %.3f ms" % (", ".join(r["layer"] for r in only), sum(r["fwd_ms"] for r in only)))
    print("of the forward-only cost: statistics epilogue (a)-(b) %.3f ms, slices / pitch (a)-(d) %.3f ms, stem %.3f ms" % (
        sa - sb, sa - sd, sum(r["fwd_ms"] for r in only)))
    if args.json:
        with open(args.json, "w") as fh:
            json.dump(dict(gpu=name, power_and_clock=q, rows=rows), fh, indent=1)


if __name__ == "__main__":
    main()
