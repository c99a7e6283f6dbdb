"""Bit-for-bit comparison of the 16-bit convolution outputs of two builds of libyb200.so, at the exact views of the YOLOX-s training plan.

Records every forward convolution and data gradient of one training step (the views, slices and addends the step passes), then runs each
call with both libraries on the same seeded operands into identically pre-filled output buffers and compares the whole enclosing buffers
bit for bit (the view and the channels around it):

  conv2d_fwd / conv2d_fwd_fold   z (fp16), and with the BatchNorm statistics: z and the fp64 Σ / Σ² of the call
  conv2d_dgrad                   dx (bf16), with the addend the step passes
  conv2d_bn_silu_fwd             the eval epilogue on each forward view, with a residual of the output's shape

    python tools/conv_bitcheck.py --ref-lib OTHER/libyb200.so [--batch 64] [--size 640]
"""
import argparse
import ctypes
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from yolov7_d2_b200 import capi, synth  # noqa: E402
from yolov7_d2_b200.engine import YoloxEngine  # noqa: E402

from conv_pairs import Recorder, act_of  # noqa: E402


def buffer_of(a, dtype, g, fill=None):
    """a fresh [n, h, w, pitch] buffer with the geometry of view `a`: seeded values, or `fill`"""
    shape = (a.n, a.h, a.w, a.c_pitch)
    if fill is not None:
        return torch.full(shape, fill, dtype=dtype, device="cuda")
    return torch.randn(shape, generator=g, device="cuda").to(dtype)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ref-lib", required=True, help="the other build's libyb200.so")
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--size", type=int, default=640)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("conv_bitcheck.py needs a CUDA device")
    dev = torch.device("cuda:0")
    eng = YoloxEngine(args.batch, args.size, args.size, device=dev)
    eng.init_weights(0)
    images, labels = synth.synthetic_batch(args.batch, args.size, seed=100)
    eng.images_u8.copy_(images.to(dev))
    eng.labels.copy_(labels.to(dev))
    rec = Recorder(eng.L)
    eng.L = rec
    eng.train_step()
    eng.L = rec._lib
    torch.cuda.synchronize()

    ref = ctypes.CDLL(os.path.abspath(args.ref_lib))
    ref.yb200_last_error.restype = ctypes.c_char_p
    libs = (("this", capi.lib()), ("ref", ref))

    def run(name, fn_name, make_args, *bufs):
        """calls fn_name of both libraries on copies of `bufs`; make_args(*copies) -> argument tuple; True when every copy is identical"""
        outs = []
        for tag, L in libs:
            o = [b.clone() for b in bufs]
            rc = getattr(L, fn_name)(*make_args(*o))
            if rc != 0:
                raise SystemExit("%s: %s (%s) failed: %s" % (name, fn_name, tag, L.yb200_last_error().decode()))
            torch.cuda.synchronize()
            outs.append(o)
        same = True
        for a, b in zip(*outs):
            bits = torch.int16 if a.element_size() == 2 else torch.int64
            diff = int((a.view(bits) != b.view(bits)).sum())
            if diff:
                same = False
                print("DIFFERENT %-40s %s: %d of %d elements" % (name, fn_name, diff, a.numel()), flush=True)
        return same

    g = torch.Generator(device="cuda").manual_seed(7)
    checked = bad = 0
    st = capi.stream_ptr()
    for i, (fname, a) in enumerate(rec.fwd):
        x, z = act_of(a[0]), act_of(a[2])
        k, s = a[3], a[4]
        fold = (a[7],) if fname == "yb200_conv2d_fwd_fold" else ()
        xb = buffer_of(x, torch.bfloat16, g)
        wt = (torch.randn(z.c, k * k * x.c, generator=g, device="cuda") / (k * k * x.c) ** 0.5).to(torch.bfloat16)
        xa = capi.Act(xb.data_ptr(), x.n, x.h, x.w, x.c, x.c_pitch, x.c_off)

        def fwd_args(o, z=z, xa=xa, wt=wt, k=k, s=s, fold=fold):
            za = capi.Act(o.data_ptr(), z.n, z.h, z.w, z.c, z.c_pitch, z.c_off)
            return (ctypes.byref(xa), capi.ptr(wt), ctypes.byref(za), k, s, None, None, *fold, st)

        bad += not run("fwd %d" % i, fname, fwd_args, buffer_of(z, torch.float16, g, fill=-7.0))
        nst = fold[0] if fold else z.c

        def stats_args(o, ssum, ssq, z=z, xa=xa, wt=wt, k=k, s=s, fold=fold):
            za = capi.Act(o.data_ptr(), z.n, z.h, z.w, z.c, z.c_pitch, z.c_off)
            return (ctypes.byref(xa), capi.ptr(wt), ctypes.byref(za), k, s, capi.ptr(ssum), capi.ptr(ssq), *fold, st)

        bad += not run("fwd+stats %d" % i, fname, stats_args, buffer_of(z, torch.float16, g, fill=-7.0),
                       torch.zeros(nst, dtype=torch.float64, device="cuda"), torch.zeros(nst, dtype=torch.float64, device="cuda"))
        checked += 2
        if fold:
            continue
        scale = (0.5 + torch.rand(z.c, generator=g, device="cuda")).float()
        shift = torch.randn(z.c, generator=g, device="cuda").float()
        res = torch.randn(z.n, z.h, z.w, z.c, generator=g, device="cuda").to(torch.bfloat16)
        ra = capi.act(res)

        def silu_args(o, z=z, xa=xa, wt=wt, k=k, s=s, scale=scale, shift=shift, ra=ra):
            oa = capi.Act(o.data_ptr(), z.n, z.h, z.w, z.c, z.c_pitch, z.c_off)
            return (ctypes.byref(xa), capi.ptr(wt), capi.ptr(scale), capi.ptr(shift), ctypes.byref(ra), ctypes.byref(oa), k, s, st)

        bad += not run("bn_silu %d" % i, "yb200_conv2d_bn_silu_fwd", silu_args, buffer_of(z, torch.bfloat16, g, fill=-7.0))
        checked += 1
    for i, d in enumerate(rec.dgrad):
        dz, dx, add = act_of(d[0]), act_of(d[2]), act_of(d[3])
        k, s = d[4], d[5]
        dzb = buffer_of(dz, torch.bfloat16, g)
        wt = (torch.randn(dx.c, k * k * dz.c, generator=g, device="cuda") / (k * k * dz.c) ** 0.5).to(torch.bfloat16)
        dza = capi.Act(dzb.data_ptr(), dz.n, dz.h, dz.w, dz.c, dz.c_pitch, dz.c_off)
        addb = buffer_of(add, torch.bfloat16, g) if add is not None else None
        adda = capi.Act(addb.data_ptr(), add.n, add.h, add.w, add.c, add.c_pitch, add.c_off) if add is not None else None

        def dgrad_args(o, dx=dx, dza=dza, wt=wt, adda=adda, k=k, s=s):
            dxa = capi.Act(o.data_ptr(), dx.n, dx.h, dx.w, dx.c, dx.c_pitch, dx.c_off)
            return (ctypes.byref(dza), capi.ptr(wt), ctypes.byref(dxa), ctypes.byref(adda) if adda is not None else None, k, s, st)

        bad += not run("dgrad %d (k%d s%d%s)" % (i, k, s, " +addend" if add is not None else ""), "yb200_conv2d_dgrad", dgrad_args,
                       buffer_of(dx, torch.bfloat16, g, fill=-7.0))
        checked += 1
    print("conv_bitcheck: %d calls compared, %d differ" % (checked, bad))
    raise SystemExit(1 if bad else 0)


if __name__ == "__main__":
    main()
