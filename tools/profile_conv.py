"""The dominant forward GEMM in isolation (head 3x3 128 -> 256 @ 80x80, batch 64), for `ncu --set full`:
   ncu --set full --clock-control none --import-source on -k regex:conv_gemm -s 2 -c 1 -o profile_out/prof_conv python tools/profile_conv.py
"""
import ctypes, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from yolov7_d2_b200 import capi

n, h, w, cin, cout, k = 64, 80, 80, 128, 256, 3
dev = torch.device("cuda:0")
x = torch.randn(n, h, w, cin, device=dev).to(torch.bfloat16)
wt = torch.randn(cout, cin, k, k, device=dev) / (cin * k * k) ** 0.5
wf = torch.empty(cout, k * k, cin, dtype=torch.bfloat16, device=dev)
L = capi.lib()
capi.check(L.yb200_pack_conv_weight(capi.ptr(wt), cout, cin, k, cout, cin, capi.ptr(wf), None, capi.stream_ptr()), "pack")
z = torch.zeros(n, h, w, cout, dtype=torch.float16, device=dev)
ssum = torch.zeros(cout, dtype=torch.float64, device=dev)
ssq = torch.zeros(cout, dtype=torch.float64, device=dev)
xa, za = capi.act(x), capi.act(z)
for _ in range(4):
    capi.check(L.yb200_conv2d_fwd(ctypes.byref(xa), capi.ptr(wf), ctypes.byref(za), k, 1, capi.ptr(ssum), capi.ptr(ssq), capi.stream_ptr()), "fwd")
torch.cuda.synchronize()
print("algorithmic bytes per launch: in %.1f MB + out %.1f MB + weights %.2f MB; flops %.1f G" %
      (x.numel() * 2 / 1e6, z.numel() * 2 / 1e6, wf.numel() * 2 / 1e6, 2.0 * n * h * w * cout * cin * k * k / 1e9))
