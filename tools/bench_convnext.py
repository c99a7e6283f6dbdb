"""ConvNeXt-T backbone forward+backward throughput (BASELINE.json configs[2]: 32 images per GPU at 640x640), CUDA events.
   python tools/bench_convnext.py [--batch 32] [--profile]   (--profile: one step between cudaProfilerStart/Stop for ncu)"""
import argparse, json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from yolov7_d2_b200 import synth
from yolov7_d2_b200.convnext import ConvNeXtEngine

ap = argparse.ArgumentParser()
ap.add_argument("--batch", type=int, default=32)
ap.add_argument("--size", type=int, default=640)
ap.add_argument("--steps", type=int, default=5)
ap.add_argument("--profile", action="store_true")
ap.add_argument("--no-graph", action="store_true")
ap.add_argument("--no-overlap", action="store_true")
a = ap.parse_args()
dev = torch.device("cuda:0")
eng = ConvNeXtEngine(a.batch, a.size, a.size, device=dev)
eng.init_weights(0)
for _n in eng.param_names:  # trained-like layer scale instead of the 1e-6 initial value
    if _n.endswith("gamma"):
        eng.params[_n].fill_(0.1)
eng.overlap_wgrad = not a.no_overlap
eng.images_u8.copy_(synth.synthetic_images(a.batch, a.size, 1).to(dev))
g = torch.Generator(device=dev).manual_seed(2)
for st in eng.stage:
    st.gout.t.copy_(torch.randn(st.gout.t.shape, generator=g, device=dev) * 1e-2)
for _ in range(2):
    eng.train_step()
torch.cuda.synchronize()
launches = eng.kernel_launches // 2
if a.profile:
    eng.trace = []
    torch.cuda.profiler.start()
    eng.train_step()
    torch.cuda.synchronize()
    torch.cuda.profiler.stop()
    os.makedirs("profile_out", exist_ok=True)
    json.dump(eng.trace, open("profile_out/trace_convnext.json", "w"))
    sys.exit(0)
graph = None
if not a.no_graph:
    graph = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        eng.train_step()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    with torch.cuda.graph(graph):
        eng.train_step()
    graph.replay()
    torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(a.steps):
    graph.replay() if graph is not None else eng.train_step()
e1.record()
torch.cuda.synchronize()
ms = e0.elapsed_time(e1) / a.steps
# forward only
e0.record()
for _ in range(a.steps):
    eng.pack_weights(); eng.forward_features()
e1.record()
torch.cuda.synchronize()
ms_f = e0.elapsed_time(e1) / a.steps
gf = 72.7 * (a.size / 640.0) ** 2  # GFLOP per image forward (SURVEY.md par.8a C1)
print(json.dumps({"workload": "ConvNeXt-T backbone fwd+bwd %dx%d bs=%d (BASELINE.json configs[2] per-GPU share)" % (a.size, a.size, a.batch),
                  "ms_per_step": ms, "images_per_s": a.batch / ms * 1e3, "tflops_fwd_bwd": 3 * gf * a.batch / ms, "fwd_only_ms": ms_f,
                  "fwd_images_per_s": a.batch / ms_f * 1e3, "launches_per_step": launches, "cuda_graph": graph is not None, "overlap_wgrad": eng.overlap_wgrad,
                  "finite": bool(torch.isfinite(eng.flat_grad).all())}))
