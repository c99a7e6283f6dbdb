"""One profiled training step (use under ncu with --profile-from-start off):
   ncu --metrics gpu__time_duration.sum --clock-control none --profile-from-start off --csv --log-file profile_out/launches.csv \
       python tools/profile_step.py --batch 64
"""
import argparse, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from yolov7_d2_b200 import synth
from yolov7_d2_b200.engine import YoloxEngine

ap = argparse.ArgumentParser()
ap.add_argument("--batch", type=int, default=64)
ap.add_argument("--size", type=int, default=640)
ap.add_argument("--warmup", type=int, default=2)
ap.add_argument("--eval", action="store_true")
a = ap.parse_args()
dev = torch.device("cuda:0")
eng = YoloxEngine(a.batch, a.size, a.size, device=dev)
eng.init_weights(0)
images, labels = synth.synthetic_batch(a.batch, a.size, 100)
eng.images_u8.copy_(images.to(dev)); eng.labels.copy_(labels.to(dev))
for _ in range(a.warmup):
    eng.eval_forward() if a.eval else eng.train_step()
torch.cuda.synchronize()
eng.trace = []
torch.cuda.profiler.start()
eng.eval_forward() if a.eval else eng.train_step()
torch.cuda.synchronize()
torch.cuda.profiler.stop()
import json
os.makedirs("profile_out", exist_ok=True)
json.dump(eng.trace, open("profile_out/trace.json", "w"))
print("profiled one step; loss", float(eng.losses[0]))
