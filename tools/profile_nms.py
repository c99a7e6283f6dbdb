"""postprocess (filter + sort + per-class greedy NMS) on the clustered stress set, for ncu:
   ncu --set full --clock-control none --import-source on -k regex:nms_ -c 2 -o profile_out/prof_nms python tools/profile_nms.py
"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from yolov7_d2_b200 import synth
from yolov7_d2_b200.modeling import postprocess

dev = torch.device("cuda:0")
pred = synth.clustered_predictions(4, 8400, 80, 7).repeat(16, 1, 1).to(dev)
for _ in range(2):
    postprocess(pred.clone(), 80, 0.001, 0.65)
torch.cuda.synchronize()
torch.cuda.profiler.start()
postprocess(pred.clone(), 80, 0.001, 0.65)
torch.cuda.synchronize()
torch.cuda.profiler.stop()
print("nms profiled")
