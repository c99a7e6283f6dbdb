"""TEST INFRASTRUCTURE -- generates tests/golden/sparseinst_encoder.npz from the UNMODIFIED reference InstanceContextEncoder
(yolov7/modeling/transcoders/encoder_sparseinst.py, loaded as oracle/gen_golden_sparseinst.py loads the decoders, plus a stand-in for
alfred.utils.log) in float64: the output, d res3 / res4 / res5 and every parameter's gradient for fixed seeded upstream gradients.  Small widths
(in-channels 32 / 48 / 64, NUM_CHANNELS 64) on non-square maps whose pyramid pooling hits MyAdaptiveAvgPool2d's floor quirk: a 5x7 top level
pools to 1x1, 1x1, 2x2, 5x3 and a 4x6 one to 1x1, 2x2, 2x3, 4x6.  Arrays are stored as in oracle/gen_golden_sparseinst_bwd.py (`pack`).
Run in the build container:   python -m oracle.gen_golden_sparseinst_encoder"""
import importlib
import os
import sys
import types

import numpy as np
import torch

from . import ref_shim
from . import sparseinst_encoder_oracle as seo
from .gen_golden_sparseinst import load_reference, ns
from .gen_golden_sparseinst_bwd import pack

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "sparseinst_encoder.npz")
IN_CHANNELS, NUM_CHANNELS = (32, 48, 64), 64
# (case name, state-dict seed, batch, res5 height, res5 width): res4 / res3 are 2x / 4x the res5 map
CASES = [("top_5x7", 11, 1, 5, 7), ("top_4x6", 12, 1, 4, 6)]


def load_encoder_module():
    load_reference()
    alfred = sys.modules["alfred"]
    alfred.__path__ = []
    ref_shim._mod("alfred.utils").__path__ = []
    ref_shim._mod("alfred.utils.log", logger=alfred.logger)
    return importlib.import_module("yolov7.modeling.transcoders.encoder_sparseinst")


def cfg_of(num_channels=NUM_CHANNELS):
    return ns(MODEL=ns(SPARSE_INST=ns(ENCODER=ns(NAME="InstanceContextEncoder", NUM_CHANNELS=num_channels, IN_FEATURES=list(seo.IN_FEATURES)))))


def input_shape(in_channels=IN_CHANNELS):
    return {k: types.SimpleNamespace(channels=c) for k, c in zip(seo.IN_FEATURES, in_channels)}


def state_dict(case):
    return seo.encoder_state_dict(case[1], IN_CHANNELS, NUM_CHANNELS)


def features(case):
    """float32 values (exact in float64), {res3, res4, res5} NCHW float64"""
    _, seed, b, h, w = case
    g = torch.Generator().manual_seed(seed + 100)
    return {k: torch.randn(b, c, h * 2 ** (2 - i), w * 2 ** (2 - i), generator=g).double() for i, (k, c) in enumerate(zip(seo.IN_FEATURES, IN_CHANNELS))}


def upstream(case):
    """fixed seeded upstream gradient of the output [B, NUM_CHANNELS, 4h, 4w]"""
    _, seed, b, h, w = case
    return torch.randn(b, NUM_CHANNELS, 4 * h, 4 * w, generator=torch.Generator().manual_seed(seed + 200), dtype=torch.float64)


def main():
    mod = load_encoder_module()
    res = {}
    for case in CASES:
        name, seed, b, h, w = case
        enc = mod.InstanceContextEncoder(cfg_of(), input_shape())
        enc.load_state_dict(state_dict(case), strict=True)
        enc.double().train()
        feats = {k: v.requires_grad_(True) for k, v in features(case).items()}
        out = enc(feats)
        out.backward(upstream(case))
        res[f"{name}/meta"] = np.array([seed, b, h, w])
        pack(res, f"{name}/out", out.detach())
        for k, v in feats.items():
            pack(res, f"{name}/d_{k}", v.grad)
        for k, p in enc.named_parameters():
            pack(res, f"{name}/grad/{k}", p.grad)
    np.savez_compressed(OUT, **res)
    print("wrote", OUT, "%.1f KB" % (os.path.getsize(OUT) / 1e3))


if __name__ == "__main__":
    main()
