"""TEST INFRASTRUCTURE -- generates tests/golden/sparseinst_bwd.npz: gradients of the UNMODIFIED reference BaseIAMDecoder and GroupIAMDecoder
(yolov7/modeling/transcoders/decoder_sparseinst.py, loaded as oracle/gen_golden_sparseinst.py loads it) in float64, for fixed seeded upstream
gradients of pred_logits / pred_masks / pred_scores: d features and every parameter's gradient, on non-square maps.  Small widths keep the file
small (the group decoder's reshape fixes 4 groups, so its dim is at least 4 x 16).  Every gradient is stored as float16 of g / max|g| with
max|g| in float32 (`pack` / `unpack`): 2^-12 of each array's largest entry, far below what the tests resolve.
Run in the build container:   python -m oracle.gen_golden_sparseinst_bwd"""
import os

import numpy as np
import torch

from . import sparseinst_oracle as sio
from .gen_golden_sparseinst import load_reference, ns

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "sparseinst_bwd.npz")
# (case name, groups, state-dict seed, batch, height, width, dims): 10 masks pad to 16 (Base) / 16 per group; 13 + 2 input channels pad to 16
CASES = [("base_7x9", 0, 5, 2, 7, 9, dict(dim=32, nm=10, kd=16, nc=4, convs=2, cin=13)),
         ("group_6x10", 4, 7, 2, 6, 10, dict(dim=64, nm=10, kd=16, nc=4, convs=1, cin=13))]


def upstream(b, nm, nc, h, w, seed):
    """fixed seeded upstream gradients of (pred_logits, pred_masks, pred_scores)"""
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(b, nm, nc, generator=g, dtype=torch.float64), torch.randn(b, nm, 2 * h, 2 * w, generator=g, dtype=torch.float64) * 0.1,
            torch.randn(b, nm, 1, generator=g, dtype=torch.float64))


def state_dict(case):
    _, groups, seed, _, _, _, d = case
    return sio.decoder_state_dict(seed, in_channels=d["cin"], dim=d["dim"], num_masks=d["nm"], kernel_dim=d["kd"], num_classes=d["nc"], num_convs=d["convs"],
                                  groups=groups)


def features(case):
    """float32 values (exact in the fixture's inputs), as float64"""
    _, _, seed, b, h, w, d = case
    return torch.randn(b, d["cin"], h, w, generator=torch.Generator().manual_seed(seed + 100)).double()


def case_upstream(case):
    _, _, seed, b, h, w, d = case
    return upstream(b, d["nm"], d["nc"], h, w, seed + 200)


def pack(res, key, t):
    s = float(t.abs().max()) or 1.0
    res[key], res[key + "/scale"] = (t / s).numpy().astype(np.float16), np.float32(s)


def unpack(gold, key):
    return torch.tensor(gold[key].astype(np.float64) * float(gold[key + "/scale"]))


def main():
    mod = load_reference()
    res = {}
    for case in CASES:
        name, groups, seed, b, h, w, d = case
        dec_cfg = ns(SCALE_FACTOR=2.0, OUTPUT_IAM=False, NUM_MASKS=d["nm"], KERNEL_DIM=d["kd"], NUM_CLASSES=d["nc"], INST=ns(DIM=d["dim"], CONVS=d["convs"]),
                     MASK=ns(DIM=d["dim"], CONVS=d["convs"]))
        if groups:
            dec_cfg.GROUPS = groups
        cfg = ns(MODEL=ns(SPARSE_INST=ns(ENCODER=ns(NUM_CHANNELS=d["cin"]), DECODER=dec_cfg)))
        dec = (mod.GroupIAMDecoder if groups else mod.BaseIAMDecoder)(cfg)
        dec.load_state_dict(state_dict(case), strict=True)
        dec.double().train()
        feat = features(case).requires_grad_(True)
        out = dec(feat)
        torch.autograd.backward([out["pred_logits"], out["pred_masks"], out["pred_scores"]], list(case_upstream(case)))
        res[f"{name}/meta"] = np.array([groups, seed, b, h, w])
        pack(res, f"{name}/d_features", feat.grad)
        for k, p in dec.named_parameters():
            pack(res, f"{name}/grad/{k}", p.grad)
    np.savez_compressed(OUT, **res)
    print("wrote", OUT, "%.1f KB" % (os.path.getsize(OUT) / 1e3))


if __name__ == "__main__":
    main()
