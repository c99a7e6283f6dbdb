"""TEST INFRASTRUCTURE -- CPU restatement (plain torch) of the reference's SparseInst InstanceContextEncoder, and the same forward with the
kernels' bf16 storage points emulated.

Reference: yolov7/modeling/transcoders/encoder_sparseinst.py -- `MyAdaptiveAvgPool2d` :18-39, `PyramidPoolingModule` :42-68,
`InstanceContextEncoder` :71-127.  Pinned by tests/golden/sparseinst_encoder.npz, produced by oracle/gen_golden_sparseinst_encoder.py from the
UNMODIFIED reference class.

`encoder_forward(features, sd)` is the reference's arithmetic; run in float64 it is the accuracy oracle.  `encoder_forward_storage(features, sd)`
rounds values, and the gradients flowing back through them, to bf16 at exactly the points where yolov7_d2_b200/sparseinst_encoder.py stores
bf16 (the inputs, every convolution's output, the pooled maps, the resized priors and outputs, the top-down sums, the weights as GEMM operands
and the bf16 addends of the top-down adjoint); run in float64 it is the yardstick of what 16-bit storage alone costs.
Only tests/ and tools/ may import it.
"""
import math

import torch
import torch.nn.functional as F

from .sparseinst_storage_oracle import _Bf16, _GradBf16, _WeightBf16

IN_FEATURES = ("res3", "res4", "res5")
PPM_SIZES = (1, 2, 3, 6)


def ppm_windows(h, w, sizes=PPM_SIZES):
    """MyAdaptiveAvgPool2d's window (= stride) per size: (ceil(H/s), ceil(W/s)); the pooled map is (H // kh, W // kw) (floor mode)"""
    return [(math.ceil(h / s), math.ceil(w / s)) for s in sizes]


def _ident(x):
    return x


def _forward(features, sd, storage, in_features=IN_FEATURES):
    s, sg, wq = (_Bf16.apply, _GradBf16.apply, _WeightBf16.apply) if storage else (_ident, _ident, _ident)

    def conv(x, name, pad=0):
        return s(F.conv2d(x, wq(sd[name + ".weight"]), sd[name + ".bias"], padding=pad))

    feats = [s(features[k]) for k in in_features][::-1]                                                     # :107-108
    lat0 = conv(feats[0], "fpn_laterals.0")
    h, w = lat0.shape[2:]
    priors = []
    for i, (kh, kw) in enumerate(ppm_windows(h, w)):                                                        # PPM :56-68
        pooled = s(F.avg_pool2d(lat0, kernel_size=(kh, kw), ceil_mode=False))                              # :36-38
        p = F.relu(conv(pooled, f"ppm.stages.{i}.1"))
        priors.append(s(F.interpolate(p, size=(h, w), mode="bilinear", align_corners=False)))
    prev = F.relu(conv(torch.cat(priors + [lat0], 1), "ppm.bottleneck"))
    outputs = [conv(prev, "fpn_outputs.0", 1)]                                                              # :110
    for lvl in range(1, len(feats)):                                                                        # :111-119
        lat = conv(feats[lvl], f"fpn_laterals.{lvl}")
        prev = s(lat + F.interpolate(sg(prev), scale_factor=2.0, mode="nearest"))
        outputs.insert(0, conv(prev, f"fpn_outputs.{lvl}", 1))
    size = outputs[0].shape[2:]                                                                             # :120-125
    cat = torch.cat([outputs[0]] + [s(F.interpolate(x, size, mode="bilinear", align_corners=False)) for x in outputs[1:]], 1)
    return conv(cat, "fusion")                                                                              # :126


def encoder_forward(features, sd, in_features=IN_FEATURES):
    """InstanceContextEncoder.forward (:106-127): features {name: NCHW} -> NCHW [B, NUM_CHANNELS, H3, W3]"""
    return _forward(features, sd, False, in_features)


def encoder_forward_storage(features, sd, in_features=IN_FEATURES):
    """encoder_forward with the kernels' bf16 storage points"""
    return _forward(features, sd, True, in_features)


def encoder_state_dict(seed=0, in_channels=(512, 1024, 2048), num_channels=256):
    """seeded parameters in the reference's names and shapes; in_channels in IN_FEATURES order (res3, res4, res5)"""
    g = torch.Generator().manual_seed(seed)

    def rn(*shape, std):
        return torch.randn(*shape, generator=g) * std

    c, c4 = num_channels, num_channels // 4
    sd = {}
    for i, cin in enumerate(reversed(in_channels)):                                                         # :88-97, index 0 = the coarsest
        sd[f"fpn_laterals.{i}.weight"], sd[f"fpn_laterals.{i}.bias"] = rn(c, cin, 1, 1, std=(1.0 / cin) ** 0.5), rn(c, std=0.05)
        sd[f"fpn_outputs.{i}.weight"], sd[f"fpn_outputs.{i}.bias"] = rn(c, c, 3, 3, std=(1.0 / (9 * c)) ** 0.5), rn(c, std=0.05)
    for i in range(len(PPM_SIZES)):
        sd[f"ppm.stages.{i}.1.weight"], sd[f"ppm.stages.{i}.1.bias"] = rn(c4, c, 1, 1, std=(2.0 / c) ** 0.5), rn(c4, std=0.1)
    sd["ppm.bottleneck.weight"], sd["ppm.bottleneck.bias"] = rn(c, c + len(PPM_SIZES) * c4, 1, 1, std=(2.0 / (2 * c)) ** 0.5), rn(c, std=0.05)
    sd["fusion.weight"], sd["fusion.bias"] = rn(c, 3 * c, 1, 1, std=(2.0 / c) ** 0.5), rn(c, std=0.05)
    return sd
