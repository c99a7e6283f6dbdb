"""oracle/detr_criterion_oracle.py against the unmodified reference HungarianMatcher / SetCriterion / DETR (tests/golden/detr_criterion.npz,
oracle/gen_golden_detr_criterion.py), the fixture's coverage, and the host-side argument checks and sm_90a build of csrc/detr_criterion.cu."""
import ctypes
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import detr_criterion_oracle as dco

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "detr_criterion.npz")
CASES = ("l6", "q100", "q300", "g_over_q", "empty")


@pytest.fixture(scope="module")
def gold():
    return np.load(GOLD, allow_pickle=False)


def load_case(gold, name, dtype=torch.float32):
    """(layers [(logits, boxes)], targets, dims, eos_coef, costs, weights [L, 3]) of one fixture case"""
    p = name + "/"
    L, B, Q, K1 = (int(v) for v in gold[p + "dims"])
    sizes = [int(s) for s in gold[p + "sizes"]]
    off = np.concatenate([[0], np.cumsum(sizes)])
    labels, tboxes = torch.tensor(gold[p + "labels"]), torch.tensor(gold[p + "tboxes"]).to(dtype)
    targets = [{"labels": labels[off[b]:off[b + 1]], "boxes": tboxes[off[b]:off[b + 1]]} for b in range(B)]
    logits = (torch.tensor(gold[p + "logit_codes"]).float() * float(gold[p + "logit_scale"])).to(dtype)  # exact: int16 codes times 2^-10
    boxes = torch.tensor(gold[p + "boxes"]).to(dtype)
    layers = [(logits[l], boxes[l]) for l in range(L)]
    costs = tuple(float(c) for c in gold[p + "costs"])
    return layers, targets, (L, B, Q, K1), float(gold[p + "eos_coef"]), costs, torch.tensor(gold[p + "weights"]).to(dtype)


def golden_indices(gold, name):
    """per layer, per image (i, j) from the fixture's flat idx arrays"""
    p = name + "/"
    L, B, Q, K1 = (int(v) for v in gold[p + "dims"])
    sizes = [int(s) for s in gold[p + "sizes"]]
    ii, jj = torch.tensor(gold[p + "idx_i"]), torch.tensor(gold[p + "idx_j"])
    out, k = [], 0
    for _ in range(L):
        per = []
        for g in sizes:
            n = min(Q, g)
            per.append((ii[k:k + n], jj[k:k + n]))
            k += n
        out.append(per)
    return out


def packed_cost(layers, targets, costs):
    return torch.cat([blk.flatten() for lg, bx in layers for blk in dco.match_cost(lg, bx, targets, *costs)] or [torch.zeros(0)])


@pytest.mark.parametrize("name", CASES)
def test_restatement_reproduces_the_reference(gold, name):
    p = name + "/"
    layers, targets, (L, B, Q, K1), eos, costs, w = load_case(gold, name)
    # cost blocks: fp32 restatement within 1e-6
    ref_cost = torch.tensor(gold[p + "cost"])
    got = packed_cost(layers, targets, costs)
    assert got.shape == ref_cost.shape
    assert torch.allclose(got, ref_cost, rtol=1e-6, atol=1e-6), (got - ref_cost).abs().max()
    # assignment
    layers = [(lg.clone().requires_grad_(True), bx.clone().requires_grad_(True)) for lg, bx in layers]
    losses, idx = dco.criterion(layers, targets, K1 - 1, eos, costs)
    for got_l, ref_l in zip(idx, golden_indices(gold, name)):
        for (gi, gj), (ri, rj) in zip(got_l, ref_l):
            assert torch.equal(gi, ri) and torch.equal(gj, rj)
    # loss values and key order
    assert list(losses.keys()) == [str(k) for k in gold[p + "keys"]]
    ref = gold[p + "losses"]
    for l in range(L):
        sfx = "" if l == L - 1 else f"_{l}"
        for k, key in enumerate(("loss_ce", "loss_bbox", "loss_giou", "cardinality_error")):
            assert abs(float(losses[key + sfx]) - ref[l, k]) <= 1e-6 * abs(ref[l, k]) + 1e-7, (key + sfx, float(losses[key + sfx]), ref[l, k])
    assert float(losses["class_error"]) == ref[L - 1, 4]
    # gradients of Σ w · loss
    total = sum(w[l, k] * losses[key + ("" if l == L - 1 else f"_{l}")] for l in range(L) for k, key in enumerate(("loss_ce", "loss_bbox", "loss_giou")))
    total.backward()
    dl, rows, db = torch.tensor(gold[p + "dlogits"]), torch.tensor(gold[p + "grad_rows"]), torch.tensor(gold[p + "dboxes"])
    got = torch.stack([lg.grad for lg, _ in layers]).reshape(-1, K1)[rows]
    assert (got - dl).abs().max() <= 1e-6 * max(dl.abs().max().item(), 1e-30)
    for l, (lg, bx) in enumerate(layers):
        assert (bx.grad - db[l]).abs().max() <= 1e-6 * max(db.abs().max().item(), 1e-30)


def test_restatement_reproduces_the_detr_tail(gold):
    sd = {k[len("heads/sd/"):]: torch.tensor(gold[k]) for k in gold.files if k.startswith("heads/sd/")}
    proj = dco.input_proj(torch.tensor(gold["heads/src"]), sd)
    assert torch.allclose(proj, torch.tensor(gold["heads/proj"]), rtol=1e-5, atol=1e-5)
    logits, boxes = dco.heads(torch.tensor(gold["heads/hs"]), sd)
    ref_l = np.concatenate([gold["heads/aux_logits"], gold["heads/pred_logits"][None]])
    ref_b = np.concatenate([gold["heads/aux_boxes"], gold["heads/pred_boxes"][None]])
    assert torch.allclose(logits, torch.tensor(ref_l), rtol=1e-5, atol=1e-5)
    assert torch.allclose(boxes, torch.tensor(ref_b), rtol=1e-5, atol=1e-6)


def test_fixture_covers_the_required_cases(gold):
    dims = {n: tuple(int(v) for v in gold[n + "/dims"]) for n in CASES}
    sizes = {n: [int(s) for s in gold[n + "/sizes"]] for n in CASES}
    assert {d[0] for d in dims.values()} >= {1, 6}
    assert {d[2] for d in dims.values()} >= {100, 300}
    assert {d[3] for d in dims.values()} >= {81, 92}
    assert any(0 in s and sum(s) > 0 for s in sizes.values()), "an image without targets next to one with targets"
    assert any(sum(s) == 0 for s in sizes.values()), "a batch without targets"
    assert any(1 in s for s in sizes.values())
    assert any(dims[n][2] in s for n, s in sizes.items()), "G = Q"
    assert any(max(s) > dims[n][2] for n, s in sizes.items()), "G > Q"
    assert any(abs(float(gold[n + "/eos_coef"]) - 0.1) > 1e-6 for n in CASES), "a non-default eos_coef"
    for n in CASES:  # the logit gradient is kept on every matched row and some unmatched rows of each (layer, image)
        L, B, Q, K1 = dims[n]
        rows = gold[n + "/grad_rows"]
        assert gold[n + "/dlogits"].shape == (len(rows), K1) and len(set(rows.tolist())) == len(rows)
        assert all(any((l * B + b) * Q <= r < (l * B + b + 1) * Q for r in rows) for l in range(L) for b in range(B))
    assert "heads/pred_logits" in gold.files and "heads/sd/input_proj.weight" in gold.files


_ARGS_SCRIPT = r"""
import ctypes, json, sys
sys.path.insert(0, sys.argv[1])
from yolov7_d2_b200 import capi
L = capi.lib()
P = ctypes.c_void_p(0x10000)
f = ctypes.c_float
def cost(**kw):
    a = dict(lg=P, bx=P, lab=P, tb=P, off=P, L=6, B=2, Q=100, K1=81, G=5, out=P)
    a.update(kw)
    return [a["lg"], a["bx"], a["lab"], a["tb"], a["off"], a["L"], a["B"], a["Q"], a["K1"], a["G"], f(1), f(5), f(2), a["out"], None]
def loss(bwd=False, **kw):
    a = dict(lg=P, bx=P, m=P, lab=P, tb=P, off=P, L=6, B=2, Q=100, K1=81, eos=0.1, nb=1.0, g=P, dl=P, db=P, out=P)
    a.update(kw)
    head = [a["lg"], a["bx"], a["m"], a["lab"], a["tb"], a["off"], a["L"], a["B"], a["Q"], a["K1"], f(a["eos"]), f(a["nb"])]
    return head + ([a["g"], a["dl"], a["db"], None] if bwd else [a["out"], None])
rows = [
    ("yb200_detr_match_cost", cost(lg=None)), ("yb200_detr_match_cost", cost(out=None)), ("yb200_detr_match_cost", cost(off=None)),
    ("yb200_detr_match_cost", cost(Q=0)), ("yb200_detr_match_cost", cost(K1=1)), ("yb200_detr_match_cost", cost(G=-1)),
    ("yb200_detr_match_cost", cost(B=2000)), ("yb200_detr_match_cost", cost(L=6, B=1000, Q=3000)),
    ("yb200_detr_set_loss", loss(m=None)), ("yb200_detr_set_loss", loss(out=None)), ("yb200_detr_set_loss", loss(nb=0.0)),
    ("yb200_detr_set_loss", loss(eos=-1.0)), ("yb200_detr_set_loss", loss(L=0)), ("yb200_detr_set_loss", loss(tb=None)),
    ("yb200_detr_set_loss_bwd", loss(True, g=None)), ("yb200_detr_set_loss_bwd", loss(True, db=None)), ("yb200_detr_set_loss_bwd", loss(True, B=-1)),
    ("yb200_detr_set_loss_bwd", loss(True, m=None)),
]
res = [(n, getattr(L, n)(*a), L.yb200_last_error().decode()) for n, a in rows]
print(json.dumps(res))
"""


def test_entry_points_reject_bad_arguments_without_gpu():
    """exact return codes and messages naming the entry point; the GPUs are hidden, so a call that wrongly passed validation would fail with
    -3 at its launch instead of running on fake pointers"""
    import json

    from yolov7_d2_b200 import build, capi

    if build.find_nvcc() is None and not os.path.exists(capi.LIB_PATH):
        pytest.skip("no nvcc and no prebuilt libyb200.so")
    build.build()
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    r = subprocess.run([sys.executable, "-c", _ARGS_SCRIPT, ROOT], capture_output=True, text=True, env=env, timeout=300)
    assert r.returncode == 0, r.stderr
    res = json.loads(r.stdout.strip().splitlines()[-1])
    want = [-1, -1, -1, -1, -1, -1, -2, -2, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1]
    assert [rc for _, rc, _ in res] == want, res
    for name, rc, msg in res:
        assert msg.startswith(name[len("yb200_"):] + ":"), (name, msg)
    assert "null" in res[0][2] and "null match" in res[8][2] and "num_boxes=0" in res[10][2] and "null grad" in res[14][2]


def test_kernels_compile_for_sm90a_without_spills():
    from yolov7_d2_b200 import build

    nvcc = build.find_nvcc()
    if nvcc is None:
        pytest.skip("nvcc not available")
    src = os.path.join(ROOT, "yolov7_d2_b200", "csrc", "detr_criterion.cu")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v", "-c", src, "-o", os.devnull],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    frames = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    assert len(frames) == 3, r.stderr
    assert all(f == ("0", "0", "0") for f in frames), r.stderr
