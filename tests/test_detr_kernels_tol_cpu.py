"""Negative controls for the attention and LayerNorm bounds of tests/test_detr_kernels_gpu.py, on the CPU.

A faithful fp32 / bf16 emulation of the attention kernels (csrc/attention.cu: 128-key tiles, running maximum in the exp2 domain, one alpha
rescale per tile, fp32 probabilities, bf16 P and dS tiles, fp32 products; the backward from the forward's lse and the bf16 O) must pass the
bounds; the same emulation with one known defect must fail them by a clear factor.  The instance, 1 image x 2 heads x 150 queries x 300
keys, spans partial tiles on both sides (two query tiles, the second of 22 rows; three key tiles, the last of 44 keys).  Keys 200 (in the
middle tile) and 290-299 are masked and, as in the GPU tests, their k and v are scaled by 64.  LayerNorm: the two-pass fp32 statistics pass
the mean / rstd bounds, the unbiased variance fails the rstd bound.  The factors are printed at the end of the module (-s).
"""
import math

import pytest
import torch

from oracle import detr_oracle as dto
from test_detr_kernels_gpu import LOG2E, SCALE, SENT_KV, TILE, attn_bwd_ref, attn_fwd_ref, ln_ref
from test_convnext_plan_gpu import excess

FACTOR = {}   # defect -> worst err / bound of the defective result
CLEAR = 4.0   # a defect must exceed the bound by at least this factor
H, LQ, LK = 2, 150, 300
SEED, P = 1234, 0.1


def _bf(t):
    return t.to(torch.bfloat16).float()


def _inputs():
    g = torch.Generator().manual_seed(7)
    q = torch.randn(H, LQ, 32, generator=g) * torch.tensor([0.25, 1.0, 3.0]).repeat(LQ // 3)[:, None]
    k = torch.randn(H, LK, 32, generator=g)
    v = torch.randn(H, LK, 32, generator=g)
    dead = torch.zeros(LK, dtype=torch.bool)
    dead[200] = True
    dead[290:] = True
    k[:, dead] *= SENT_KV
    v[:, dead] *= SENT_KV
    do = torch.randn(H, LQ, 32, generator=g)
    return _bf(q), _bf(k), _bf(v), _bf(do), dead


def _mult(p, shift=0):
    """[H, Lq, Lk] dropout multiplier of the kernels' hash (columns shifted by `shift`), or None"""
    if p <= 0:
        return None
    return dto.attention_dropout_multiplier(SEED, 1, H, LQ, LK + shift, p)[0, :, :, shift:]


def emu_fwd(q, k, v, dead, mult, drop_last_tile=False, unmask_key=None, norm_dropped=False):
    """attention_fwd_kernel in fp32: -> (bf16 o, fp32 lse)"""
    sc2 = torch.tensor(SCALE, dtype=torch.float32) * torch.tensor(LOG2E, dtype=torch.float32)
    s = q @ k.transpose(-1, -2)
    bias = torch.where(dead, torch.tensor(-math.inf), torch.tensor(0.0))
    if unmask_key is not None:
        bias[unmask_key] = 0.0
    m = torch.full((H, LQ, 1), -math.inf)
    l = torch.zeros(H, LQ, 1)
    acc = torch.zeros(H, LQ, 32)
    ntiles = -(-LK // TILE) - (1 if drop_last_tile else 0)
    for j in range(ntiles):
        cols = slice(j * TILE, min(LK, (j + 1) * TILE))
        t = s[..., cols] * sc2 + bias[cols]
        mx = torch.maximum(m, t.amax(-1, keepdim=True))
        m_safe = torch.where(mx == -math.inf, torch.zeros_like(mx), mx)
        alpha = torch.exp2(m - m_safe)
        acc, l, m = acc * alpha, l * alpha, mx
        p = torch.exp2(t - m_safe)
        f = torch.ones_like(p) if mult is None else mult[..., cols]
        l = l + ((p * f) if norm_dropped else p).sum(-1, keepdim=True)
        acc = acc + _bf(p * f) @ v[:, cols]
    o = _bf(acc * torch.where(l > 0, 1.0 / l, torch.zeros_like(l)))
    lse = (m + torch.log2(l)) * torch.tensor(math.log(2.0), dtype=torch.float32)
    return o, lse[..., 0]


def emu_bwd(q, k, v, o, do, lse, dead, mult, lse_as_log2=False, dv_undropped=False, dq_mult=None, d_neighbour=False, dk_neighbour_head=False):
    """attention_bwd_{prep, kv, q}_kernel in fp32 -> bf16 (dq, dk, dv)"""
    sc2 = torch.tensor(SCALE, dtype=torch.float32) * torch.tensor(LOG2E, dtype=torch.float32)
    lse_log2 = lse if lse_as_log2 else lse * torch.tensor(LOG2E, dtype=torch.float32)
    bias = torch.where(dead, torch.tensor(-math.inf), torch.tensor(0.0))
    p = torch.exp2(q @ k.transpose(-1, -2) * sc2 + bias - lse_log2[..., None])
    g = do @ v.transpose(-1, -2)
    d = (do * o).sum(-1, keepdim=True)
    if d_neighbour:
        d = d.view(H, LQ // 2, 2, 1).flip(2).reshape(H, LQ, 1)

    def tiles(f):
        f = torch.ones_like(p) if f is None else f
        return _bf(p * f), _bf(p * (g * f - d) * SCALE)

    pt, ds = tiles(mult)
    if dv_undropped:
        pt = _bf(p)
    dv = _bf(pt.transpose(-1, -2) @ do)
    dk = _bf(ds.transpose(-1, -2) @ (q.flip(0) if dk_neighbour_head else q))
    dq = _bf((tiles(dq_mult)[1] if dq_mult is not None else ds) @ k)
    return dict(dq=dq, dk=dk, dv=dv)


def _fwd_ratio(p, **defect):
    q, k, v, _, dead = _inputs()
    mult = _mult(p)
    o, lse = emu_fwd(q, k, v, dead, mult, **defect)
    ro, bo, rl, bl = attn_fwd_ref(q.double(), k.double(), v.double(), dead, SCALE, None if mult is None else mult.double())
    return max(excess(o, ro, bo), excess(lse, rl, bl))


def _bwd_ratio(p, **defect):
    q, k, v, do, dead = _inputs()
    mult = _mult(p)
    o, lse = emu_fwd(q, k, v, dead, mult)
    got = emu_bwd(q, k, v, o, do, lse, dead, mult, **defect)
    refs = attn_bwd_ref(q.double(), k.double(), v.double(), o.double(), do.double(), lse.double(), dead, SCALE, None if mult is None else mult.double())
    return max(excess(got[n], r, b) for n, (r, b) in refs.items())


def _ln_ratio(unbiased=False):
    """rstd of the two-pass fp32 LayerNorm statistics (or with the unbiased variance) against the rstd bound, over rows with |mean| >> std,
    ordinary rows and rows of variance below eps"""
    g = torch.Generator().manual_seed(8)
    x = torch.randn(96, 256, generator=g) * 2 + 0.5
    x[1::4] = torch.randn(24, 256, generator=g) * 1.5 + torch.rand(24, 1, generator=g) * 136 + 64
    x[2::8] = 0.25 + torch.randn(12, 256, generator=g) * 2.0 ** -9
    x = _bf(x)
    eps = float(torch.tensor(1e-5, dtype=torch.float32))
    mean = x.sum(-1, keepdim=True) * (1.0 / 256)
    var = ((x - mean) ** 2).sum(-1, keepdim=True) / (255.0 if unbiased else 256.0)
    rstd = torch.rsqrt(var + eps)[:, 0]
    xd = x.double()
    _, _, rm, bm, rr, br = ln_ref(xd, torch.ones(256, dtype=torch.float64), torch.zeros(256, dtype=torch.float64), eps)
    return max(excess(mean[:, 0], rm, bm), excess(rstd, rr, br))


GOOD = {"forward p=0": lambda: _fwd_ratio(0.0), "forward p=0.1": lambda: _fwd_ratio(P), "backward p=0": lambda: _bwd_ratio(0.0),
        "backward p=0.1": lambda: _bwd_ratio(P), "LayerNorm statistics": lambda: _ln_ratio()}
DEFECTS = {
    "last partial key tile dropped": lambda: _fwd_ratio(0.0, drop_last_tile=True),
    "mask ignored for key 200 (middle tile)": lambda: _fwd_ratio(0.0, unmask_key=200),
    "normaliser from the dropped probabilities": lambda: _fwd_ratio(P, norm_dropped=True),
    "lse (natural log) read as log2": lambda: _bwd_ratio(0.0, lse_as_log2=True),
    "dV from the undropped P": lambda: _bwd_ratio(P, dv_undropped=True),
    "dQ kernel's dropout column base one tile off": lambda: _bwd_ratio(P, dq_mult=_mult(P, TILE)),
    "D from the neighbouring query row": lambda: _bwd_ratio(0.0, d_neighbour=True),
    "dK from the neighbouring head's q": lambda: _bwd_ratio(0.0, dk_neighbour_head=True),
    "LayerNorm with the unbiased variance": lambda: _ln_ratio(unbiased=True),
}


@pytest.mark.parametrize("case", list(GOOD))
def test_emulation_is_accepted(case):
    r = GOOD[case]()
    assert r <= 1.0, f"{case}: the fp32 / bf16 emulation of the kernel exceeds the bound ({r:.3g})"
    assert r > 1e-4, f"{case}: the bound is {1 / r:.3g} times wider than the error of the emulation"


@pytest.mark.parametrize("defect", list(DEFECTS))
def test_defect_is_rejected(defect):
    r = DEFECTS[defect]()
    FACTOR[defect] = r
    assert r > CLEAR, f"the bound accepts a result with this defect: {defect}, or rejects it by only {r:.3g}x"


@pytest.fixture(scope="module", autouse=True)
def _report_factors():
    yield
    if FACTOR:
        print("\nworst err / bound of each defect: " + "; ".join(f"{k}: {v:.3g}" for k, v in sorted(FACTOR.items())))
