"""Negative controls for the bounds of tests/test_sparseinst_kernels_gpu.py, on the CPU.

For small instances of each SparseInst case class, the result a correct kernel could return -- the operation computed in fp32 on the
same operands, then rounded to the storage type -- must pass the bound, and the same computation with one known defect must fail it by a
clear factor: image b using image b + 1's kernels (past the last image: the zeros TMA reads beyond the tensor), the last 64 kernel
columns (one BLOCK_K = 64 k-block of kernel_dim 128) dropped, the last 16-row slice of a 112-wide column tile dropped, one 128-pixel tile of
the pixel contraction or the column sums dropped or counted twice, the normaliser not clamped at 1e-6, the sigmoid read from the
neighbouring channel.  The factors are printed at the end of the module (-s).
"""
import pytest
import torch

from test_convnext_plan_gpu import R_BF16, bound, excess, wgrad_ref
from test_sparseinst_kernels_gpu import (BATCHED_ACCEPTED, BATCHED_REFUSED, CLAMP, batched_accepts, bmm_ref, choose_tile, colsum_ref, normalize_ref,
                                         sigmoid_ref)

FACTOR = {}  # case class - defect -> worst err / bound of the defective result
CLEAR = 4.0  # a defect must exceed the bound by at least this factor


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _bf(*shape, seed, scale=1.0):
    return (torch.randn(*shape, generator=_gen(seed)) * scale).to(torch.bfloat16).double()


N, H, W = 2, 8, 16  # 128 pixels per image: one pixel tile each


def _mask_gemm():
    """the batch's mask GEMM, fp32 NCHW: kernel dim 128 (two k-blocks of 64), 112 kernels per image (7 of the 8 16-row slices of a
    128-wide column tile); image b's kernels are scaled by 2^(12 b)"""
    x = _bf(N, H, W, 128, seed=1)
    w = _bf(N, 112, 128, seed=2, scale=128 ** -0.5) * torch.tensor([2.0 ** (12 * b) for b in range(N)]).double()[:, None, None]
    ref, mag, k = bmm_ref(x, w)
    run = lambda x, w: bmm_ref(x.float(), w.float())[0].double()

    def neighbour():
        w2 = torch.zeros_like(w)
        w2[:-1] = w[1:]
        return run(x, w2)

    def kblock():
        w2 = w.clone()
        w2[..., 64:] = 0
        return run(x, w2)

    def slice16():
        o = run(x, w)
        o[:, 96:112] = 0
        return o

    return ref, bound(ref, mag, k, 0.0), run(x, w), dict(neighbour=neighbour, kblock=kblock, slice16=slice16)


PIX = 16 * 24  # three 128-pixel tiles


def _probs(c, seed):
    return torch.sigmoid(_bf(1, 16, 24, c, seed=seed, scale=3.0)).to(torch.bfloat16).double()


def _tile(t, lo, hi):
    """t with every pixel outside [lo, hi) zeroed"""
    d = torch.zeros_like(t).view(-1, t.shape[-1])
    d[lo:hi] = t.reshape(-1, t.shape[-1])[lo:hi]
    return d.view(t.shape)


def _contraction():
    """raw = iam_prob^T features, fp32 [112][64]: the weight-gradient GEMM with K = pixels"""
    f, p = _bf(1, 16, 24, 64, seed=3), _probs(112, 4)
    ref, mag, k = wgrad_ref(f, p, 1, 1)
    run = lambda f, p: wgrad_ref(f.float(), p.float(), 1, 1)[0].double()
    return ref, bound(ref, mag, k, 0.0), run(f, p), dict(tile_dropped=lambda: run(f, p - _tile(p, 128, 256)),
                                                         tile_twice=lambda: run(f, p + _tile(p, 128, 256)))


def _colsum():
    """normaliser = column sums of the probabilities, fp32 [112], K = pixels"""
    p = _probs(112, 5)
    ref, mag, k = colsum_ref(p)
    run = lambda p: colsum_ref(p.float())[0].double()
    return ref, bound(ref, mag, k, 0.0), run(p), dict(tile_dropped=lambda: run(p - _tile(p, 256, 384)), tile_twice=lambda: run(p + _tile(p, 0, 128)))


def _normalize():
    """inst = raw / max(norm, 1e-6) -> bf16: real maps' normalisers and the padded maps' PIX * 9.4e-14 (clamped)"""
    raw = torch.randn(112, 64, generator=_gen(6)).float().double()
    norm = (torch.rand(112, generator=_gen(7)) * 100 + 0.01).float().double()
    norm[100:] = PIX * 9.4e-14
    norm[:4] = torch.tensor([0.5e-6, 0.999e-6, CLAMP, 1.001e-6]).double()
    ref, bnd = normalize_ref(raw, norm)
    run = lambda clamp: (raw.float() / norm.float().clamp_min(clamp)[:, None]).bfloat16().double()
    return ref, bnd, run(CLAMP), dict(unclamped=lambda: run(0.0))


def _sigmoid():
    """probabilities, bf16: logits N(0, 8^2) with the padded maps' -30 and +-90"""
    x = _bf(2, 8, 8, 112, seed=8, scale=8.0)
    x[0, 0, :3] = torch.tensor([-30.0, 90.0, -90.0]).double()[:, None]
    ref, bnd = sigmoid_ref(x)
    run = lambda x: torch.sigmoid(x.float()).bfloat16().double()
    return ref, bnd, run(x), dict(neighbour_channel=lambda: run(torch.roll(x, -1, -1)))


CLASSES = dict(mask_gemm=_mask_gemm, contraction=_contraction, colsum=_colsum, normalize=_normalize, sigmoid=_sigmoid)
CONTROLS = [(c, p) for c, f in CLASSES.items() for p in f()[3]]


@pytest.mark.parametrize("cls", list(CLASSES))
def test_correct_result_is_accepted(cls):
    ref, bnd, good, _ = CLASSES[cls]()
    r = excess(good, ref, bnd)
    assert r <= 1.0, f"{cls}: an fp32-computed, storage-rounded result exceeds the bound ({r:.3g})"
    assert r > 1e-3, f"{cls}: the bound is {1 / r:.3g} times wider than the error of a correct result"


@pytest.mark.parametrize("cls,defect", CONTROLS, ids=[f"{c}-{p}" for c, p in CONTROLS])
def test_defect_is_rejected(cls, defect):
    ref, bnd, _, defects = CLASSES[cls]()
    r = excess(defects[defect](), ref, bnd)
    FACTOR[f"{cls}-{defect}"] = r
    assert r > CLEAR, f"{cls}: the bound accepts a result with {defect}, or rejects it by only {r:.3g}x"


def test_choose_tile_predicts_batched_acceptance():
    """the batched mask GEMM runs where each 128-pixel tile holds one image: the default 640-pixel input's 80x80 map, 64x64, 72x96, 96x96,
    any map at batch 1, and maps like 1x65 whose tiles overhang the image; it is refused at 40x40, 12x20 and 60x80 (two images per tile)"""
    assert all(batched_accepts(*m) for m in BATCHED_ACCEPTED), [(m, choose_tile(*m)) for m in BATCHED_ACCEPTED]
    assert not any(batched_accepts(*m) for m in BATCHED_REFUSED), [(m, choose_tile(*m)) for m in BATCHED_REFUSED]
    assert choose_tile(2, 80, 80) == (4, 3) and choose_tile(2, 1, 65) == (7, 0) and choose_tile(2, 40, 40) == (3, 3)


@pytest.fixture(scope="module", autouse=True)
def _report_factors():
    yield
    if FACTOR:
        print("\nworst err / bound of each defect: " + "; ".join(f"{k}: {v:.3g}" for k, v in sorted(FACTOR.items())))
