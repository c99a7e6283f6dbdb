"""Negative controls for the error bound of tests/test_convnext_plan_gpu.py, on the CPU.

For small instances of each case class, the result a correct kernel could return -- the operation computed in fp32 on the same bf16
operands, then rounded to the storage type -- must pass the bound, and the same computation with one known defect must fail it: a dropped
16-channel k-block, a dropped 3x3 tap, a dropped last partial column tile, a weight-gradient split counted twice, a border pixel read one
pixel off.  This shows that the GPU tests' bound is tight enough to see a subtly wrong kernel.
"""
import pytest
import torch

from test_convnext_plan_gpu import R_BF16, R_F16, bound, conv_ref, dgrad_ref, dw7_ref, dw7_wgrad_ref, excess, wgrad_ref


def _bf(*shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(torch.bfloat16).double()


def _border(t):
    """the last column of the map read one pixel off: it holds its neighbour's values"""
    t = t.clone()
    t[:, :, -1] = t[:, :, -2]
    return t


N, H, W = 2, 12, 12


def _fwd():
    """forward, fp16 z: cin 48 (16-channel k-blocks), cout 192 (a full and a partial 128-wide column tile)"""
    x, w = _bf(N, H, W, 48, seed=1), _bf(192, 48, 3, 3, seed=2, scale=432 ** -0.5)
    ref, mag, k = conv_ref(x, w, 3, 1)
    run = lambda x, w: conv_ref(x.float(), w.float(), 3, 1)[0].half().double()

    def kblock():
        w2 = w.clone()
        w2[:, 16:32, 1, 1] = 0
        return run(x, w2)

    def tap():
        w2 = w.clone()
        w2[:, :, 0, 2] = 0
        return run(x, w2)

    def coltile():
        z = run(x, w)
        z[..., 128:] = 0
        return z

    return ref, bound(ref, mag, k, R_F16), run(x, w), dict(kblock=kblock, tap=tap, coltile=coltile, border=lambda: run(_border(x), w))


def _dgrad():
    """data gradient, bf16 dx: dz 48 channels (16-channel k-blocks), dx 192 (a partial second column tile)"""
    dz, w = _bf(N, H, W, 48, seed=3), _bf(48, 192, 3, 3, seed=4, scale=1728 ** -0.5)
    shape = (N, H, W, 192)
    ref, mag, k = dgrad_ref(dz, w, 3, 1, shape)
    run = lambda dz, w: dgrad_ref(dz.float(), w.float(), 3, 1, shape)[0].bfloat16().double()

    def kblock():
        w2 = w.clone()
        w2[16:32, :, 1, 1] = 0
        return run(dz, w2)

    def tap():
        w2 = w.clone()
        w2[:, :, 2, 1] = 0
        return run(dz, w2)

    def coltile():
        dx = run(dz, w)
        dx[..., 128:] = 0
        return dx

    return ref, bound(ref, mag, k, R_BF16), run(dz, w), dict(kblock=kblock, tap=tap, coltile=coltile, border=lambda: run(_border(dz), w))


def _wgrad():
    """weight gradient, fp32: K = pixels in blocks of 64 (kWgPix), cin 48 in 16-wide tiles, split-K over the pixel range"""
    x, dz = _bf(N, H, W, 48, seed=5), _bf(N, H, W, 96, seed=6)
    ref, mag, k = wgrad_ref(x, dz, 3, 1)
    run = lambda x, dz: wgrad_ref(x.float(), dz.float(), 3, 1)[0].double()

    def pixels(lo, hi):
        d = torch.zeros_like(dz).view(-1, 96)
        d[lo:hi] = dz.view(-1, 96)[lo:hi]
        return d.view(dz.shape)

    def kblock():
        return run(x, dz - pixels(64, 128))

    def tap():
        g = run(x, dz)
        g[:, :, 1, 0] = 0
        return g

    def coltile():
        g = run(x, dz)
        g[:, 32:] = 0
        return g

    def split_twice():
        return run(x, dz) + run(x, pixels(96, 192))

    return ref, bound(ref, mag, k, 0.0), run(x, dz), dict(kblock=kblock, tap=tap, coltile=coltile, split_twice=split_twice,
                                                          border=lambda: run(_border(x), dz))


def _dwconv7():
    """depthwise 7x7, bf16 out: channels in 32-wide slices"""
    x, w = _bf(N, H, W, 96, seed=7), torch.randn(96, 7, 7, generator=torch.Generator().manual_seed(8)).double() * 0.15
    ref, mag, k = dw7_ref(x, w, 0)
    run = lambda x, w: dw7_ref(x.float(), w.float(), 0)[0].bfloat16().double()

    def tap():
        w2 = w.clone()
        w2[:, 3, 4] = 0
        return run(x, w2)

    def coltile():
        o = run(x, w)
        o[..., 64:] = 0
        return o

    return ref, bound(ref, mag, k, R_BF16), run(x, w), dict(tap=tap, coltile=coltile, border=lambda: run(_border(x), w))


def _dwconv7_wgrad():
    """depthwise weight gradient, fp32: per-CTA partial sums over pixel ranges, reduced afterwards"""
    x, dy = _bf(N, H, W, 64, seed=9), _bf(N, H, W, 64, seed=10)
    ref, mag, k = dw7_wgrad_ref(x, dy)
    run = lambda x, dy: dw7_wgrad_ref(x.float(), dy.float())[0].double()
    half = dy.clone()
    half[1:] = 0

    def tap():
        g = run(x, dy)
        g[:, 0, 6] = 0
        return g

    return ref, bound(ref, mag, k, 0.0), run(x, dy), dict(tap=tap, split_twice=lambda: run(x, dy) + run(x, half), border=lambda: run(_border(x), dy))


CLASSES = dict(fwd=_fwd, dgrad=_dgrad, wgrad=_wgrad, dwconv7=_dwconv7, dwconv7_wgrad=_dwconv7_wgrad)
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
    assert r > 1.0, f"{cls}: the bound accepts a result with {defect} (worst err / bound {r:.3g})"
