"""Why tests/test_headline_plan_gpu.py probes the pixel-long sums with exact integers, on the CPU, at the 64 x 640 x 640 plan's K.

A weight gradient of the stem sums K = 64 * 320 * 320 = 6.5 M products.  Emulated the way the kernel adds them (fp32 sums of 64-pixel
blocks, fp32 partials per split, the splits added in fp32), the correct result passes the random-operand bound of
tests/test_convnext_plan_gpu.py -- and so does the same sum with one 64-pixel block dropped or one split counted twice.  On {0, 1}
operands the same emulation is exact, and both defects miss the exact count.  Likewise a BatchNorm statistic over 6.5 M pixels: fp32
per 128-pixel tile, fp32 over a CTA's walk of tiles, fp64 across CTAs; one dropped tile passes the statistics bound of
tests/test_train_bn_gpu.py but not the exact-integer probe.
"""
import pytest
import torch

from test_convnext_plan_gpu import U, bound, excess

K = 64 * 320 * 320
BLOCK, SPLITS = 64, 264           # the weight gradient's pixel block; the split count of the plan's 160 x 160 1x1 layers on 132 SMs
TILE, WALK = 128, 97              # the statistics' pixel tile; tiles per CTA of the stem's forward on 132 SMs


def _wgrad_fp32(x, d, defect=None):
    """fp32 sums of every block, fp32 sum of each split's blocks, fp32 sum of the splits; x [K, c], d [K]"""
    prod = (x * d[:, None]).float()
    blocks = prod.view(-1, BLOCK, x.shape[1]).sum(1)
    if defect == "drop_block":
        blocks[1000] = 0
    per = -(-blocks.shape[0] // SPLITS)
    parts = [blocks[i:i + per].sum(0) for i in range(0, blocks.shape[0], per)]
    if defect == "split_twice":
        parts.append(parts[3])
    out = torch.zeros(x.shape[1], dtype=torch.float32)
    for p in parts:
        out = out + p
    return out.double()


def _stat_fp32(z, defect=None):
    """fp32 per tile, fp32 over each CTA's walk of WALK tiles, fp64 across CTAs"""
    tiles = z.float().view(-1, TILE).sum(1)
    if defect == "drop_tile":
        tiles[777] = 0
    pad = -tiles.numel() % WALK
    walks = torch.cat([tiles, tiles.new_zeros(pad)]).view(-1, WALK).sum(1)
    return walks.double().sum()


def _random(seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(K, 4, generator=g).to(torch.bfloat16).double()
    d = torch.randn(K, generator=g).to(torch.bfloat16).double()
    return x, d


def _bits(seed, p, c=None):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(K, *([c] if c else []), generator=g) < p).double()


@pytest.mark.parametrize("defect", [None, "drop_block", "split_twice"])
def test_wgrad_random_bound_cannot_see_a_dropped_block_or_split(defect):
    x, d = _random(1)
    ref = (x * d[:, None]).sum(0)
    mag = (x.abs() * d.abs()[:, None]).sum(0)
    assert excess(_wgrad_fp32(x, d, defect), ref, bound(ref, mag, K, 0.0)) <= 1.0


@pytest.mark.parametrize("defect", [None, "drop_block", "split_twice"])
def test_wgrad_integer_probe_sees_them(defect):
    p = 0.35  # ~8 coincidences per output and block; each output ~0.8 M < 2^20
    x, d = _bits(2, p, 4), _bits(3, p)
    ref = (x * d[:, None]).sum(0)
    assert float(ref.max()) < 2 ** 20
    got = _wgrad_fp32(x, d, defect)
    assert torch.equal(got, ref) == (defect is None)


@pytest.mark.parametrize("defect", [None, "drop_tile"])
def test_stat_bound_cannot_see_a_dropped_tile(defect):
    g = torch.Generator().manual_seed(4)
    z = torch.randn(K, generator=g).to(torch.float16).double()
    ref = z.sum()
    for tiles in (WALK, K // TILE):  # the per-CTA walk, and every tile of the map
        k = 5 + tiles + 2
        assert float((_stat_fp32(z, defect) - ref).abs()) <= k * U * float(z.abs().sum())


@pytest.mark.parametrize("defect", [None, "drop_tile"])
def test_stat_integer_probe_sees_it(defect):
    g = torch.Generator().manual_seed(5)
    z = (torch.rand(K, 4, generator=g) < 0.02).double().sum(1)  # z in [0, 4], as four unit weights over {0, 1} activations give
    ref = z.sum()
    assert float((z * z).sum()) < 2 ** 20
    assert torch.equal(_stat_fp32(z, defect), ref) == (defect is None)
