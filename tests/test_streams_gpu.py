"""Stream ordering of `YOLOX.prefetch` and bit-reproducibility of the training step's fixed-order sums.

The prefetch tests stage each hazard deterministically: a bounded `torch.cuda._sleep` holds one stream back, so that a missing wait or a
missing `record_stream` lets the other stream read or write the wrong bytes every time, not by luck.  Each test uses a plan shape
(batch, H, W) that no other test here uses, so the plan's alternate buffers are created inside the test.  A sleep is at most 1e8 cycles:
about 50 ms at the H100's 1.98 GHz, under 100 ms at any SM clock above 1 GHz.
"""
import ctypes
import types

import pytest
import torch

from oracle import yolox_oracle as orc

pytestmark = pytest.mark.gpu

SHORT = 40_000_000   # cycles: ~20 ms at 1.98 GHz
LONG = 100_000_000   # cycles: ~50 ms at 1.98 GHz


@pytest.fixture(scope="module")
def model(cuda):
    import bench
    from yolov7_d2_b200.modeling import YOLOX

    m = YOLOX(bench.yolox_s_cfg("cuda"))
    m.load_state_dict(orc.yolox_state_dict(4), strict=True)
    m.train()
    return m


def _loss(m, batch):
    with torch.no_grad():
        return m(batch)["total_loss"].clone()


def _reference(m, batch):
    """loss and staged buffers of forward(batch) without prefetch (the copies run on the current stream, in order)"""
    loss = _loss(m, batch)
    eng = m._plan_for(batch)[0]
    torch.cuda.synchronize()
    return loss, eng.labels.clone(), eng.hw_valid.clone()


def _assert_staged(m, batch_images, loss, ref):
    ref_loss, ref_labels, ref_hw = ref
    eng = m._plan(batch_images.shape[0], batch_images.shape[2], batch_images.shape[3])
    torch.cuda.synchronize()
    assert torch.equal(eng.images_u8.cpu(), batch_images), "images_u8 differs from the batch"
    assert torch.equal(eng.labels, ref_labels), "labels differ from the batch's ground truth"
    assert torch.equal(eng.hw_valid, ref_hw), "hw_valid differs from the batch's image sizes"
    assert torch.equal(loss, ref_loss), (float(loss), float(ref_loss))


def test_prefetch_alternate_buffers_wait_for_the_current_stream(model):
    """The alternate buffers are allocated on the current stream.  The caching allocator hands them a block that the current stream has
    freed while work queued on it still writes that block; the copy stream must not fill them before that work has run."""
    import bench

    m = model
    images, labels = orc.synthetic_batch(2, 192, 81, max_gt=4)
    batch = bench.batched_inputs_from(images, labels)
    ref = _reference(m, batch)
    eng = m._plan_for(batch)[0]
    assert getattr(eng, "_alt", None) is None
    torch.cuda.synchronize()
    t = torch.empty(eng.images_u8.numel(), dtype=torch.uint8, device=eng.images_u8.device)
    t_ptr = t.data_ptr()
    torch.cuda._sleep(LONG)
    t.fill_(0xA5)           # still queued when prefetch() starts its copies
    del t                   # the block goes back to the current stream's pool at once: its pending fill is ordered on that stream
    m.prefetch(batch)
    # alloc(s), free, alloc(s) with nothing in between returns the same block: the hazard is staged, not hoped for
    assert eng._alt[0].data_ptr() == t_ptr, "the allocator did not reuse the freed block: the test stages nothing"
    loss = _loss(m, batch)
    _assert_staged(m, images, loss, ref)


def _device_batch(host_batch, fill_img=0, fill_box=-1.0):
    """the same batch with images and ground truth in fresh CUDA tensors that hold wrong values until _write_device_batch runs"""
    import bench

    imgs = [torch.full_like(x["image"], fill_img, device="cuda") for x in host_batch]
    boxes = [torch.full_like(x["instances"].gt_boxes.tensor, fill_box, device="cuda") for x in host_batch]
    classes = [torch.full_like(x["instances"].gt_classes, 7, device="cuda") for x in host_batch]
    batch = [{"image": i, "instances": types.SimpleNamespace(gt_boxes=bench._GtBoxes(b), gt_classes=c), "height": 640, "width": 640}
             for i, b, c in zip(imgs, boxes, classes)]
    src = [(x["image"].cuda(), x["instances"].gt_boxes.tensor.cuda(), x["instances"].gt_classes.cuda()) for x in host_batch]
    return batch, imgs + boxes + classes, src


def _write_device_batch(batch, src):
    for x, (i, b, c) in zip(batch, src):
        x["image"].copy_(i)
        x["instances"].gt_boxes.tensor.copy_(b)
        x["instances"].gt_classes.copy_(c)


def _drop_and_overwrite(batch, owned):
    """the caller lets go of its device tensors as soon as prefetch() returns and reuses the memory on its own stream"""
    specs = [(t.shape, t.dtype) for t in owned]
    for x in batch:
        x["image"] = torch.empty(x["image"].shape, dtype=torch.uint8)  # host placeholder: forward() reads only the shape
        del x["instances"]                                             # a prefetched batch is not staged again
    owned.clear()
    junk = [torch.empty(s, dtype=d, device="cuda") for s, d in specs]
    for j in junk:
        j.fill_(0x5A if j.dtype == torch.uint8 else 3)
    return junk


def _warm(m, host_batch):
    """reference forward without prefetch, then one prefetched step on device inputs that are ready: creates the plan, its alternate buffers
    and the copy stream, and leaves the copy stream's memory pool holding the temporaries that staging device inputs allocates.  Otherwise
    the staging under test would call cudaMalloc, which can synchronize the device and so hide a missing wait."""
    ref = _reference(m, host_batch)
    batch, owned, src = _device_batch(host_batch)
    _write_device_batch(batch, src)
    torch.cuda.synchronize()
    m.prefetch(batch)
    _loss(m, batch)
    torch.cuda.synchronize()
    return ref


def test_prefetch_reads_device_inputs_after_the_current_stream(model):
    """Images and gt_boxes produced on the current stream, behind a sleep, and handed to prefetch() right away: the copy stream must
    wait for the current stream before it reads them."""
    import bench

    m = model
    images, labels = orc.synthetic_batch(3, 96, 82, max_gt=4)
    host = bench.batched_inputs_from(images, labels)
    ref = _warm(m, host)
    batch, owned, src = _device_batch(host)
    torch.cuda.synchronize()
    torch.cuda._sleep(SHORT)
    _write_device_batch(batch, src)
    m.prefetch(batch)
    junk = _drop_and_overwrite(batch, owned)
    loss = _loss(m, batch)
    del junk
    _assert_staged(m, images, loss, ref)


def test_prefetch_keeps_dropped_device_inputs_alive(model):
    """The copy stream is held back past the caller's later work: after prefetch() returns the caller drops its device tensors and writes
    new ones of the same sizes on its own stream.  `record_stream` must keep the dropped memory from being handed out until the copy stream
    has read it."""
    import bench

    m = model
    images, labels = orc.synthetic_batch(2, 224, 83, max_gt=4)
    host = bench.batched_inputs_from(images, labels)
    ref = _warm(m, host)
    batch, owned, src = _device_batch(host)
    torch.cuda.synchronize()
    with torch.cuda.stream(m._copy_stream):
        torch.cuda._sleep(LONG)
    torch.cuda._sleep(SHORT)
    _write_device_batch(batch, src)
    m.prefetch(batch)
    junk = _drop_and_overwrite(batch, owned)   # runs on the current stream while the copy stream still sleeps
    loss = _loss(m, batch)
    del junk
    _assert_staged(m, images, loss, ref)


@pytest.mark.parametrize("hw", [20, 13])
def test_spp_pool_bwd_tiled_is_bit_reproducible(cuda, hw):
    """The shared-memory SPP backward adds the gradients routed to each input in a fixed order (branch 5, 9, 13, then source pixel): two
    runs give the same bytes.  Tie-heavy inputs route many gradients to one position, where an unordered sum would show."""
    from yolov7_d2_b200 import capi

    L = capi.lib()
    n, c = 4, 64
    g = torch.Generator().manual_seed(11)
    x = (torch.round(torch.randn(n, c, hw, hw, generator=g) * 2) / 2).to(torch.bfloat16)
    x[0, :16] = 0.0
    cat = torch.zeros(n, hw, hw, 4 * c, dtype=torch.bfloat16, device=cuda)
    cat[..., :c] = x.permute(0, 2, 3, 1).to(cuda)
    arg = torch.empty(3, n, hw, hw, c, dtype=torch.uint8, device=cuda)
    v = [capi.act(cat, i * c, c) for i in range(4)]
    capi.check(L.yb200_spp_pool(ctypes.byref(v[0]), ctypes.byref(v[1]), ctypes.byref(v[2]), ctypes.byref(v[3]), capi.ptr(arg), capi.stream_ptr()),
               "spp_pool")
    dcat = (torch.randn(n, hw, hw, 4 * c, generator=g) * torch.rand(n, hw, hw, 4 * c, generator=g).pow(4) * 100).to(torch.bfloat16).to(cuda)
    d = [capi.act(dcat, i * c, c) for i in range(4)]
    scratch = torch.empty(n * hw * hw * c, dtype=torch.float32, device=cuda)
    outs = []
    for _ in range(2):
        dx = torch.empty(n, hw, hw, c, dtype=torch.bfloat16, device=cuda)
        capi.check(L.yb200_spp_pool_bwd(ctypes.byref(d[0]), ctypes.byref(d[1]), ctypes.byref(d[2]), ctypes.byref(d[3]), capi.ptr(arg), capi.ptr(scratch),
                                        ctypes.byref(capi.act(dx)), capi.stream_ptr()), "spp_pool_bwd")
        outs.append(dx)
    torch.cuda.synchronize()
    assert torch.equal(outs[0].view(torch.int16), outs[1].view(torch.int16))
