"""The meta-architectures' input batching (SparseInst.preprocess_inputs, Detr.preprocess_image): normalise every image and zero-pad the batch
in one `yb200_normalize_pad` launch, bit-identical to torch's `(image - pixel_mean) / pixel_std` followed by `ImageList.from_tensors`."""
import numpy as np
import torch

from . import capi


def pinned_to(arr, device):
    return torch.from_numpy(np.ascontiguousarray(arr)).pin_memory().to(device, non_blocking=True)


def normalize_pad(L, imgs, pixel_mean, pixel_std, size_divisibility, who):
    """L: the loaded library (capi.lib()).  images [3, H, W] uint8 or fp32 (any device) -> fp32 [B, 3, Hp, Wp] on the device of `pixel_mean`
    ([3, 1, 1]), padded to the batch maximum rounded up to a multiple of `size_divisibility` (0: no rounding), and the images' (h, w).  One
    copy per image into one staging buffer, then one launch."""
    if not imgs:
        raise capi.Yb200Error(f"{who}: empty batch")
    for i, im in enumerate(imgs):
        if im.dim() != 3 or im.shape[0] != 3 or im.dtype not in (torch.uint8, torch.float32) or im.numel() == 0:
            raise capi.Yb200Error(f"{who}: image {i} is {tuple(im.shape)} {im.dtype} (expected [3, H, W] uint8 or float32)")
    device = pixel_mean.device
    is_f32 = any(im.dtype == torch.float32 for im in imgs)
    dtype = torch.float32 if is_f32 else torch.uint8
    sizes = [(int(im.shape[1]), int(im.shape[2])) for im in imgs]
    s = max(int(size_divisibility), 1)
    hp = (max(h for h, _ in sizes) + s - 1) // s * s
    wp = (max(w for _, w in sizes) + s - 1) // s * s
    counts = [im.numel() for im in imgs]
    offs = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    staged = torch.empty(int(offs[-1]), dtype=dtype, device=device)
    for im, o, n in zip(imgs, offs, counts):
        staged[int(o):int(o) + n].copy_(im.reshape(-1), non_blocking=True)  # one copy per image; uint8 -> fp32 is exact
    table = pinned_to(np.array([(o, h, w) for o, (h, w) in zip(offs[:-1], sizes)], dtype=np.int64), device)
    out = torch.empty(len(imgs), 3, hp, wp, device=device)
    capi.check(L.yb200_normalize_pad(capi.ptr(staged), int(is_f32), capi.ptr(table), len(imgs), capi.ptr(pixel_mean), capi.ptr(pixel_std), hp,
                                              wp, capi.ptr(out), capi.stream_ptr()), "normalize_pad")
    return out, sizes
