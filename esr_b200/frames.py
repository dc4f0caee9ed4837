"""The recordings' image frames as the dataset formats them (H5Dataset.__getitem__'s gt_img, gt_inp_size_img and frame,
dataloader/h5dataset.py:297-315), on the GPU.

The reference reads `ori_images/image%09d`, flips it as augment_frame does (h5dataset.py:672-685), resizes it with
cv2.resize(..., interpolation=cv2.INTER_CUBIC) and divides by 255 (base_dataset.py:36-38), on the host, twice per item.
Here the image blocks stay in their files (numpy memmaps: the page cache holds what is read); per batch the distinct frames
the batch reads are copied once, through pinned staging, into HBM, and one esr_resize_frames_cubic launch makes every
entry of the batch at both target sizes.  A recording's frames are never made resident as a whole: a 720 x 1280 x 3 frame
is 2.76 MB, so a recording of a few thousand frames holds gigabytes.
"""
import numpy as np
import torch

from . import _lib

# struct esr_frame_resize_desc and esr_frame_resize_u8_desc of include/esr_b200.h
_DESC = np.dtype([("src", np.uint64), ("out0", np.uint64), ("out1", np.uint64), ("flips", np.int32), ("pad", np.int32)])
_DESC_U8 = np.dtype([("src", np.uint64), ("out", np.uint64), ("flips", np.int32), ("pad", np.int32)])
_MAX_LAUNCH = 65535                                     # frames per launch (gridDim.y)


def resize_frames(src, flips, out0, out1, shape, size0, size1, dev):
    """Frame i = uint8 image at address src[i] of `shape` (H, W, C), mirrored by flips[i] (bit 0 horizontal, bit 1
    vertical), resized to size0 into fp32 address out0[i] and, where out1[i] != 0, to size1 into out1[i].  All on `dev`."""
    n = len(src)
    if n == 0:
        return
    d = np.zeros(n, _DESC)
    d["src"], d["out0"], d["out1"], d["flips"] = src, out0, out1, np.asarray(flips, np.int32) & 3
    H, W, C = shape
    desc = torch.from_numpy(d.view(np.uint8)).to(dev)
    with torch.cuda.device(dev):
        for s in range(0, n, _MAX_LAUNCH):
            k = min(_MAX_LAUNCH, n - s)
            _lib.check(_lib.lib().esr_resize_frames_cubic(_lib.ptr(desc[s * _DESC.itemsize:]), k, H, W, C, size0[0], size0[1],
                                                          size1[0], size1[1], _lib.stream_ptr()), "esr_resize_frames_cubic")


def resize_frames_u8(src, flips, out, shape, size, dev):
    """Frame i = uint8 image at address src[i] of `shape` (H, W, C), mirrored by flips[i], resized to `size` into the uint8
    address out[i]: cv2.resize's own levels, the value resize_frames divides by 255.  All on `dev`."""
    n = len(src)
    if n == 0:
        return
    d = np.zeros(n, _DESC_U8)
    d["src"], d["out"], d["flips"] = src, out, np.asarray(flips, np.int32) & 3
    H, W, C = shape
    desc = torch.from_numpy(d.view(np.uint8)).to(dev)
    with torch.cuda.device(dev):
        for s in range(0, n, _MAX_LAUNCH):
            k = min(_MAX_LAUNCH, n - s)
            _lib.check(_lib.lib().esr_resize_frames_cubic_u8(_lib.ptr(desc[s * _DESC_U8.itemsize:]), k, H, W, C, size[0], size[1],
                                                             _lib.stream_ptr()), "esr_resize_frames_cubic_u8")


def gt_images_u8(requests, n, gt_res, dev):
    """The uint8 gt_img of n window positions, unflipped: requests as stage_frames takes them (images, image index,
    positions) -> uint8 CUDA tensor [n, H, W(, 3)] at gt_res, one launch."""
    staged, addr = stage_frames(requests, n, dev)
    shape = staged.shape[1:]
    C = shape[2] if len(shape) == 3 else 1
    out = torch.empty((n, *gt_res) + ((3,) if C == 3 else ()), dtype=torch.uint8, device=dev)
    rows = np.uint64(out.data_ptr()) + np.arange(n, dtype=np.uint64) * np.uint64(out[0].numel())
    resize_frames_u8(addr, np.zeros(n, np.int32), rows, (shape[0], shape[1], C), tuple(gt_res), dev)
    return out, staged


def stage_frames(requests, n, dev):
    """Copy the distinct frames that `requests` read into HBM, once each.
    requests: [(images [N, H, W(, 3)] uint8 array or memmap, index int64 [k], positions int64 [k])]; every position in [0, n)
    -> (the staged uint8 HBM tensor, which must outlive the launch reading it; uint64 [n] device address of each position)."""
    shape = requests[0][0].shape[1:]
    uniq, inv = [], []
    for images, index, _ in requests:
        if images.shape[1:] != shape:
            raise _lib.ESRError(f"a batch mixes image shapes {tuple(shape)} and {tuple(images.shape[1:])}")
        index = np.asarray(index, np.int64)
        if index.size and (index.min() < 0 or index.max() >= len(images)):
            raise _lib.ESRError(f"image index out of range [0, {len(images)})")
        u, i = np.unique(index, return_inverse=True)
        uniq.append(u)
        inv.append(i)
    total = sum(len(u) for u in uniq)
    host = torch.empty((total, *shape), dtype=torch.uint8, pin_memory=True)
    h = host.numpy()
    base, addr = 0, np.zeros(n, np.uint64)
    frame_bytes = int(np.prod(shape))
    bases = []
    for (images, _, _), u in zip(requests, uniq):
        np.take(images, u, axis=0, out=h[base:base + len(u)])
        bases.append(base)
        base += len(u)
    staged = host.to(dev, non_blocking=True)
    for (_, _, pos), b, i in zip(requests, bases, inv):
        addr[np.asarray(pos, np.int64)] = np.uint64(staged.data_ptr()) + (np.uint64(b) + i.astype(np.uint64)) * np.uint64(frame_bytes)
    return staged, addr


def frame_bank(B, L, res, C, dev):
    """An empty fp32 bank [B, L, 1, H, W(, 3)] (frame_formatting's [1, H, W(, 3)] per frame)."""
    return torch.empty((B, L, 1, *res) + ((3,) if C == 3 else ()), dtype=torch.float32, device=dev)


def row_addresses(out):
    """Addresses of the rows of a contiguous fp32 CUDA tensor [F, ...] (one formatted frame per row)."""
    assert out.is_contiguous() and out.dtype == torch.float32 and out.is_cuda
    return np.uint64(out.data_ptr()) + np.arange(out.shape[0], dtype=np.uint64) * np.uint64(out[0].numel() * 4)


def batch_frames(gt, frame, flips, B, L, inp_res, gt_res, dev):
    """The image entries of a batch of B sequences of L frames (B * L frame positions, sequence-major).
    gt / frame: None or [(images, index, positions)] as stage_frames takes them: the ground-truth image of every position
    -> 'gt_img' at gt_res and 'gt_inp_size_img' at inp_res; the frame-mode image -> 'frame' at gt_res.
    flips: int32 [B * L] (bit 0 horizontal, bit 1 vertical).  -> {name: fp32 bank [B, L, 1, ., .(, 3)]}."""
    F = B * L
    reqs = (gt or []) + [(im, ix, np.asarray(pos, np.int64) + F) for im, ix, pos in (frame or [])]
    if not reqs:
        return {}
    staged, addr = stage_frames(reqs, 2 * F, dev)
    shape = staged.shape[1:]
    C = shape[2] if len(shape) == 3 else 1
    bank, src, out0, out1, fl = {}, [], [], [], []
    if gt:
        bank["gt_img"] = frame_bank(B, L, gt_res, C, dev)
        bank["gt_inp_size_img"] = frame_bank(B, L, inp_res, C, dev)
        src.append(addr[:F])
        out0.append(row_addresses(bank["gt_img"].view(F, -1)))
        out1.append(row_addresses(bank["gt_inp_size_img"].view(F, -1)))
        fl.append(flips)
    if frame:
        bank["frame"] = frame_bank(B, L, gt_res, C, dev)
        src.append(addr[F:])
        out0.append(row_addresses(bank["frame"].view(F, -1)))
        out1.append(np.zeros(F, np.uint64))
        fl.append(flips)
    resize_frames(np.concatenate(src), np.concatenate(fl), np.concatenate(out0), np.concatenate(out1), (shape[0], shape[1], C),
                  tuple(gt_res), tuple(inp_res), dev)
    return bank
