"""GPU mirror of the reference's dataloader/encodings.py for the functions on the hot path.

Same names, positional arguments and side effects as the reference:
  events_to_image(xs, ys, ps, sensor_size)        encodings.py:243-268
  events_to_channels(xs, ys, ps, sensor_size)     encodings.py:289-304
  events_to_stack_no_polarity(xs, ys, ts, ps, B, device, sensor_size)   encodings.py:204-240 (+ :77-99)
  events_to_voxel(xs, ys, ts, ps, num_bins, sensor_size)                encodings.py:271-286
  events_to_mask(xs, ys, ps, sensor_size)                               encodings.py:307-331
  cython_event_redistribute(event_stack, mode)    encodings.py:466-484
  multiprocess_cython(event_stack, mode)          encodings.py:495-533 (per-sample calls, no process pool)
  stack2cnt(stack)                                encodings.py:652-670
plus the batched entry point the GPU pipeline uses:
  encode_frames(xs, ys, ps, frame_off, lr_size, hr_size)  -> [F,2,kH,kW] on the GPU, fusing the LR->HR lift of
                                                            dataloader/h5dataset.py:508-528.
CPU tensors are accepted (copied to the current CUDA device, result and in-place side effects copied back);
CUDA tensors are processed in place.  There is no CPU implementation here.
"""
import numpy as np
import torch

from . import _lib
from . import event_redistribute as c_event_redistribute  # noqa: F401  (the reference exposes its Cython module here, encodings.py:5)
from .expand import expand


def _dev():
    return torch.device("cuda", torch.cuda.current_device())


def _to_dev_f32(t, dev):
    """(device fp32 contiguous tensor, needs_copy_back)"""
    if t.is_cuda and t.dtype == torch.float32 and t.is_contiguous():
        return t, False
    return t.detach().to(device=dev, dtype=torch.float32).contiguous(), True


def events_to_image(xs, ys, ps, sensor_size=(180, 240)):
    """Accumulate events into an image (raw weights).  xs, ys, ps are modified in place like the reference."""
    dev = xs.device if xs.is_cuda else _dev()
    dx, cbx = _to_dev_f32(xs, dev)
    dy, cby = _to_dev_f32(ys, dev)
    dp, cbp = _to_dev_f32(ps, dev)
    H, W = int(sensor_size[0]), int(sensor_size[1])
    out = torch.empty((H, W), dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().esr_scatter_image(_lib.ptr(dx), _lib.ptr(dy), _lib.ptr(dp), dx.numel(), H, W, 1,
                                                _lib.ptr(out), _lib.stream_ptr()), "esr_scatter_image")
    for src, d, cb in ((xs, dx, cbx), (ys, dy, cby), (ps, dp, cbp)):
        if cb and src.dtype == torch.float32:
            src.copy_(d)
    return out if xs.is_cuda else out.cpu()


def events_to_mask(xs, ys, ps, sensor_size=(180, 240)):
    """Binary-style mask (encodings.py:307-331): mask[y,x] = |ps| of the last event on the pixel; xs, ys, ps are modified
    in place for out-of-range events like the reference."""
    dev = xs.device if xs.is_cuda else _dev()
    dx, cbx = _to_dev_f32(xs, dev)
    dy, cby = _to_dev_f32(ys, dev)
    dp, cbp = _to_dev_f32(ps, dev)
    H, W = int(sensor_size[0]), int(sensor_size[1])
    out = torch.empty((H, W), dtype=torch.float32, device=dev)
    tmp = torch.empty((H * W,), dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().esr_scatter_mask(_lib.ptr(dx), _lib.ptr(dy), _lib.ptr(dp), dx.numel(), H, W, 1, _lib.ptr(tmp),
                                               _lib.ptr(out), _lib.stream_ptr()), "esr_scatter_mask")
    for src, d, cb in ((xs, dx, cbx), (ys, dy, cby), (ps, dp, cbp)):
        if cb and src.dtype == torch.float32:
            src.copy_(d)
    return out if xs.is_cuda else out.cpu()


def events_to_stack_no_polarity(xs, ys, ts, ps, B, device=None, sensor_size=(180, 240)):
    """Signed per-time-bin event sums [B,H,W] (encodings.py:204-240).  Bin edges come from the reference's own binary
    search semantics (esr_time_bin_bounds); each bin is one events_to_image pass over its slice, so the slices of the
    caller's xs/ys/ps are modified in place exactly as in the reference."""
    dev = xs.device if xs.is_cuda else _dev()
    H, W = int(sensor_size[0]), int(sensor_size[1])
    n = len(ts)
    if n <= 3 or float(ts.sum()) == 0:
        z = torch.zeros([B, H, W], device=dev)
        return z if xs.is_cuda else z.cpu()
    assert len(xs) == len(ys) and len(ys) == len(ts) and len(ts) == len(ps)
    dx, cbx = _to_dev_f32(xs, dev)
    dy, cby = _to_dev_f32(ys, dev)
    dp, cbp = _to_dev_f32(ps, dev)
    dt, _ = _to_dev_f32(ts, dev)
    L = _lib.lib()
    bounds = torch.empty((B, 2), dtype=torch.int64, device=dev)
    out = torch.empty((B, H, W), dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        _lib.check(L.esr_time_bin_bounds(_lib.ptr(dt), n, int(B), _lib.ptr(bounds), _lib.stream_ptr()), "esr_time_bin_bounds")
        bh = bounds.cpu().tolist()
        for bi, (beg, end) in enumerate(bh):
            beg, end = max(0, min(beg, n)), max(0, min(end, n))          # python slice clamping
            cnt = max(0, end - beg)
            _lib.check(L.esr_scatter_image(_lib.ptr(dx[beg:]) if cnt else None, _lib.ptr(dy[beg:]) if cnt else None,
                                           _lib.ptr(dp[beg:]) if cnt else None, cnt, H, W, 1, _lib.ptr(out[bi]),
                                           _lib.stream_ptr()), "esr_scatter_image")
    for src, d, cb in ((xs, dx, cbx), (ys, dy, cby), (ps, dp, cbp)):
        if cb and src.dtype == torch.float32:
            src.copy_(d)
    return out if xs.is_cuda else out.cpu()


def events_to_voxel(xs, ys, ts, ps, num_bins, sensor_size=(180, 240)):
    """Voxel grid with temporal bilinear interpolation [num_bins,H,W] (encodings.py:271-286); xs, ys are modified in
    place for out-of-range events like the reference (and, like it, such events then land on pixel (0,0) of bins >= 1)."""
    assert len(xs) == len(ys) and len(ys) == len(ts) and len(ts) == len(ps)
    dev = xs.device if xs.is_cuda else _dev()
    dx, cbx = _to_dev_f32(xs, dev)
    dy, cby = _to_dev_f32(ys, dev)
    dp, _ = _to_dev_f32(ps, dev)
    dt, _ = _to_dev_f32(ts, dev)
    H, W = int(sensor_size[0]), int(sensor_size[1])
    out = torch.empty((int(num_bins), H, W), dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().esr_scatter_voxel(_lib.ptr(dx), _lib.ptr(dy), _lib.ptr(dt), _lib.ptr(dp), dx.numel(), int(num_bins),
                                                H, W, 1, _lib.ptr(out), _lib.stream_ptr()), "esr_scatter_voxel")
    if cbx and xs.dtype == torch.float32:
        xs.copy_(dx)
    if cby and ys.dtype == torch.float32:
        ys.copy_(dy)
    return out if xs.is_cuda else out.cpu()


def events_to_channels(xs, ys, ps, sensor_size=(180, 240)):
    """Two-channel event count image [2,H,W] (0: positive, 1: negative).  xs, ys are modified in place
    (out-of-range coordinates -> 0) exactly as the reference does."""
    assert len(xs) == len(ys) and len(ys) == len(ps)
    dev = xs.device if xs.is_cuda else _dev()
    dx, cbx = _to_dev_f32(xs, dev)
    dy, cby = _to_dev_f32(ys, dev)
    dp, _ = _to_dev_f32(ps, dev)
    H, W = int(sensor_size[0]), int(sensor_size[1])
    out = torch.empty((2, H, W), dtype=torch.float32, device=dev)
    n = dx.numel()
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().esr_scatter_cnt(_lib.ptr(dx), _lib.ptr(dy), _lib.ptr(dp), None, 1, n, H, W,
                                              0, 0, 0, 0, 1, _lib.ptr(out), _lib.stream_ptr()), "esr_scatter_cnt")
    if cbx and xs.dtype == torch.float32:
        xs.copy_(dx)
    if cby and ys.dtype == torch.float32:
        ys.copy_(dy)
    return out if xs.is_cuda else out.cpu()


def encode_frames(xs, ys, ps, frame_off, lr_size=None, hr_size=(180, 240), n_max_frame=None, out=None, sanitised=False):
    """F frames of events -> [F,2,H,W] count images in one launch.

    sanitised=True reproduces the call ORDER of H5Dataset.__getitem__ (h5dataset.py:337-354): create_stack_encoding runs first
    and zeroes x, y, p of out-of-range events in place (frames of more than 3 events), so they add nothing to the count tensors;
    the default is the standalone events_to_channels, where an out-of-range NEGATIVE event lands on neg[0, 0].

    xs, ys, ps: CUDA fp32 [n_total]; frame_off: CUDA int64 [F+1].  With lr_size=(H_lr,W_lr) the coordinates
    are lifted x/W_lr*W_hr (two fp32 roundings, h5dataset.py:515,526) before the scatter = `inp_scaled_cnt`."""
    assert xs.is_cuda and ys.is_cuda and ps.is_cuda and frame_off.is_cuda
    F = frame_off.numel() - 1
    H, W = int(hr_size[0]), int(hr_size[1])
    if out is None:
        out = torch.empty((F, 2, H, W), dtype=torch.float32, device=xs.device)
    assert out.is_cuda and out.is_contiguous() and tuple(out.shape) == (F, 2, H, W)
    if n_max_frame is None:
        n_max_frame = xs.numel()
    lift = (int(lr_size[1]), W, int(lr_size[0]), H) if lr_size is not None else (0, 0, 0, 0)
    with torch.cuda.device(xs.device):
        _lib.check(_lib.lib().esr_scatter_cnt(_lib.ptr(xs), _lib.ptr(ys), _lib.ptr(ps), _lib.ptr(frame_off), F,
                                              int(n_max_frame), H, W, *lift, 2 if sanitised else 0, _lib.ptr(out), _lib.stream_ptr()),
                   "esr_scatter_cnt")
    return out


def interpolate_planes(x, size, mode):
    """F.interpolate(x.unsqueeze(0), size=size, mode=mode[, align_corners=False]).squeeze(0) for x [C, H, W] with mode
    'bicubic' or 'nearest' (dataloader/h5dataset.py:341-344, infer_ours_cnt.py:76-78), on the GPU (esr_resize_planes).
    CPU tensors are moved to the device and the result returned on the CPU, like the other encodings."""
    if mode not in ('bicubic', 'nearest'):
        raise ValueError(f"mode {mode!r} is not supported (bicubic | nearest)")
    dev = x.device if x.is_cuda else _dev()
    dx, _ = _to_dev_f32(x, dev)
    lead = dx.shape[:-2]
    Hin, Win = int(dx.shape[-2]), int(dx.shape[-1])
    Hout, Wout = int(size[0]), int(size[1])
    planes = int(np.prod(lead)) if len(lead) else 1
    out = torch.empty(tuple(lead) + (Hout, Wout), dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().esr_resize_planes(_lib.ptr(dx), planes, Hin, Win, Hout, Wout, 1 if mode == 'bicubic' else 0,
                                                _lib.ptr(out), _lib.stream_ptr()), "esr_resize_planes")
    return out if x.is_cuda else out.cpu()


def cython_event_redistribute(event_stack, mode='linear'):
    if mode == 'linear':
        cmode = 0
    elif mode == 'random':
        cmode = 1
    else:
        raise Exception(f'Not support {mode}')
    if len(event_stack.shape) not in (4, 5):
        raise Exception('wrong event stack')
    dev = event_stack.device if event_stack.is_cuda else _dev()
    return expand(event_stack.detach().to(dev, torch.float32), 1, cmode).cpu()


def multiprocess_cython(event_stack, mode='linear'):
    """Reference: one Pool() task per batch element (each reseeding numpy to 123); here one GPU call per element."""
    if mode == 'linear':
        cmode = 0
    elif mode == 'random':
        cmode = 1
    else:
        raise Exception(f'Not support {mode}')
    if len(event_stack.shape) not in (4, 5):
        raise Exception('wrong event stack')
    dev = event_stack.device if event_stack.is_cuda else _dev()
    st = event_stack.detach().to(dev, torch.float32)
    clouds = [expand(st[i:i + 1], 1, cmode) for i in range(st.shape[0])]
    maxlen = max(c.shape[1] for c in clouds)
    out = torch.zeros((st.shape[0], maxlen, 4), dtype=torch.float32, device=dev)
    for i, c in enumerate(clouds):
        out[i, :c.shape[1]] = c[0]
    return out.cpu()


def stack2cnt(stack):
    """stack BxTBxHxW -> Bx2xHxW (0 positive, 1 negative).  encodings.py:652-670 (pure tensor algebra)."""
    stack = stack.clone().detach().round()
    pos = stack.clamp(min=0).sum(1)
    neg = (-stack.clamp(max=0)).sum(1)
    return torch.stack([pos, neg], dim=1).cpu()
