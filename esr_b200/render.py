"""Event-count images of the evaluation script on the GPU.

`render_event_cnt(cnt[B, 2, H, W], ...)` returns, for every sample b, the uint8 array that the reference's
`event_visualisation().plot_event_cnt(cnt[b].transpose(1, 2, 0), is_save=False, ...)`
(myutils/vis_events/matplotlib_plot_events.py:125-248) returns, bit for bit: all three colour schemes, both backgrounds,
is_norm on and off, and the cv2.cvtColor(BGR2RGB) channel swap unless use_opencv is set.  One C-ABI call
(esr_render_event_cnt: a radix select for the 1st / 99th percentiles of every plane, numpy 2.x's float32 values, then one
colour-map pass) renders the whole batch.

The gray scheme yields a 2-D image per sample ([B, H, W]); the script then calls cvtColor(BGR2RGB) on it, which OpenCV
refuses for one channel, so gray is only accepted with use_opencv=True.  The images are the arrays plot_event_cnt returns,
not the matplotlib figures it saves.
"""
import torch

from . import _lib

SCHEMES = {"gray": 0, "green_red": 1, "blue_red": 2}


def render_event_cnt(cnt, color_scheme="green_red", is_black_background=True, is_norm=True, use_opencv=False,
                     return_percentiles=False):
    """cnt: CUDA fp32 [B, 2, H, W] -> CUDA uint8 [B, H, W, 3] ([B, H, W] for gray).  With return_percentiles, also the
    fp32 [B, 2, 2] {np.percentile(plane, 1), np.percentile(plane, 99)} of both planes of every sample."""
    if color_scheme not in SCHEMES:
        raise ValueError(f"Not support {color_scheme}")
    if color_scheme == "gray" and not use_opencv:
        raise _lib.ESRError("render_event_cnt: the gray scheme gives a one-channel image, which cv2.cvtColor(BGR2RGB) refuses; "
                            "pass use_opencv=True")
    if not cnt.is_cuda:
        raise _lib.ESRError("esr_b200.render needs a CUDA tensor (there is no CPU path)")
    if cnt.dim() != 4 or cnt.shape[1] != 2:
        raise ValueError(f"render_event_cnt: expected [B, 2, H, W], got {tuple(cnt.shape)}")
    x = cnt.detach()
    if x.dtype != torch.float32 or not x.is_contiguous():
        x = x.float().contiguous()
    B, _, H, W = x.shape
    shape = (B, H, W) if color_scheme == "gray" else (B, H, W, 3)
    L = _lib.lib()
    with torch.cuda.device(x.device):
        out = torch.empty(shape, dtype=torch.uint8, device=x.device)
        pct = torch.empty((B, 2, 2), dtype=torch.float32, device=x.device) if return_percentiles else None
        nbytes = L.esr_render_workspace_bytes(B, H, W)
        ws = torch.empty((max(nbytes, 256),), dtype=torch.uint8, device=x.device)
        _lib.check(L.esr_render_event_cnt(_lib.ptr(x), B, H, W, SCHEMES[color_scheme], int(bool(is_black_background)),
                                          int(bool(is_norm)), int(bool(use_opencv)), _lib.ptr(out), _lib.ptr(pct), _lib.ptr(ws),
                                          nbytes, _lib.stream_ptr()), "esr_render_event_cnt")
    return (out, pct) if return_percentiles else out
