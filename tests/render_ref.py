"""TEST INFRASTRUCTURE ONLY -- numpy restatement of the evaluation script's event-count image
(myutils/vis_events/matplotlib_plot_events.py:125-248, plot_event_cnt with is_save=False).

It follows the reference's numpy dtypes at every step: float32 percentiles (np.percentile on the float32 plane) and
normalisation, float32 `1 - v`, a float64 image, `* 255` in float64, truncating astype(uint8); channel order BGR, reversed
unless use_opencv (cv2.cvtColor(BGR2RGB) on a 3-channel uint8 image is a channel reversal).  esr_b200.render must equal it
bit for bit; tests/golden/render_golden.npz pins it against the reference's own function.
"""
import numpy as np


def render_one(cnt, color_scheme="green_red", is_black_background=True, is_norm=True, use_opencv=False):
    """cnt: float32 [2, H, W] -> uint8 [H, W, 3] ([H, W] for gray, which needs use_opencv=True)."""
    pos = np.array(cnt[0], dtype=np.float32)
    neg = np.array(cnt[1], dtype=np.float32)
    p_lo, p_hi = np.percentile(pos, 1), np.percentile(pos, 99)
    n_lo, n_hi = np.percentile(neg, 1), np.percentile(neg, 99)
    top = p_hi if p_hi > n_hi else n_hi
    if is_norm:
        if p_lo != top:
            pos = (pos - p_lo) / (top - p_lo)
        if n_lo != top:
            neg = (neg - n_lo) / (top - n_lo)
    else:
        pos_wins = (pos >= neg) & (pos != 0)
        neg_wins = (pos < neg) & (neg != 0)
        pos = np.where(pos_wins, np.float32(1), np.where(neg_wins, np.float32(0), pos))
        neg = np.where(pos_wins, np.float32(0), np.where(neg_wins, np.float32(1), neg))
    pos = np.clip(pos, 0, 1)
    neg = np.clip(neg, 0, 1)
    if color_scheme == "gray":
        if not use_opencv:
            raise ValueError("cv2.cvtColor(BGR2RGB) refuses a one-channel image")
        img = 0.5 + (pos * np.float32(0.5) + neg * np.float32(-0.5)).astype(np.float64)
        return (img * 255).astype(np.uint8)
    H, W = pos.shape
    if is_black_background:
        img = np.zeros((H, W, 3), np.float64)
        img[..., 1 if color_scheme == "green_red" else 0] = np.where(pos > 0, pos, 0)
        img[..., 2] = np.where(neg > 0, neg, 0)
    else:
        img = np.ones((H, W, 3), np.float64)
        pos_px = (pos > 0) & (pos >= neg)
        neg_px = ~pos_px & (neg > 0)
        one_m_pos = (np.float32(1) - pos).astype(np.float64)
        one_m_neg = (np.float32(1) - neg).astype(np.float64)
        for c in ((0, 2) if color_scheme == "green_red" else (1, 2)):
            img[..., c] = np.where(pos_px, one_m_pos, img[..., c])
        for c in (0, 1):
            img[..., c] = np.where(neg_px, one_m_neg, img[..., c])
    out = (img * 255).astype(np.uint8)
    return out if use_opencv else np.ascontiguousarray(out[..., ::-1])


def render(cnt, **kw):
    """cnt: float32 [B, 2, H, W] -> stacked render_one per sample."""
    return np.stack([render_one(c, **kw) for c in np.asarray(cnt, np.float32)])
