"""Evaluation metrics of the reference's inference loop on the GPU (SURVEY.md 8f rank 3).

infer_ours_cnt.py:81-100 computes, per evaluated frame, nn.L1Loss / nn.MSELoss on CPU tensors and the two wrappers of
loss/restore.py -- `ssim_loss` (:42-61) and `psnr_loss` (:64-90) -- which move the tensors to numpy and call skimage once
per channel.  Here one C-ABI call (esr_metrics_planes: three kernel launches) produces every per-plane statistic of a whole
batch on the device; only 6 doubles per plane travel to the host.

    ssim_loss()(pred, tgt), psnr_loss()(pred, tgt)   same call signatures and semantics as loss/restore.py
    l1(pred, tgt), mse(pred, tgt)                      nn.L1Loss() / nn.MSELoss() values
    evaluate(pred, tgt)                                {"l1", "mse", "ssim", "psnr"} in one pass (the dict the loop tracks)

skimage conventions restated (skimage.metrics, 0.16-0.21 behaviour for float images):
  structural_similarity(im1, im2): win_size 7, uniform window, use_sample_covariance, K1 0.01, K2 0.03,
      data_range = 2 for floating-point inputs (dtype range -1..1), mean of S over the image cropped by 3 pixels;
  peak_signal_noise_ratio(true, test, data_range): 10 log10(data_range^2 / mean((true - test)^2)); with data_range=None and a
      float image it is 1 if true.min() >= 0 else 2.
There is no CPU fallback: tensors must be CUDA fp32.
"""
import math

import torch

from . import _lib

WIN = 7
FLOAT_DATA_RANGE = 2.0


def plane_stats(pred, tgt, win=WIN, data_range=FLOAT_DATA_RANGE):
    """pred, tgt: CUDA fp32 [..., H, W] of equal shape -> CPU float64 [n_planes, 6]:
    {sum |d|, sum d^2, max tgt, min tgt, SSIM-map sum over the valid region, valid pixel count} per plane."""
    return plane_stats_device(pred, tgt, win, data_range).cpu()


def plane_stats_device(pred, tgt, win=WIN, data_range=FLOAT_DATA_RANGE):
    """plane_stats left on the device (no synchronisation): CUDA float64 [n_planes, 6]."""
    if not (pred.is_cuda and tgt.is_cuda):
        raise _lib.ESRError("esr_b200.metrics needs CUDA tensors (no CPU fallback)")
    assert pred.shape == tgt.shape and pred.dim() >= 2
    H, W = int(pred.shape[-2]), int(pred.shape[-1])
    p = pred.detach().float().contiguous().view(-1, H, W)
    t = tgt.detach().float().contiguous().view(-1, H, W)
    n = p.shape[0]
    L = _lib.lib()
    with torch.cuda.device(p.device):
        nbytes = L.esr_metrics_workspace_bytes(n, H, W, win)
        ws = torch.empty((max(nbytes, 256),), dtype=torch.uint8, device=p.device)
        stats = torch.zeros((n, 6), dtype=torch.float64, device=p.device)
        _lib.check(L.esr_metrics_planes(_lib.ptr(p), _lib.ptr(t), n, H, W, int(win), float(data_range), _lib.ptr(stats),
                                        _lib.ptr(ws), nbytes, _lib.stream_ptr()), "esr_metrics_planes")
    return stats


def l1(pred, tgt):
    s = plane_stats(pred, tgt)
    return torch.tensor(float(s[:, 0].sum()) / pred.numel(), dtype=torch.float32)


def mse(pred, tgt):
    s = plane_stats(pred, tgt)
    return torch.tensor(float(s[:, 1].sum()) / pred.numel(), dtype=torch.float32)


def _psnr(err, data_range):
    return 10.0 * math.log10((data_range ** 2) / err) if err > 0 else float("inf")


def _reference_reduce(s, shape):
    """The two wrappers' channel logic (loss/restore.py:50-59, 72-86) from the per-plane statistics of ONE sample whose
    squeezed shape is [C, H, W] (C > 1) or [H, W]."""
    HW = shape[-2] * shape[-1]
    ssim_pl = s[:, 4] / s[:, 5]
    if s.shape[0] > 1:
        gmin = float(s[:, 3].min())                            # `tgt.min()`: over ALL channels (restore.py:80)
        psnr = sum(_psnr(float(s[c, 1]) / HW, float(s[c, 2]) - gmin) for c in range(s.shape[0])) / s.shape[0]
        return float(ssim_pl.mean()), psnr
    return float(ssim_pl[0]), None


class ssim_loss:
    """loss/restore.py:42-61.  pred, tgt: 1xNxHxW (N channels averaged) or 1x1xHxW."""

    def __call__(self, pred, tgt):
        assert pred.size() == tgt.size()
        p, t = pred.squeeze(), tgt.squeeze()
        if p.dim() not in (2, 3):
            raise ValueError("ssim_loss: expected a 1xNxHxW tensor (the reference evaluates with batch size 1)")
        return _reference_reduce(plane_stats(p, t), tuple(p.shape))[0]


class psnr_loss:
    """loss/restore.py:64-90.  pred, tgt: 1xNxHxW: per channel PSNR(tgt[c], pred[c], data_range = tgt[c].max() - tgt.min()),
    averaged; a single plane is clipped to [0, 1] first and uses skimage's default range for float images."""

    def __call__(self, pred, tgt):
        assert pred.size() == tgt.size()
        p, t = pred.squeeze(), tgt.squeeze()
        if p.dim() == 3:
            return _reference_reduce(plane_stats(p, t), tuple(p.shape))[1]
        if p.dim() != 2:
            raise ValueError("psnr_loss: expected a 1xNxHxW tensor (the reference evaluates with batch size 1)")
        # restore.py:86 calls PSNR(pred.clip(0,1), tgt.clip(0,1)): image_true = the clipped PREDICTION, min >= 0 -> data_range 1
        s = plane_stats(p.clamp(0, 1), t.clamp(0, 1))
        return _psnr(float(s[0, 1]) / p.numel(), 1.0)


def evaluate(pred, tgt):
    """The four scalars infer_ours_cnt.py:81-84 tracks for (esr_cnt, gt_cnt) [B, C, H, W], from ONE statistics pass.
    B > 1 (not used by the reference, whose evaluation loader has batch size 1): SSIM / PSNR are the mean over samples of the
    reference's per-sample value."""
    assert pred.shape == tgt.shape and pred.dim() == 4
    B, C, H, W = pred.shape
    s = plane_stats(pred, tgt).view(B, C, 6)
    out = {"l1": float(s[..., 0].sum()) / pred.numel(), "mse": float(s[..., 1].sum()) / pred.numel()}
    ss, ps = [], []
    for b in range(B):
        if C > 1:
            a, p = _reference_reduce(s[b], (C, H, W))
        else:
            a = float(s[b, 0, 4] / s[b, 0, 5])
            p = psnr_loss()(pred[b:b + 1], tgt[b:b + 1])
        ss.append(a)
        ps.append(p)
    out["ssim"] = sum(ss) / B
    out["psnr"] = sum(ps) / B
    return out


def evaluate_from_stats(s, shape):
    """evaluate() of ONE sample from its per-plane statistics s [C, 6] (CPU float64) and its shape (C, H, W), C > 1:
    the same arithmetic, so a batch's statistics computed once give every sample's values bit for bit."""
    C, H, W = shape
    assert C > 1 and s.shape[0] == C
    a, p = _reference_reduce(s, (C, H, W))
    return {"l1": float(s[:, 0].sum()) / (C * H * W), "mse": float(s[:, 1].sum()) / (C * H * W), "ssim": a, "psnr": p}
