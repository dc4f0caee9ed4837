"""Drop-in for the reference's `dataloader.cython_cnt2event.cnt2event` Cython module and its
`cnt2event_api` wrapper, backed by the sm_90a kernels.

  cnt2event(event_cnt: np.ndarray[float32, ndim=4], mode: int) -> np.ndarray[float32, (B, maxlen, 4)]
        same signature / dtype checks as cnt2event.pyx:18-19
  cnt2eventAPI(event_cnt: torch.Tensor, mode=0) -> torch.Tensor (CPU), as cnt2event_api.py:25-35
  cnt2event_cuda(event_cnt: CUDA tensor, mode=0) -> CUDA tensor   (no host round trip of the payload)
"""
import numpy as np
import torch

from .expand import expand


def cnt2event_cuda(event_cnt, mode=0):
    return expand(event_cnt, 0, int(mode))


def cnt2event(event_cnt, mode):
    if not isinstance(event_cnt, np.ndarray) or event_cnt.dtype != np.float32:
        raise ValueError("Buffer dtype mismatch, expected 'float' but got something else")
    if event_cnt.ndim != 4:
        raise ValueError("Buffer has wrong number of dimensions (expected 4, got %d)" % event_cnt.ndim)
    assert event_cnt.shape[1] == 2, "Wrong event count data!"
    dev = torch.device("cuda", torch.cuda.current_device())
    out = expand(torch.from_numpy(np.ascontiguousarray(event_cnt)).to(dev), 0, int(mode))
    return out.cpu().numpy()


def cnt2eventAPI(event_cnt, mode=0):
    if event_cnt.is_cuda:
        return expand(event_cnt.detach(), 0, int(mode)).cpu()
    cnt_np = event_cnt.detach().cpu().numpy().astype(np.float32)
    return torch.from_numpy(cnt2event(cnt_np, mode))
