"""Drop-in for the reference's `dataloader.cython_event_redistribute.event_redistribute` Cython module
(event_redistribute.pyx:17-153), backed by the sm_90a kernels.  numpy in, numpy out, like the original."""
import numpy as np
import torch

from .expand import expand


def _run(event_stack, mode, ndim):
    if not isinstance(event_stack, np.ndarray) or event_stack.dtype != np.float32:
        raise ValueError("Buffer dtype mismatch, expected 'float' but got something else")
    if event_stack.ndim != ndim:
        raise ValueError("Buffer has wrong number of dimensions (expected %d, got %d)" % (ndim, event_stack.ndim))
    dev = torch.device("cuda", torch.cuda.current_device())
    return expand(torch.from_numpy(np.ascontiguousarray(event_stack)).to(dev), 1, int(mode)).cpu().numpy()


def event_redistribute_PolarityStack(event_stack, mode):
    """event_stack [B, P, C, Y, X] -> [B, max_num_event, 4] (x, y, t, p)"""
    return _run(event_stack, mode, 5)


def event_redistribute_NoPolarityStack(event_stack, mode):
    """event_stack [B, C, Y, X] -> [B, max_num_event, 4] (x, y, t, p)"""
    return _run(event_stack, mode, 4)


def event_redistribute_cuda(event_stack, mode=0):
    """CUDA tensor in, CUDA tensor out."""
    return expand(event_stack, 1, int(mode))
