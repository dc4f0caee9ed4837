"""LPIPS on the GPU: the perceptual distance of infer_ours_cnt.py:85,90 (esr_lpips / bicubic_lpips).

The reference builds `loss/restore.py:perceptual_loss` (:10-39), i.e. LPIPS version 0.1 with torchvision's ImageNet AlexNet
(`tv.alexnet(pretrained=True)`, sliced at relu1 .. relu5) and the linear heads shipped as
`loss/PerceptualSimilarity/models/weights/v0.1/alex.pth`.  Here the whole distance runs as CUDA kernels of libesr_b200
(esr_lpips_forward: conv1 im2col on the tensor cores, the other convolutions on the wgmma implicit GEMM, split-bf16
three-term products, fp64 per-pair reductions); there is no CPU or PyTorch fallback.

    LPIPS(alexnet, lin)                     weights: paths or state dicts (torchvision's alexnet checkpoint, the v0.1 heads)
    LPIPS.distances(planes, channel_src, pair_a, pair_b, normalize)   per-pair distances, CUDA float64
    LPIPS.window_pairs(esr, bicubic, gt)    the evaluation's two values per window, gt's features computed once
    perceptual_loss(weight, net, use_gpu, gpu_ids)   loss/restore.py's wrapper, same call signature and channel rules

Weights are not downloaded: perceptual_loss resolves them at its first call (explicit paths, then torchvision's hub cache
and the reference checkout's heads when its `loss` package is importable).
"""
import ctypes
import importlib.util
import os
from collections.abc import Mapping

import numpy as np
import torch

from . import _lib

CHANNELS = (64, 192, 384, 256, 256)
ALEXNET_KEYS = (("features.0.weight", (64, 3, 11, 11)), ("features.0.bias", (64,)),
                ("features.3.weight", (192, 64, 5, 5)), ("features.3.bias", (192,)),
                ("features.6.weight", (384, 192, 3, 3)), ("features.6.bias", (384,)),
                ("features.8.weight", (256, 384, 3, 3)), ("features.8.bias", (256,)),
                ("features.10.weight", (256, 256, 3, 3)), ("features.10.bias", (256,)))
LIN_KEYS = tuple((f"lin{l}.model.1.weight", (1, c, 1, 1)) for l, c in enumerate(CHANNELS))
TORCHVISION_ALEXNET = "alexnet-owt-7be5be79.pth"     # the file tv.alexnet(pretrained=True) keeps in torch.hub's cache
MIN_SIDE = 31                                        # below this AlexNet's second max-pool has no output (torch raises)
WORKSPACE_BUDGET = 1 << 30                           # bytes of activations one plan may hold; larger batches run in chunks
MAX_PLAN_IMAGES = 256


def _state_dict(src, what):
    if isinstance(src, (str, os.PathLike)):
        if not os.path.isfile(src):
            raise _lib.ESRError(f"LPIPS: {what} weights {src} not found")
        src = torch.load(src, map_location="cpu", weights_only=True)
    if not isinstance(src, Mapping):
        raise _lib.ESRError(f"LPIPS: {what} weights must be a path or a state dict, not {type(src).__name__}")
    return src


def _pick(sd, keys, what):
    out = []
    for k, shape in keys:
        if k not in sd:
            raise _lib.ESRError(f"LPIPS: {what} weights have no key {k}")
        t = sd[k]
        if not torch.is_tensor(t) or tuple(t.shape) != shape:
            got = tuple(t.shape) if torch.is_tensor(t) else type(t).__name__
            raise _lib.ESRError(f"LPIPS: {what} weight {k} has shape {got}, expected {shape}")
        out.append(t.detach().to(torch.float32).contiguous())
    return out


class _Plan:
    def __init__(self, n_img, H, W, blob, device):
        lib = _lib.lib()
        nbytes = lib.esr_lpips_workspace_bytes(n_img, H, W)
        self.ws = torch.empty((nbytes,), dtype=torch.uint8, device=device)
        self.handle = ctypes.c_void_p()
        _lib.check(lib.esr_lpips_create(ctypes.byref(self.handle), n_img, H, W, _lib.ptr(blob), _lib.ptr(self.ws), nbytes),
                   "esr_lpips_create")
        self.n_img = n_img

    def __del__(self):
        if getattr(self, "handle", None) and _lib._lib is not None:
            _lib._lib.esr_lpips_destroy(self.handle)
            self.handle = None


class LPIPS:
    """LPIPS v0.1 with the AlexNet backbone.  alexnet: torchvision's checkpoint format (features.{0,3,6,8,10}.{weight,bias};
    classifier.* is ignored); lin: the reference's v0.1 heads (lin{0..4}.model.1.weight).  Each is a path or a state dict;
    a missing key or a wrong shape raises ESRError."""

    def __init__(self, alexnet, lin):
        self._params = _pick(_state_dict(alexnet, "alexnet"), ALEXNET_KEYS, "alexnet") + \
            _pick(_state_dict(lin, "lin"), LIN_KEYS, "lin")
        self._blobs = {}
        self._plans = {}

    def _blob(self, device):
        blob = self._blobs.get(device)
        if blob is None:
            L = _lib.lib()
            tensors = [p.to(device) for p in self._params]
            arr = (ctypes.c_void_p * len(tensors))(*[t.data_ptr() for t in tensors])
            blob = torch.empty((L.esr_lpips_param_bytes(),), dtype=torch.uint8, device=device)
            _lib.check(L.esr_lpips_pack_params(arr, _lib.ptr(blob), _lib.stream_ptr()), "esr_lpips_pack_params")
            torch.cuda.current_stream().synchronize()      # `tensors` are temporaries
            self._blobs[device] = blob
        return blob

    @staticmethod
    def capacity(H, W):
        """Images one plan holds at H x W (the chunk size of larger calls)."""
        L = _lib.lib()
        one = L.esr_lpips_workspace_bytes(1, H, W)
        if one == 0:
            raise _lib.ESRError(f"LPIPS: a {H} x {W} image is too small for AlexNet's second max-pool "
                                f"(LPIPS needs at least {MIN_SIDE} x {MIN_SIDE})")
        per = max(1, L.esr_lpips_workspace_bytes(2, H, W) - one)
        return int(max(1, min(MAX_PLAN_IMAGES, WORKSPACE_BUDGET // per)))

    def _plan(self, n_img, H, W, device):
        key = (device, n_img, H, W)
        p = self._plans.get(key)
        if p is None:
            p = self._plans[key] = _Plan(n_img, H, W, self._blob(device), device)
        return p

    def distances(self, planes, channel_src, pair_a, pair_b, normalize=True):
        """planes: CUDA fp32 [P, H, W]; channel_src: int [n_img, 3], the plane of each input channel of each image;
        pair_a, pair_b: int sequences of image indices.  -> CUDA float64 [n_pairs]: LPIPS(image pair_a[p], image pair_b[p]).
        normalize: the images are in [0, 1] and are mapped to [-1, 1] first (perceptual_loss's default).  Pairs are
        processed in chunks whose images fit one plan; a pair's value does not depend on the chunking."""
        if not planes.is_cuda:
            raise _lib.ESRError("LPIPS needs CUDA tensors (no CPU fallback)")
        if planes.dim() != 3:
            raise ValueError("LPIPS.distances: planes must be [P, H, W]")
        P, H, W = (int(s) for s in planes.shape)
        cap = self.capacity(H, W)
        src = np.asarray(channel_src, dtype=np.int64).reshape(-1, 3)
        pa, pb = np.asarray(pair_a, dtype=np.int64).ravel(), np.asarray(pair_b, dtype=np.int64).ravel()
        if pa.shape != pb.shape or pa.size == 0:
            raise ValueError("LPIPS.distances: pair_a and pair_b must be non-empty and of equal length")
        if src.size and (src.min() < 0 or src.max() >= P):
            raise ValueError("LPIPS.distances: channel_src indexes a plane outside planes")
        if min(pa.min(), pb.min()) < 0 or max(pa.max(), pb.max()) >= len(src):
            raise ValueError("LPIPS.distances: a pair indexes an image outside channel_src")
        dev = planes.device
        x = planes.detach().to(torch.float32).contiguous()
        out = torch.empty((pa.size,), dtype=torch.float64, device=dev)
        L = _lib.lib()
        with torch.cuda.device(dev):
            # greedy chunks of consecutive pairs whose distinct images fit `cap`
            i = 0
            while i < pa.size:
                imgs, j = {}, i
                while j < pa.size:
                    new = [k for k in sorted({int(pa[j]), int(pb[j])}) if k not in imgs]
                    if len(imgs) + len(new) > cap or j - i >= cap:
                        break
                    for k in new:
                        imgs[k] = len(imgs)
                    j += 1
                order = list(imgs)
                n = len(order)
                plan = self._plan(self._plan_size(max(n, j - i), cap), H, W, dev)
                host = np.concatenate([src[order].reshape(-1),
                                       [imgs[int(k)] for k in pa[i:j]], [imgs[int(k)] for k in pb[i:j]]]).astype(np.int32)
                idx = torch.as_tensor(host).to(dev, non_blocking=False)
                np_ = j - i
                _lib.check(L.esr_lpips_forward(plan.handle, _lib.ptr(x), _lib.ptr(idx), n, 1 if normalize else 0, np_,
                                               _at(idx, 3 * n), _at(idx, 3 * n + np_), _lib.ptr(out[i:j]),
                                               _lib.stream_ptr()), "esr_lpips_forward")
                i = j
        return out

    @staticmethod
    def _plan_size(n, cap):
        """Plans come in powers of two up to cap, so that steps of varying size share a few plans."""
        s = 1
        while s < n:
            s *= 2
        return min(s, cap)

    def window_pairs(self, esr, bicubic, gt):
        """esr, bicubic, gt: CUDA fp32 [n, C, H, W] -> CUDA float64 [2, n]: perceptual_loss()(esr[j:j+1], gt[j:j+1]) and
        the same of bicubic, per window j -- each of the C planes repeated to three channels, distances averaged over the
        C planes (loss/restore.py:33-37), with gt's features computed once for both pairs."""
        n, C, H, W = esr.shape
        assert bicubic.shape == esr.shape and gt.shape == esr.shape
        planes = torch.cat([esr, bicubic, gt]).reshape(3 * n * C, H, W)
        src = np.repeat(np.arange(3 * n * C), 3).reshape(-1, 3)
        k = np.arange(n * C)
        # the reference calls PerceptualLoss.forward(pred, target) -> DistModel.forward(target, pred)
        d = self.distances(planes, src, np.concatenate([2 * n * C + k, 2 * n * C + k]), np.concatenate([k, n * C + k]))
        return d.view(2, n, C).mean(dim=2)


def _at(t, offset):
    """Device address of element `offset` of a contiguous int32 tensor."""
    return ctypes.c_void_p(t.data_ptr() + 4 * offset)


def _hub_alexnet():
    return os.path.join(torch.hub.get_dir(), "checkpoints", TORCHVISION_ALEXNET)


def _reference_heads():
    """The reference checkout's v0.1 AlexNet heads, when its `loss` package is importable (found, not imported: importing it
    pulls in skimage and IPython)."""
    try:
        spec = importlib.util.find_spec("loss")
    except (ImportError, ValueError):
        return None
    if spec is None or not spec.submodule_search_locations:
        return None
    return os.path.join(list(spec.submodule_search_locations)[0], "PerceptualSimilarity", "models", "weights", "v0.1", "alex.pth")


class perceptual_loss:
    """loss/restore.py:10-39 on the GPU.  perceptual_loss(weight=1.0, net='alex', use_gpu=True, gpu_ids=[0]) -- only 'alex'
    exists -- then loss(pred, target, normalize=True) with N x C x H x W CUDA tensors: C = 1 is repeated to 3 channels, C = 3
    is used as is, any other C averages the distances of each channel repeated to 3 (which the reference only supports for
    N = 1: its repeat makes a 1 x 3N-channel tensor that AlexNet refuses, and so does this).  Returns weight * mean over the
    batch as a 0-dim CUDA fp32 tensor.
    Weights are resolved at the first call (the training script constructs one and never calls it): alexnet / lin paths
    given here; else torchvision's hub-cache file for the backbone and the reference checkout's v0.1 heads; else ESRError
    naming the missing file."""

    def __init__(self, weight=1.0, net='alex', use_gpu=True, gpu_ids=[0], alexnet=None, lin=None):
        if net != 'alex':
            raise _lib.ESRError(f"perceptual_loss: net={net!r} is not implemented (only 'alex')")
        self.weight = weight
        self._alexnet, self._lin = alexnet, lin
        self.model = None

    def _resolve(self):
        if self.model is None:
            a = self._alexnet if self._alexnet is not None else _hub_alexnet()
            h = self._lin if self._lin is not None else _reference_heads()
            if h is None:
                raise _lib.ESRError("perceptual_loss: no LPIPS heads given and the reference's `loss` package (its "
                                    "PerceptualSimilarity/models/weights/v0.1/alex.pth) is not importable")
            self.model = LPIPS(a, h)
        return self.model

    def __call__(self, pred, target, normalize=True):
        assert pred.size() == target.size()
        model = self._resolve()
        B, C, H, W = pred.shape
        planes = torch.cat([pred.detach(), target.detach()]).reshape(2 * B * C, H, W)
        if C == 3:
            src = np.arange(2 * B * 3).reshape(-1, 3)
            d = model.distances(planes, src, np.arange(B, 2 * B), np.arange(B), normalize)
        else:
            if C != 1 and B != 1:
                raise _lib.ESRError(f"perceptual_loss: {C}-channel input with batch {B}: the reference's per-channel repeat "
                                    f"gives a 1 x {3 * B}-channel tensor, which AlexNet's 3-channel conv1 refuses")
            src = np.repeat(np.arange(2 * B * C), 3).reshape(-1, 3)
            n = B * C
            d = model.distances(planes, src, np.arange(n, 2 * n), np.arange(n), normalize)
            if C != 1:
                d = d.view(B, C).mean(dim=1)
        return (self.weight * d.mean()).to(torch.float32)
