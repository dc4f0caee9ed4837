"""Generate tests/golden/render_golden.npz from the REFERENCE's own plot_event_cnt (build container only).

myutils/vis_events/matplotlib_plot_events.py is imported unmodified.  Its imports that are absent here or irrelevant to the
returned array are stubbed: matplotlib, mpl_toolkits, open3d, the visualization module and the dataloader modules it imports
names from.  `event_visualisation.plot_data` (the matplotlib figure) is made a no-op.  `cv2.cvtColor(img, COLOR_BGR2RGB)` is
stubbed as a channel reversal, which is OpenCV's definition of that conversion for a 3-channel uint8 image; like OpenCV, the
stub refuses any other channel count, so the gray scheme (a 2-D image) raises unless use_opencv=True.

Cases ([2, H, W] float32 planes): Poisson counts, real-valued bicubic planes with negative undershoot (torch's CPU bicubic
resize of Poisson counts), all-zero and constant planes, pos_min == max, mostly-zero planes, sizes 1x1 to 720x1280.  Every
option combination runs on the small cases; the two large ones (96 x 128 real-valued, 720 x 1280 sparse) run a subset, and
their images are stored as SHA-256 digests of the array bytes, which still pin them bit for bit, to keep the file small.
Integer-valued inputs in 0..255 are stored as uint8 (the tests cast them back to float32, which is exact).  Each input is
passed as a fresh array (the is_norm=False branch writes into it, as the reference does).
"""
import hashlib
import itertools
import os
import sys
import types
from unittest import mock

import numpy as np
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, "/root/reference")

cv2 = types.ModuleType("cv2")
cv2.COLOR_BGR2RGB = 4


def _cvt(img, code):
    assert code == cv2.COLOR_BGR2RGB
    if img.ndim != 3 or img.shape[2] != 3:
        raise ValueError("cv2.cvtColor(BGR2RGB): invalid number of channels in input image")
    return np.ascontiguousarray(img[:, :, ::-1])


cv2.cvtColor = _cvt
sys.modules["cv2"] = cv2
for name in ("matplotlib", "matplotlib.pyplot", "matplotlib.animation", "mpl_toolkits", "mpl_toolkits.axes_grid1", "open3d",
             "myutils", "myutils.vis_events", "myutils.vis_events.visualization", "dataloader", "dataloader.h5dataset",
             "dataloader.h5dataloader", "dataloader.encodings"):
    m = types.ModuleType(name)
    m.__dict__.setdefault("__path__", [])
    sys.modules[name] = m
sys.modules["matplotlib"].pyplot = sys.modules["matplotlib.pyplot"]
sys.modules["matplotlib.pyplot"].style = mock.MagicMock()
sys.modules["mpl_toolkits.axes_grid1"].ImageGrid = mock.MagicMock()
sys.modules["dataloader.h5dataset"].H5Dataset = mock.MagicMock()
sys.modules["dataloader.h5dataloader"].InferenceHDF5DataLoader = mock.MagicMock()
sys.modules["myutils.vis_events"].__path__ = [os.path.join("/root/reference", "myutils", "vis_events")]

from myutils.vis_events.matplotlib_plot_events import event_visualisation  # noqa: E402  (the reference)

event_visualisation.plot_data = lambda self, *a, **k: None

SCHEMES = ("gray", "green_red", "blue_red")
OPTIONS = [dict(color_scheme=s, is_black_background=bg, is_norm=nm, use_opencv=cv)
           for s, bg, nm, cv in itertools.product(SCHEMES, (True, False), (True, False), (True, False))]


def opt_key(o):
    return f"{o['color_scheme']}_{'black' if o['is_black_background'] else 'white'}_{'norm' if o['is_norm'] else 'raw'}_" \
           f"{'bgr' if o['use_opencv'] else 'rgb'}"


def bicubic(lr, size):
    return F.interpolate(torch.from_numpy(lr)[None], size=size, mode="bicubic", align_corners=False)[0].numpy()


def cases():
    rng = np.random.default_rng(7)
    pois = lambda lam, H, W: rng.poisson(lam, (2, H, W)).astype(np.float32)
    c = {}
    c["p1x1"] = pois(2.0, 1, 1)
    c["p1x7"] = pois(1.0, 1, 7)
    c["n5x3"] = rng.normal(0.0, 1.0, (2, 5, 3)).astype(np.float32)
    c["p48x64"] = pois(0.5, 48, 64)
    c["p33x47"] = pois(3.0, 33, 47)
    c["b48x64"] = bicubic(pois(0.7, 12, 16), (48, 64))
    c["zero"] = np.zeros((2, 32, 32), np.float32)
    c["const"] = np.full((2, 32, 32), 2.0, np.float32)
    pm = pois(1.0, 32, 32)
    pm[0] = 3.0
    pm[1] = np.minimum(pm[1], 3.0)                        # pos_min == pos_max == max
    c["posmin_eq_max"] = pm
    sp = np.zeros((2, 64, 96), np.float32)
    m = rng.random((2, 64, 96)) < 0.01
    sp[m] = rng.integers(1, 6, m.sum())
    c["sparse64x96"] = sp
    c["b96x128"] = bicubic(pois(0.4, 24, 32), (96, 128))
    big = np.zeros((2, 720, 1280), np.float32)
    m = rng.random((2, 720, 1280)) < 0.03
    big[m] = rng.integers(1, 4, m.sum())
    c["sparse720x1280"] = big
    return c


LARGE = {"b96x128", "sparse720x1280"}
LARGE_OPTIONS = [o for o in OPTIONS if o["color_scheme"] != "gray" and o["use_opencv"] is False and o["is_black_background"] != o["is_norm"]] + \
                [dict(color_scheme="green_red", is_black_background=True, is_norm=True, use_opencv=False)]


def main():
    vis = event_visualisation()
    out = {}
    names = []
    for name, cnt in cases().items():
        names.append(name)
        integral = np.array_equal(cnt, np.round(cnt)) and cnt.min() >= 0 and cnt.max() <= 255 and not np.signbit(cnt).any()
        out[f"{name}_cnt"] = cnt.astype(np.uint8) if integral else cnt
        out[f"{name}_pct"] = np.array([[np.percentile(cnt[p], 1), np.percentile(cnt[p], 99)] for p in range(2)], np.float32)
        keys = []
        for o in (LARGE_OPTIONS if name in LARGE else OPTIONS):
            k = opt_key(o)
            if k in keys:
                continue
            try:
                img = vis.plot_event_cnt(np.array(cnt).transpose(1, 2, 0), is_save=False, **o)
            except ValueError:
                assert o["color_scheme"] == "gray" and not o["use_opencv"]
                continue
            keys.append(k)
            if name in LARGE:
                out[f"{name}_{k}_sha256"] = np.frombuffer(hashlib.sha256(np.ascontiguousarray(img).tobytes()).digest(), np.uint8)
                out[f"{name}_{k}_shape"] = np.array(img.shape)
            else:
                out[f"{name}_{k}"] = img
        out[f"{name}_options"] = np.array(keys)
    out["names"] = np.array(names)
    path = os.path.join(HERE, "render_golden.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    main()
