"""Generate tests/golden/lpips_golden.npz: the REFERENCE's perceptual_loss (loss/restore.py:10-39) on seeded inputs
(build container only; needs /root/reference).

The reference's own loss.restore.perceptual_loss runs on the CPU (use_gpu=False) with three stand-ins: IPython and
scikit-image (imported by the PerceptualSimilarity modules but not used on this path) and torchvision.models.alexnet, which
returns an AlexNet whose features carry tests/lpips_ref.seeded_alexnet(0) (the ImageNet checkpoint is not available
offline).  The linear heads are the reference's vendored weights/v0.1/alex.pth, loaded by the reference itself; the fixture
stores them as data.  Every case runs in fp32 and again in fp64 (the same model .double()).

Cases: 2-channel counts at 180 x 320 and 90 x 160, the 32 x 32 minimum, C = 1 with B = 2, an RGB image in [0, 1],
normalize=False, a bicubic-like plane with negative values; and the two inputs the reference refuses (24 x 24; B = 2 with
C = 2), stored with the exception's type.
"""
import os
import sys
import types

import numpy as np
import torch
import torchvision

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REFERENCE = "/root/reference"
sys.path.insert(0, os.path.dirname(HERE))
import lpips_ref  # noqa: E402  (tests/lpips_ref.py)

for name in ("IPython", "skimage", "skimage.metrics", "skimage.color", "skimage.transform"):
    sys.modules[name] = types.ModuleType(name)
sys.modules["IPython"].embed = lambda *a, **k: None
sys.modules["skimage"].color = sys.modules["skimage.color"]
sys.modules["skimage"].metrics = sys.modules["skimage.metrics"]
sys.modules["skimage"].transform = sys.modules["skimage.transform"]
sys.modules["skimage.metrics"].structural_similarity = None
sys.modules["skimage.metrics"].peak_signal_noise_ratio = None


def _seeded_alexnet(pretrained=False, **kw):
    m = torchvision.models.AlexNet()
    missing = m.load_state_dict(lpips_ref.seeded_alexnet(0), strict=False)
    assert not missing.unexpected_keys and all(k.startswith("classifier") for k in missing.missing_keys)
    return m


torchvision.models.alexnet = _seeded_alexnet
sys.path.insert(0, REFERENCE)
from loss.restore import perceptual_loss  # noqa: E402  (the reference)


def counts(g, shape, rate):
    return torch.poisson(torch.rand(shape, generator=g) * rate, generator=g)


def cases():
    g = torch.Generator().manual_seed(2024)
    out = []
    t = counts(g, (1, 2, 180, 320), 3.0)
    out.append(("counts_180x320", t + counts(g, t.shape, 1.0) - counts(g, t.shape, 1.0).clamp(max=1), t, True))
    t = counts(g, (1, 2, 90, 160), 2.0)
    out.append(("counts_90x160", counts(g, t.shape, 2.0), t, True))
    out.append(("min_32x32", counts(g, (1, 2, 32, 32), 2.0), counts(g, (1, 2, 32, 32), 2.0), True))
    out.append(("c1_b2", counts(g, (2, 1, 64, 96), 2.0), counts(g, (2, 1, 64, 96), 2.0), True))
    out.append(("rgb", torch.rand((1, 3, 64, 80), generator=g), torch.rand((1, 3, 64, 80), generator=g), True))
    out.append(("no_normalize", torch.rand((1, 3, 48, 80), generator=g) * 2 - 1, torch.rand((1, 3, 48, 80), generator=g) * 2 - 1,
                False))
    t = counts(g, (1, 2, 90, 160), 2.0)
    out.append(("bicubic_negative", t + torch.randn(t.shape, generator=g) * 0.6, t, True))
    return out


RAISING = (("too_small_24x24", (1, 2, 24, 24)), ("b2_c2", (2, 2, 40, 40)))


def main():
    torch.manual_seed(0)
    pl = perceptual_loss(net='alex', use_gpu=False)
    net = pl.model.model.net
    net.eval()
    heads = {k: v.detach().clone() for k, v in net.state_dict().items() if k.startswith("lin")}
    data = {f"heads/{k}": v.numpy() for k, v in heads.items()}
    names = []
    with torch.no_grad():
        for name, pred, target, normalize in cases():
            net.float()
            v32 = float(pl(pred.float(), target.float(), normalize=normalize))
            net.double()
            v64 = float(pl(pred.double(), target.double(), normalize=normalize))
            assert v64 >= 1e-3, (name, v64)
            print(f"{name:18s} fp32 {v32:.9g}  fp64 {v64:.17g}  rel {abs(v32 - v64) / v64:.2e}")
            data[f"{name}/pred"] = pred.numpy().astype(np.float32)
            data[f"{name}/target"] = target.numpy().astype(np.float32)
            data[f"{name}/normalize"] = np.array(normalize)
            data[f"{name}/fp32"] = np.array(v32)
            data[f"{name}/fp64"] = np.array(v64)
            names.append(name)
        net.float()
        for name, shape in RAISING:
            x = torch.rand(shape, generator=torch.Generator().manual_seed(7))
            try:
                pl(x, x)
            except Exception as e:          # the reference's own failure
                print(f"{name:18s} raises {type(e).__name__}: {str(e).splitlines()[0][:80]}")
                data[f"{name}/shape"] = np.array(shape)
                data[f"{name}/raises"] = np.array(type(e).__name__)
            else:
                raise AssertionError(f"{name}: the reference did not raise")
    data["cases"] = np.array(names)
    data["raising"] = np.array([n for n, _ in RAISING])
    np.savez_compressed(os.path.join(HERE, "lpips_golden.npz"), **data)


if __name__ == "__main__":
    main()
