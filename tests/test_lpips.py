"""CPU: the LPIPS restatement (tests/lpips_ref.py) against the reference's own perceptual_loss (tests/golden/lpips_golden.npz),
weight loading and its errors, and the inputs too small for AlexNet."""
import os

import numpy as np
import pytest
import torch

from esr_b200 import _lib, lpips
from tests import lpips_ref

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "lpips_golden.npz")


def golden():
    g = np.load(GOLD)
    heads = {k[len("heads/"):]: torch.from_numpy(g[k]) for k in g.files if k.startswith("heads/")}
    return g, heads


def test_oracle_matches_reference_golden():
    g, heads = golden()
    sd = lpips_ref.seeded_alexnet(0)
    assert len(g["cases"]) == 7
    for name in g["cases"]:
        pred, target = torch.from_numpy(g[f"{name}/pred"]), torch.from_numpy(g[f"{name}/target"])
        norm = bool(g[f"{name}/normalize"])
        v32 = float(lpips_ref.perceptual_loss(pred, target, sd, heads, normalize=norm))
        v64 = float(lpips_ref.perceptual_loss(pred.double(), target.double(), sd, heads, normalize=norm))
        assert v64 >= 1e-3
        assert abs(v32 - float(g[f"{name}/fp32"])) <= 1e-6 * abs(v64), name
        assert abs(v64 - float(g[f"{name}/fp64"])) <= 1e-12 * abs(v64), name


def test_oracle_raises_where_the_reference_raises():
    g, heads = golden()
    sd = lpips_ref.seeded_alexnet(0)
    for name in g["raising"]:
        assert str(g[f"{name}/raises"]) == "RuntimeError"
        x = torch.rand(tuple(int(s) for s in g[f"{name}/shape"]))
        with pytest.raises(RuntimeError):
            lpips_ref.perceptual_loss(x, x, sd, heads)
    lpips_ref.perceptual_loss(torch.rand(1, 2, 31, 31), torch.rand(1, 2, 31, 31), sd, heads)   # the smallest that works


def test_workspace_refuses_images_too_small_for_the_second_pool():
    L = _lib.lib()
    assert L.esr_lpips_param_bytes() > 0
    for H, W in ((24, 24), (30, 64), (64, 30), (32, 24)):
        assert L.esr_lpips_workspace_bytes(1, H, W) == 0, (H, W)
    for H, W in ((31, 31), (32, 32), (180, 320), (720, 1280)):
        assert L.esr_lpips_workspace_bytes(1, H, W) > 0, (H, W)
    assert L.esr_lpips_workspace_bytes(0, 64, 64) == 0
    with pytest.raises(_lib.ESRError, match="too small"):
        lpips.LPIPS.capacity(24, 24)
    assert lpips.LPIPS.capacity(720, 1280) >= 1


def _weights():
    sd = lpips_ref.seeded_alexnet(0)
    sd["classifier.1.weight"] = torch.zeros(4096, 9216)           # torchvision's checkpoint carries it; ignored
    return sd, lpips_ref.seeded_heads(1)


def test_weights_load_from_state_dicts_and_paths(tmp_path):
    sd, heads = _weights()
    lpips.LPIPS(sd, heads)
    torch.save(sd, tmp_path / "alexnet.pth")
    torch.save(heads, tmp_path / "alex.pth")
    m = lpips.LPIPS(str(tmp_path / "alexnet.pth"), str(tmp_path / "alex.pth"))
    assert len(m._params) == 15
    assert torch.equal(m._params[0], sd["features.0.weight"]) and torch.equal(m._params[14], heads["lin4.model.1.weight"])


@pytest.mark.parametrize("which, key, value, match", [
    ("alexnet", "features.3.weight", None, "no key features.3.weight"),
    ("alexnet", "features.6.bias", torch.zeros(383), "shape"),
    ("lin", "lin2.model.1.weight", None, "no key lin2"),
    ("lin", "lin0.model.1.weight", torch.zeros(1, 63, 1, 1), "shape"),
])
def test_missing_keys_and_wrong_shapes_raise(which, key, value, match):
    sd, heads = _weights()
    d = sd if which == "alexnet" else heads
    if value is None:
        del d[key]
    else:
        d[key] = value
    with pytest.raises(_lib.ESRError, match=match):
        lpips.LPIPS(sd, heads)


def test_missing_files_raise(tmp_path):
    sd, heads = _weights()
    with pytest.raises(_lib.ESRError, match="not found"):
        lpips.LPIPS(str(tmp_path / "nope.pth"), heads)
    with pytest.raises(_lib.ESRError, match="path or a state dict"):
        lpips.LPIPS(sd, 3)


def test_perceptual_loss_resolves_weights_at_the_first_call(tmp_path, monkeypatch):
    with pytest.raises(_lib.ESRError, match="only 'alex'"):
        lpips.perceptual_loss(net='vgg')
    monkeypatch.setattr(torch.hub, "get_dir", lambda: str(tmp_path / "hub"))
    loss = lpips.perceptual_loss()                                # constructing it needs no weights
    assert loss.model is None and loss.weight == 1.0
    x = torch.zeros(1, 2, 32, 32)
    _, heads = _weights()
    with pytest.raises(_lib.ESRError, match=lpips.TORCHVISION_ALEXNET):
        lpips.perceptual_loss(lin=heads)(x, x)                    # the hub-cache file the backbone falls back to
    sd, _ = _weights()
    ckpt = tmp_path / "hub" / "checkpoints"
    ckpt.mkdir(parents=True)
    torch.save(sd, ckpt / lpips.TORCHVISION_ALEXNET)
    loss = lpips.perceptual_loss(lin=heads)
    assert isinstance(loss._resolve(), lpips.LPIPS)
    with pytest.raises(_lib.ESRError, match="not found"):
        lpips.perceptual_loss(alexnet=sd, lin=str(tmp_path / "alex.pth"))(x, x)
