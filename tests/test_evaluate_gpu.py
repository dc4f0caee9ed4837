"""GPU: the count-image renderer and the batched evaluation loop against the reference (tests/golden/render_golden.npz,
eval_golden.npz), batching against one-at-a-time evaluation, the two window paths, and per-sample state resets."""
import os

import numpy as np
import pytest
import torch

from esr_b200 import evaluate, render
from esr_b200.eventstore import EventStore
from esr_b200.model import DeepRecurrNet
from oracle import model_ref
from tests import render_ref
from tests.test_evaluate import GOLD, golden_cnt, matches_golden, parse_option

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def _model(seed, N):
    net = DeepRecurrNet(inch=2, basech=8, num_frame=N)
    net.load_state_dict(model_ref.seeded_state_dict(seed, num_frame=N))
    return net.to(DEV).eval()


def _config(base, seql, step, seqn):
    c = eval(base) if isinstance(base, str) else dict(base)
    c["sequence"] = dict(c["sequence"], sequence_length=seql, step_size=step, seqn=seqn)
    return c


def _collect(model, stores, cfg, batch, chunk=4, consecutive=None):
    """(recording, window) -> CPU copies of esr, bicubic, gt, lr, scaled and the [2, 2, 6] statistics."""
    out = {}
    for st in evaluate.iter_windows(model, stores, cfg, batch=batch, chunk=chunk, consecutive=consecutive):
        for j, (r, w) in enumerate(zip(st["rec"], st["win"])):
            out[(r, w)] = {k: st[k][j].cpu() for k in ("esr", "bicubic", "gt", "lr", "scaled")}
            out[(r, w)]["stats"] = st["stats"][:, j].cpu()
    return out


# ---- renderer ---------------------------------------------------------------------------------------------------------
def test_render_matches_reference_golden():
    g = np.load(os.path.join(GOLD, "render_golden.npz"))
    n = 0
    for name in g["names"]:
        cnt = torch.from_numpy(golden_cnt(g, name)[None]).to(DEV)
        _, pct = render.render_event_cnt(cnt, return_percentiles=True)
        np.testing.assert_array_equal(pct[0].cpu().numpy(), g[f"{name}_pct"])
        for key in g[f"{name}_options"]:
            got = render.render_event_cnt(cnt, **parse_option(str(key)))[0].cpu().numpy()
            assert matches_golden(g, name, str(key), got), (name, key)
            n += 1
    assert n >= 200


def test_render_matches_numpy_on_1024_batches():
    rng = np.random.default_rng(3)
    cnt = np.stack([rng.poisson(0.8, (2, 1024, 1024)), rng.normal(0.3, 1.0, (2, 1024, 1024)),
                    rng.poisson(3.0, (2, 1024, 1024)) * (rng.random((2, 1024, 1024)) < 0.02)]).astype(np.float32)
    d = torch.from_numpy(cnt).to(DEV)
    _, pct = render.render_event_cnt(d, return_percentiles=True)
    want_pct = np.array([[[np.percentile(c[p], q) for q in (1, 99)] for p in range(2)] for c in cnt], np.float32)
    np.testing.assert_array_equal(pct.cpu().numpy(), want_pct)
    for opt in (dict(), dict(color_scheme="blue_red", is_black_background=False), dict(is_norm=False, use_opencv=True),
                dict(color_scheme="gray", use_opencv=True)):
        got = render.render_event_cnt(d, **opt).cpu().numpy()
        assert np.array_equal(got, render_ref.render(cnt, **opt)), opt


def test_render_refuses_gray_without_opencv():
    with pytest.raises(Exception):
        render.render_event_cnt(torch.zeros((1, 2, 4, 4), device=DEV), color_scheme="gray")


# ---- per-sample state reset ---------------------------------------------------------------------------------------------
def test_reset_sample_states_zeroes_one_sample():
    net = _model(3, 3)
    x = torch.poisson(torch.full((3, 3, 2, 32, 48), 0.8, device=DEV))
    with torch.no_grad():
        net.reset_states()
        net(x)
        before = torch.stack(net.states(3, 3, 32, 48))
        assert (before[:, 1] != 0).any()
        net.reset_sample_states([1])
        after = torch.stack(net.states(3, 3, 32, 48))
    assert torch.equal(after[:, 1], torch.zeros_like(after[:, 1]))          # both directions of sample 1
    assert torch.equal(after[:, 0], before[:, 0]) and torch.equal(after[:, 2], before[:, 2])


# ---- evaluation against the reference --------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def golden_store(tmp_path_factory):
    g = np.load(os.path.join(GOLD, "eval_golden.npz"))
    cols = {p: {k: g[f"{p}_{k}"] for k in ("xs", "ys", "ts", "ps")} for p in ("down4", "down2")}
    path = str(tmp_path_factory.mktemp("eval") / "eval.esr")
    EventStore.write(path, cols, g["sensor"])
    return g, EventStore(path)


@pytest.mark.parametrize("name", ["s1n3", "snone", "clamp", "s1n5"])
def test_evaluate_matches_reference(golden_store, name):
    g, store = golden_store
    seql, step, seqn, wseed, _, n = (int(v) for v in g[f"{name}_meta"])
    cfg = _config(str(g["config"][0]), seql, None if step < 0 else step, seqn)
    net = _model(wseed, seqn)
    got = _collect(net, [store], cfg, batch=1)
    assert sorted(got) == [(0, w) for w in range(n)]
    esr = torch.stack([got[(0, w)]["esr"] for w in range(n)]).numpy()
    bic = torch.stack([got[(0, w)]["bicubic"] for w in range(n)]).numpy()
    gt = torch.stack([got[(0, w)]["gt"] for w in range(n)]).numpy()
    np.testing.assert_array_equal(gt, g[f"{name}_gt"])
    want = g[f"{name}_esr"]
    assert np.abs(esr - want).max() <= 1e-3 * np.abs(want).max()
    wb = g[f"{name}_bicubic"]
    assert np.abs(bic - wb).max() <= 1e-6 * np.abs(wb).max()
    res, mean = evaluate.evaluate_recordings(net, [store], cfg, batch=1)
    peak = np.abs(want).max()
    for key, tol in (("esr_l1", 1e-3 * peak), ("esr_mse", 1e-3 * peak), ("esr_ssim", 1e-3), ("esr_psnr", 1e-2),
                     ("bicubic_l1", 1e-6), ("bicubic_mse", 1e-6), ("bicubic_ssim", 1e-6), ("bicubic_psnr", 1e-4)):
        ref = float(np.mean(g[f"{name}_{key}"]))
        assert abs(res[key]["eval.esr"] - ref) <= tol, (key, res[key]["eval.esr"], ref)
        assert mean[key] == res[key]["eval.esr"]
    assert res["params"]["eval.esr"] == sum(p.numel() for p in net.parameters()) / 1e6
    assert res["time"]["eval.esr"] > 0
    assert set(res) == set(evaluate.METRIC_KEYS)


# ---- batching ----------------------------------------------------------------------------------------------------------
def _synth_store(path, seed, length, sensor=(64, 96)):
    """a recording of `length` dataset frames at the golden config (window 160, sliding 40 -> 120 events per frame)"""
    rng = np.random.default_rng(seed)
    cols = {}
    for prex, div, per in (("down4", 4, 120), ("down2", 2, 480)):
        n = length * per + 8
        H, W = sensor[0] // div, sensor[1] // div
        cols[prex] = {"xs": rng.integers(0, W, n), "ys": rng.integers(0, H, n), "ts": np.sort(rng.random(n)) + 1.0,
                      "ps": rng.choice([-1.0, 1.0], n)}
    EventStore.write(path, cols, sensor)
    return EventStore(path)


@pytest.fixture(scope="module")
def ragged(tmp_path_factory):
    d = tmp_path_factory.mktemp("ragged")
    stores = [_synth_store(str(d / f"rec{i}.esr"), 40 + i, L) for i, L in enumerate((12, 20, 10, 16, 11))]
    g = np.load(os.path.join(GOLD, "eval_golden.npz"))
    return stores, str(g["config"][0])


def _assert_same(a, b):
    assert sorted(a) == sorted(b)
    for k in a:
        for f in a[k]:
            assert torch.equal(a[k][f], b[k][f]), (k, f)


@pytest.mark.parametrize("step", [1, None])
def test_batched_is_bit_identical_to_one_at_a_time(ragged, step, tmp_path):
    stores, base = ragged
    cfg = _config(base, 9, step, 3)
    net = _model(3, 3)
    one = _collect(net, stores, cfg, batch=1)
    three = _collect(net, stores, cfg, batch=3)                              # 5 recordings: slots refill
    _assert_same(one, three)
    # a recording evaluated after others in the same slot equals a fresh run of it alone
    fresh = _collect(_model(3, 3), stores[3:4], cfg, batch=1)
    _assert_same({(0, w): v for (r, w), v in one.items() if r == 3}, fresh)
    if step == 1:                                                            # the frame-bank path gives the same outputs
        _assert_same(one, _collect(net, stores, cfg, batch=3, consecutive=False))
    # results and images
    r1, m1 = evaluate.evaluate_recordings(net, stores, cfg, batch=1, image_dir=str(tmp_path / "b1"))
    r3, m3 = evaluate.evaluate_recordings(net, stores, cfg, batch=3, image_dir=str(tmp_path / "b3"))
    for key in evaluate.METRIC_KEYS:
        if key != "time":
            assert r1[key] == r3[key] and m1[key] == m3[key], key
    n_img = 0
    for s in stores:
        nm = os.path.basename(s.path)
        for kind in evaluate.IMAGE_KINDS:
            d1, d3 = tmp_path / "b1" / nm / "event_img" / kind, tmp_path / "b3" / nm / "event_img" / kind
            files = sorted(os.listdir(d1))
            assert files == sorted(os.listdir(d3)) and files[0] == "000000000.png"
            for f in files:
                assert (d1 / f).read_bytes() == (d3 / f).read_bytes()
                n_img += 1
    assert n_img == 5 * sum(1 for (r, w) in one)


def test_images_are_the_rendered_arrays(ragged, tmp_path):
    from PIL import Image
    stores, base = ragged
    cfg = _config(base, 9, 1, 3)
    net = _model(3, 3)
    frames = _collect(net, stores[:1], cfg, batch=1)
    evaluate.evaluate_recordings(net, stores[:1], cfg, batch=1, image_dir=str(tmp_path))
    root = tmp_path / os.path.basename(stores[0].path) / "event_img"
    f = frames[(0, 2)]
    for kind, src in (("lr_event_img", f["lr"]), ("hr_scaled_event_img", f["scaled"]), ("hr_bicubic_event_img", f["bicubic"]),
                      ("hr_esr_event_img", f["esr"].round()), ("hr_gt_event_img", f["gt"])):
        img = np.asarray(Image.open(root / kind / "000000002.png"))
        assert np.array_equal(img, render_ref.render(src.numpy()[None])[0]), kind
