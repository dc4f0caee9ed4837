"""GPU: LPIPS (esr_lpips_forward) against the reference's values (tests/golden/lpips_golden.npz) and the float64 restatement
(tests/lpips_ref.py), its invariants (LPIPS(x, x) = 0, a pair alone = the pair in a batch, graph replay = eager), the
perceptual_loss wrapper's channel rules, the 5x5 tensor-core convolution, and esr_lpips / bicubic_lpips in the evaluation."""
import ctypes
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from esr_b200 import _lib, evaluate, layers, lpips
from tests import lpips_ref
from tests.test_evaluate_gpu import _config, _model, _synth_store
from tests.test_lpips import GOLD, golden

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
SD = lpips_ref.seeded_alexnet(0)
TOL = 1e-4


@pytest.fixture(scope="module")
def heads():
    return golden()[1]


@pytest.fixture(scope="module")
def model(heads):
    return lpips.LPIPS(SD, heads)


def _oracle64(a, b, heads, normalize=True):
    """LPIPS of image a vs image b ([3, H, W]) in float64 on the GPU."""
    return lpips_ref.pair_distance(a.to(DEV, torch.float64), b.to(DEV, torch.float64), SD, heads, normalize)


def test_reference_golden_values(heads):
    g = np.load(GOLD)
    loss = lpips.perceptual_loss(alexnet=SD, lin=heads)
    for name in g["cases"]:
        pred, target = torch.from_numpy(g[f"{name}/pred"]).to(DEV), torch.from_numpy(g[f"{name}/target"]).to(DEV)
        v = loss(pred, target, normalize=bool(g[f"{name}/normalize"]))
        assert v.is_cuda and v.dim() == 0 and v.dtype == torch.float32
        ref = float(g[f"{name}/fp64"])
        rel = abs(float(v) - ref) / ref
        print(f"[lpips] golden {name}: {float(v):.9g} vs {ref:.9g}, rel {rel:.2e}")
        assert rel <= TOL, name


@pytest.mark.parametrize("H, W, n", [(720, 1280, 2), (180, 320, 6), (90, 160, 4), (31, 31, 3), (33, 47, 2), (97, 61, 2)])
def test_random_shapes_vs_fp64(model, heads, H, W, n):
    g = torch.Generator().manual_seed(H * 7 + W)
    planes = torch.poisson(torch.rand((2 * n, H, W), generator=g) * 3.0, generator=g)
    planes[n:] += torch.randn((n, H, W), generator=g) * 0.5              # bicubic-like: negative values too
    src = np.repeat(np.arange(2 * n), 3).reshape(-1, 3)
    got = model.distances(planes.to(DEV), src, np.arange(n), np.arange(n, 2 * n)).cpu()
    worst = 0.0
    for p in range(n):
        ref = _oracle64(planes[p].expand(3, H, W), planes[n + p].expand(3, H, W), heads)
        worst = max(worst, abs(float(got[p]) - ref) / ref)
    print(f"[lpips] {H} x {W}: worst relative error {worst:.2e} over {n} pairs")
    assert worst <= TOL


def test_rgb_and_no_normalize_vs_fp64(model, heads):
    g = torch.Generator().manual_seed(5)
    planes = torch.rand((12, 64, 80), generator=g) * 2 - 1
    src = np.arange(12).reshape(4, 3)
    for normalize in (True, False):
        got = model.distances(planes.to(DEV), src, [0, 2], [1, 3], normalize=normalize).cpu()
        for p, (a, b) in enumerate(((0, 1), (2, 3))):
            ref = _oracle64(planes[3 * a:3 * a + 3], planes[3 * b:3 * b + 3], heads, normalize)
            assert abs(float(got[p]) - ref) <= TOL * ref


def test_identical_images_give_zero(model):
    x = torch.poisson(torch.full((2, 96, 128), 2.0)).to(DEV)
    planes = torch.cat([x, x])
    src = np.repeat(np.arange(4), 3).reshape(-1, 3)
    d = model.distances(planes, src, [0, 1, 0, 1], [2, 3, 0, 1])
    assert torch.equal(d, torch.zeros_like(d))


def test_a_pair_alone_equals_the_pair_in_a_batch(model):
    g = torch.Generator().manual_seed(11)
    planes = torch.poisson(torch.rand((48, 90, 160), generator=g) * 4.0, generator=g).to(DEV)
    src = np.repeat(np.arange(48), 3).reshape(-1, 3)
    batch = model.distances(planes, src, np.arange(24), np.arange(24, 48))
    for p in (0, 7, 23):
        alone = model.distances(planes, src, [p], [24 + p])
        assert torch.equal(alone, batch[p:p + 1]), p


def test_graph_replay_equals_eager(model):
    H, W, n = 180, 320, 6
    g = torch.Generator().manual_seed(12)
    planes = torch.poisson(torch.rand((n, H, W), generator=g) * 3.0, generator=g).to(DEV)
    plan = model._plan(n, H, W, DEV)
    idx = torch.tensor(np.concatenate([np.repeat(np.arange(n), 3), [0, 1, 2], [3, 4, 5]]), dtype=torch.int32, device=DEV)
    L = _lib.lib()
    out = torch.zeros(3, dtype=torch.float64, device=DEV)

    def run():
        _lib.check(L.esr_lpips_forward(plan.handle, _lib.ptr(planes), _lib.ptr(idx), n, 1, 3, ctypes.c_void_p(idx.data_ptr() + 4 * 3 * n),
                                       ctypes.c_void_p(idx.data_ptr() + 4 * (3 * n + 3)), _lib.ptr(out), _lib.stream_ptr()),
                   "esr_lpips_forward")
    run()
    torch.cuda.synchronize()
    eager = out.clone()
    out.zero_()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            run()
    torch.cuda.current_stream().wait_stream(s)
    out.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, eager)
    assert torch.equal(eager, model.distances(planes, idx[:3 * n].cpu().numpy().reshape(-1, 3), [0, 1, 2], [3, 4, 5]))


def test_perceptual_loss_channel_rules_and_errors(heads):
    loss = lpips.perceptual_loss(weight=0.5, alexnet=SD, lin=heads)
    g = torch.Generator().manual_seed(13)
    for shape in ((2, 1, 48, 64), (2, 3, 48, 64), (1, 2, 48, 64), (1, 4, 40, 40)):
        pred, target = torch.rand(shape, generator=g), torch.rand(shape, generator=g)
        ref = 0.5 * float(lpips_ref.perceptual_loss(pred.to(DEV, torch.float64), target.to(DEV, torch.float64), SD, heads))
        got = float(loss(pred.to(DEV), target.to(DEV)))
        assert abs(got - ref) <= TOL * ref, shape
    x = torch.rand((2, 2, 40, 40), device=DEV)
    with pytest.raises(RuntimeError):                                     # the reference: 1 x 6-channel input to AlexNet
        loss(x, x)
    y = torch.rand((1, 2, 24, 24), device=DEV)
    with pytest.raises(RuntimeError):                                     # the reference: max-pool output size 0
        loss(y, y)
    with pytest.raises(AssertionError):
        loss(x[:1], y)


def test_conv5x5_vs_fp64_at_evaluation_tile_counts():
    """AlexNet's conv2 (64 -> 192, 5x5, pad 2) on k_conv_tc<192, 5> at the pool1 sizes of 180 x 320 (12 images: one
    evaluation step of 2 windows x 3 kinds x 2 channels) and 720 x 1280 (2 images)."""
    g = torch.Generator().manual_seed(14)
    w = torch.randn((192, 64, 5, 5), generator=g) * (2.0 / 1600) ** 0.5
    b = torch.rand((192,), generator=g) * 0.1
    wp, bp = layers.pack_weight(w.to(DEV)), layers.pad_bias(b.to(DEV), 192)
    for n, H, W in ((12, 21, 39), (2, 89, 159)):
        x = torch.relu(torch.randn((n, 64, H, W), generator=g))
        out = layers.Split(n, 192, H, W, DEV)
        layers.conv_tc([layers.Split.from_nchw(x.to(DEV))], wp, bp, 192, ntaps=25, act="relu", out=out)
        got = out.to_nchw().cpu().double()
        ref = torch.relu(F.conv2d(x.double(), w.double(), b.double(), padding=2))
        err = (got - ref).abs().max().item() / ref.abs().max().item()
        print(f"[lpips] conv 5x5 {n} x {H} x {W}: max error / max value {err:.2e}")
        assert err <= 2e-5


def test_conv1_vs_fp64_through_the_first_head(heads):
    """conv1 (11x11 / 4 with the input transform) alone decides the distance when only the first head is non-zero."""
    only0 = {k: (v if k.startswith("lin0") else torch.zeros_like(v)) for k, v in heads.items()}
    m = lpips.LPIPS(SD, only0)
    g = torch.Generator().manual_seed(15)
    for H, W, n in ((180, 320, 12), (720, 1280, 2)):
        planes = torch.poisson(torch.rand((2 * n, H, W), generator=g) * 3.0, generator=g)
        src = np.repeat(np.arange(2 * n), 3).reshape(-1, 3)
        got = m.distances(planes.to(DEV), src, np.arange(n), np.arange(n, 2 * n)).cpu()
        for p in range(n):
            ref = _oracle64(planes[p].expand(3, H, W), planes[n + p].expand(3, H, W), only0)
            assert abs(float(got[p]) - ref) <= 2e-5 * ref, (H, W, p)


@pytest.fixture(scope="module")
def recordings(tmp_path_factory):
    d = tmp_path_factory.mktemp("lpips_eval")
    stores = [_synth_store(str(d / f"rec{i}.esr"), 60 + i, L) for i, L in enumerate((12, 20, 10))]
    g = np.load(os.path.join(os.path.dirname(GOLD), "eval_golden.npz"))
    return stores, str(g["config"][0])


@pytest.mark.parametrize("step", [1, None])
def test_evaluate_recordings_with_lpips(model, heads, recordings, step):
    stores, base = recordings
    cfg = _config(base, 9, step, 3)
    net = _model(3, 3)
    plain, plain_mean = evaluate.evaluate_recordings(net, stores, cfg, batch=2)
    res3, mean3 = evaluate.evaluate_recordings(net, stores, cfg, batch=3, lpips=model)
    res1, mean1 = evaluate.evaluate_recordings(net, stores, cfg, batch=1, lpips=model)
    assert set(plain) == set(evaluate.METRIC_KEYS)
    assert set(res3) == set(evaluate.METRIC_KEYS) | set(evaluate.LPIPS_KEYS)
    for key in evaluate.METRIC_KEYS:
        if key != "time":
            assert res3[key] == plain[key], key
    for key in evaluate.LPIPS_KEYS:
        assert res3[key] == res1[key] and mean3[key] == mean1[key], key
    # the oracle on the same planes, averaged the same way
    per = {}
    for st in evaluate.iter_windows(net, stores, cfg, batch=1):
        for j, (r, w) in enumerate(zip(st["rec"], st["win"])):
            gt = st["gt"][j].cpu()
            for kind in ("esr", "bicubic"):
                x = st[kind][j].cpu()
                v = sum(_oracle64(x[c].expand(3, *x.shape[-2:]), gt[c].expand(3, *x.shape[-2:]), heads) for c in range(2)) / 2
                per.setdefault((r, kind), []).append((w, v))
    for r, s in enumerate(stores):
        name = os.path.basename(s.path)
        for kind in ("esr", "bicubic"):
            vals = [v for _, v in sorted(per[(r, kind)])]
            ref = sum(vals) / len(vals)
            assert abs(res3[f"{kind}_lpips"][name] - ref) <= TOL * ref, (name, kind)
