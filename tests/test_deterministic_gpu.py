"""Deterministic mode of the training operators (esr_b200.train.deterministic(): torch.use_deterministic_algorithms(True) or
torch.backends.cudnn.deterministic = True, as the reference trainer's init_seeds sets).

Operators: every case of the float64 tests of test_tc_fp64_gpu.py (k_wgrad_tc layers, DCNv2) and test_small_conv_fp64_gpu.py
(the narrow layers on every CUDA-core dispatch branch), and the fp32 cases of test_train_gpu.py, run in deterministic mode:
each passes its own tolerance (DESIGN.md 3), and every backward call is repeated on the same inputs and must give the same
bits.  Then the whole iteration: train_step at cfg2 size, CUDA-graph replays, the oracle loss trajectory, and the paths that
have no deterministic variant.
"""
import pytest
import torch

from oracle import model_ref
from tests import test_small_conv_fp64_gpu as sc
from tests import test_tc_fp64_gpu as tc
from tests import test_train_gpu as tg

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    import bench
    torch.set_num_threads(bench.usable_cores())
    return torch.device("cuda:0")


@pytest.fixture
def cudnn_det(monkeypatch):
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)


@pytest.fixture
def torch_det(monkeypatch):
    monkeypatch.setenv("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    yield
    torch.use_deterministic_algorithms(prev)


def _same_bits(a, b):
    if a is None or b is None:
        return a is None and b is None
    return a.shape == b.shape and torch.equal(a.detach().contiguous().view(torch.int32), b.detach().contiguous().view(torch.int32))


class _Repeat:
    """Wraps a backward function: records the inputs and outputs of every call; again() calls it once more on each recorded
    input and asserts bitwise equal outputs."""

    def __init__(self, fn):
        self.fn, self.calls = fn, []

    def __call__(self, *args, **kw):
        out = self.fn(*args, **kw)
        self.calls.append((args, kw, [None if t is None else t.clone() for t in out]))
        return out

    def again(self):
        from esr_b200 import train
        assert self.calls and train.deterministic()
        for args, kw, first in self.calls:
            second = self.fn(*args, **kw)
            for i, (a, b) in enumerate(zip(first, second)):
                assert _same_bits(a, b), (i, (a - b).abs().max().item() if a is not None and b is not None else None)


def _repeat_conv(monkeypatch):
    from esr_b200 import train
    rep = _Repeat(train._conv2d_backward_raw)
    monkeypatch.setattr(train, "_conv2d_backward_raw", rep)
    return rep


# ------------------------------------------------------------------------------------------------------------------ operators
@pytest.mark.parametrize("name", list(tc.TRAIN_CASES))
def test_tc_layer_deterministic_vs_fp64(dev, cudnn_det, monkeypatch, name):
    """k_wgrad_tc (per-slice partial tiles + ordered sum), the bias gradient from fp32 g, the deferred ConvGRU flush."""
    rep = _repeat_conv(monkeypatch)
    tc.test_train_conv2d_vs_fp64(dev, name)
    rep.again()


@pytest.mark.parametrize("name", list(sc.TRAIN_NARROW))
def test_narrow_layer_deterministic_vs_fp64(dev, cudnn_det, monkeypatch, name):
    """k_conv_wgrad_r / k_conv_wgrad_g<1> (per-split partials + ordered sum) and k_bias_grad's partials."""
    rep = _repeat_conv(monkeypatch)
    sc.test_train_narrow_conv2d_vs_fp64(dev, name)
    rep.again()


@pytest.mark.parametrize("B,Cin,Cout,k,stride,act,H,W", tg.CONV_CASES)
def test_conv2d_cases_deterministic(dev, cudnn_det, monkeypatch, B, Cin, Cout, k, stride, act, H, W):
    rep = _repeat_conv(monkeypatch)
    tg.test_conv2d_forward_backward_vs_torch(dev, B, Cin, Cout, k, stride, act, H, W)
    rep.again()


@pytest.mark.parametrize("case", ["production_96x32x32", "lattice_borders"])
def test_dcn_backward_deterministic_vs_fp64(dev, cudnn_det, monkeypatch, case):
    """grad_input in int64 fixed point, grad_weight / grad_bias from per-slice partials: the five gradients reproduce bit for
    bit and stay within test_tc_fp64_gpu's DCN tolerances."""
    from esr_b200 import dcn_v2_ext
    rep = _Repeat(dcn_v2_ext.dcn_v2_backward)
    monkeypatch.setattr(dcn_v2_ext, "dcn_v2_backward", rep)
    tc.test_dcn_v2_vs_fp64(dev, case)
    rep.again()


def test_dcn_colliding_samples_deterministic_vs_fp64(dev, cudnn_det):
    """Offsets that pull every sample of an image onto a 2 x 2 pixel neighbourhood of a few points: thousands of scattered
    values per grad_input element.  Bitwise reproducible and within the float64 tolerances."""
    from esr_b200 import dcn_v2_ext as ext
    g = torch.Generator().manual_seed(5)
    B, C, G, H, W = 4, 64, 8, 24, 40
    pts = torch.tensor([[3.25, 5.5], [11.75, 20.125], [20.5, 33.375]])
    pick = torch.randint(0, len(pts), (B, G, 9, H, W), generator=g)
    jitter = 0.4 * torch.rand(B, G, 9, 2, H, W, generator=g)
    yy = torch.arange(H).view(H, 1).float()
    xx = torch.arange(W).view(1, W).float()
    off = torch.empty(B, G, 9, 2, H, W)
    for kk in range(9):
        i, j = kk // 3, kk % 3
        off[:, :, kk, 0] = pts[pick[:, :, kk], 0] + jitter[:, :, kk, 0] - (yy - 1 + i)
        off[:, :, kk, 1] = pts[pick[:, :, kk], 1] + jitter[:, :, kk, 1] - (xx - 1 + j)
    off = off.reshape(B, G * 18, H, W)
    x = tc._rand(g, B, C, H, W)
    w = tc._rand(g, C, C, 3, 3, scale=1 / 24)
    b = tc._rand(g, C, scale=0.1)
    m = torch.rand(B, G * 9, H, W, generator=g)
    go = tc._rand(g, B, C, H, W)
    args = [t.to(dev) for t in (x, w, b, off, m)] + [go.to(dev)]
    got = [t.cpu() for t in ext.dcn_v2_backward(*args, 3, 3, 1, 1, 1, 1, 1, 1, G)]
    again = [t.cpu() for t in ext.dcn_v2_backward(*args, 3, 3, 1, 1, 1, 1, 1, 1, G)]
    for a, bb in zip(got, again):
        assert _same_bits(a, bb)

    leaves = [t.double().requires_grad_() for t in (x, off, m)]
    cols = tc.dcn_columns64(leaves[0], leaves[1], leaves[2], G)
    gcols = torch.einsum("ok,bohw->bkhw", w.reshape(C, C * 9).double(), go.double()).view_as(cols)
    ref = torch.autograd.grad(cols, leaves, gcols)
    gw = torch.einsum("bohw,bkhw->ok", go.double(), cols.detach().flatten(1, 2)).view(C, C, 3, 3)
    for name, got_, ref_ in zip(["grad_input", "grad_offset", "grad_mask"], got[:3], ref):
        tc.check(f"dcn_collide.{name}", f"dcn_{name}", got_, ref_, None)
    tc.check("dcn_collide.grad_weight", "dcn_grad_weight", got[3], gw, None)
    tc.check("dcn_collide.grad_bias", "dcn_grad_bias", got[4], go.double().sum((0, 2, 3)), None)


# ------------------------------------------------------------------------------------------------------------------ iterations
def _state(net, opt, losses):
    return {"losses": [l.clone() for l in losses], "log": opt.log.clone(),
            "grads": {n: p.grad.detach().clone() for n, p in net.named_parameters()},
            "params": opt.flat.clone(), "exp_avg": opt.exp_avg.clone(), "exp_avg_sq": opt.exp_avg_sq.clone(),
            "max_exp_avg_sq": opt.max_exp_avg_sq.clone(), "step": opt.step_dev.clone()}


def _assert_same_state(a, b):
    for i, (x, y) in enumerate(zip(a["losses"], b["losses"])):
        assert _same_bits(x, y), ("loss", i, x.item(), y.item())
    assert len(a["grads"]) == 68
    bad = [n for n in a["grads"] if not _same_bits(a["grads"][n], b["grads"][n])]
    assert not bad, bad
    for k in ("log", "params", "exp_avg", "exp_avg_sq", "max_exp_avg_sq", "step"):
        assert _same_bits(a[k], b[k]), k


def _cfg2_iterations(dev, sd, batches):
    from esr_b200 import train
    net = tg._net(sd, dev)
    opt = train.Adam(net.parameters(), lr=1e-3, weight_decay=1e-4, amsgrad=True)
    losses = [train.train_step(net, opt, f, g) for f, g in batches]
    torch.cuda.synchronize()
    return _state(net, opt, losses)


@pytest.mark.parametrize("switch", ["use_deterministic_algorithms", "cudnn.deterministic"])
def test_train_step_cfg2_bitwise_reproducible(dev, monkeypatch, switch):
    """Four train_step iterations at cfg2 size (B=8, L=8, 256 x 256), twice from the same seeded state: losses, the logging
    scalars, all 68 gradients, the parameters and the Adam moments are bitwise identical."""
    from esr_b200 import train
    monkeypatch.setenv("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    prev = torch.are_deterministic_algorithms_enabled()
    if switch == "cudnn.deterministic":
        monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    else:
        torch.use_deterministic_algorithms(True)
    try:
        assert train.deterministic()
        sd = model_ref.seeded_state_dict(81)
        batches = [tuple(t.to(dev) for t in tg._frames(8, 8, 256, 256, 200 + i, lam=0.1)) for i in range(4)]
        first = _cfg2_iterations(dev, sd, batches)
        second = _cfg2_iterations(dev, sd, batches)
        _assert_same_state(first, second)
    finally:
        torch.use_deterministic_algorithms(prev)


def test_graphed_train_step_bitwise(dev, torch_det):
    """Two separately captured GraphedTrainSteps replay bitwise identically, and equal the eager iterations bit for bit."""
    from esr_b200 import train
    sd = model_ref.seeded_state_dict(61)
    shape = (2, 4, 2, 32, 32)
    runs = []
    for _ in range(2):
        net = tg._net(sd, dev)
        opt = train.Adam(net.parameters(), lr=1e-3, weight_decay=1e-4, amsgrad=True)
        step = train.GraphedTrainStep(net, opt, shape, dev)
        losses = []
        for it in range(3):
            f, g = tg._frames(*shape[:2], *shape[3:], 100 + it)
            losses.append(step(f.to(dev), g.to(dev)).clone())
        torch.cuda.synchronize()
        runs.append(_state(net, opt, losses))
    _assert_same_state(runs[0], runs[1])
    net = tg._net(sd, dev)
    opt = train.Adam(net.parameters(), lr=1e-3, weight_decay=1e-4, amsgrad=True)
    losses = []
    for it in range(3):
        f, g = tg._frames(*shape[:2], *shape[3:], 100 + it)
        losses.append(train.train_step(net, opt, f.to(dev), g.to(dev)))
    torch.cuda.synchronize()
    _assert_same_state(_state(net, opt, losses), runs[0])


def test_deterministic_train_step_tracks_oracle_losses(dev, torch_det):
    tg.test_train_step_tracks_oracle_losses(dev)


# ------------------------------------------------------------------------------------------------------------------ errors
def test_generic_dcn_backward_raises_in_deterministic_mode(dev, cudnn_det):
    """The reference's own DCN test configuration (2 -> 2 channels, 1 group) runs on the generic kernels: no deterministic
    variant."""
    from esr_b200 import _lib
    from esr_b200 import dcn_v2_ext as ext
    B, C, H, W, G = 2, 2, 9, 11, 1
    x = torch.randn(B, C, H, W, device=dev)
    w = torch.randn(C, C, 3, 3, device=dev)
    b = torch.zeros(C, device=dev)
    off = torch.randn(B, G * 18, H, W, device=dev)
    m = torch.rand(B, G * 9, H, W, device=dev)
    with pytest.raises(_lib.ESRError, match="deterministic"):
        ext.dcn_v2_backward(x, w, b, off, m, torch.randn(B, C, H, W, device=dev), 3, 3, 1, 1, 1, 1, 1, 1, G)


def test_graphed_train_step_refuses_another_mode(dev, monkeypatch):
    from esr_b200 import _lib, train
    net = tg._net(model_ref.seeded_state_dict(3), dev)
    opt = train.Adam(net.parameters(), lr=1e-3, weight_decay=1e-4, amsgrad=True)
    shape = (1, 3, 2, 16, 16)
    step = train.GraphedTrainStep(net, opt, shape, dev)
    f, g = (t.to(dev) for t in tg._frames(1, 3, 16, 16, 1))
    step(f, g)
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    with pytest.raises(_lib.ESRError, match="deterministic mode off"):
        step(f, g)
