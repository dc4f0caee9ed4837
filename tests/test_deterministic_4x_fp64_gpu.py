"""Deterministic mode against float64 at the benchmark's 4x configurations: every deterministic reduction at cfg4's counts,
and the graphed deterministic iteration at cfg3 and cfg4.

Deterministic mode (esr_b200.train.deterministic(), which the reference trainer's init_seeds turns on through
torch.backends.cudnn.deterministic) replaces every fp32 atomic reduction of the backward: k_wgrad_tc_det adds its flushes
in order to its slice's slot, k_conv_wgrad_r_det / k_conv_wgrad_g_det<1> / k_bias_grad_det / k_dcn_wgrad_det /
k_dcn_bgrad_det write per-block partials that k_sum_slices adds in slot order, and the DCN grad_input accumulates in int64
fixed point.  At cfg4 those chains are far longer than at cfg2 (test_chain_lengths_at_cfg4 prints them), so this module
runs them there:

  1. the chain lengths cfg4 reaches, from the launch rules (and a CPU test that the rules' constants are the kernels');
  2. every convolution of test_train_4x_fp64_gpu.CONV4 through train.conv2d in deterministic mode, the ConvGRU gates
     deferred over 42 steps: y / dx / dw / db against float64 under TOL4, every backward call repeated bit for bit;
  3. DCN backward at DCN4 (56 x 64 x 128²) with random and lattice offsets, and with every sample of an image pulled onto
     three points: float64 bars, bitwise repeats (the default mode's fp32-atomic error is printed beside it);
  4. in 2 and 3, every workspace is the first nbytes of a longer buffer whose tail holds a sentinel, so a partial buffer
     sized too small by esr_conv2d_workspace_bytes_ex / esr_dcn_v2_backward_workspace_bytes_ex shows up as a changed tail;
  5. one GraphedTrainStep replay at cfg4 on bench.py's weights and inputs against float64, a second capture and an eager
     train_step from the same state bit for bit equal to it; at cfg3 the eager step equals the replay bit for bit.

Norm and rule: err = max|got - ref64| / max|ref64| <= TOL <= err(degraded) / 4 (tests/test_tc_fp64_gpu.py).
"""
import math
import os
import re
import time

import pytest
import torch

from tests import test_train_4x_fp64_gpu as t4
from tests.test_deterministic_gpu import _Repeat, _assert_same_state, _same_bits, _state
from tests.test_small_conv_fp64_gpu import train_branches
from tests.test_tc_fp64_gpu import dcn_columns64, rel, wgrad_geometry

pytestgpu = pytest.mark.gpu

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "esr_b200", "csrc")

# launch constants of the deterministic reductions (test_launch_constants_are_the_kernels ties them to the sources)
WG_FLUSH_TILES = 32     # k_wgrad_tc: tiles accumulated in registers between two flushes to the slot
WG_PSL = 512            # k_dcn_wgrad: pixels per slot
BG_BLOCKS = 148         # k_dcn_bgrad: blocks of 4 pixel lanes
WR_NSPLIT = 10          # k_conv_wgrad_r: pixel splits per block (k_conv_wgrad_g<1>: 256 / G_C)
G_C = 8                 # k_conv_wgrad_r / _g: channels per block side


@pytest.fixture(scope="module")
def dev():
    import bench
    torch.set_num_threads(bench.usable_cores())
    return torch.device("cuda:0")


@pytest.fixture
def cudnn_det(monkeypatch):
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)


# ------------------------------------------------------------------------------------------------------------------
# 1. chain lengths at cfg4
# ------------------------------------------------------------------------------------------------------------------
def test_launch_constants_are_the_kernels():
    src = {f: open(os.path.join(CSRC, f)).read() for f in ("wgrad_tc.cu", "dcn_bwd.cu", "train_ops.cu")}
    for f, name, v in (("wgrad_tc.cu", "WG_FLUSH_TILES", WG_FLUSH_TILES), ("dcn_bwd.cu", "WG_PSL", WG_PSL),
                       ("dcn_bwd.cu", "BG_BLOCKS", BG_BLOCKS), ("train_ops.cu", "WR_NSPLIT", WR_NSPLIT),
                       ("train_ops.cu", "G_C", G_C)):
        m = re.search(rf"constexpr int (?:\w+ = \d+, )*{name} = (\d+)[,;]", src[f])
        assert m and int(m.group(1)) == v, (f, name, m and m.group(0))
    # the slot count of the CUDA-core weight gradients: about 8 blocks per SM, at most one per (image, tile) item
    assert "int slices = (dev_info().sm_count * 8 + pairs - 1) / pairs;" in src["train_ops.cu"]
    assert "return ksz == 3 ? WR_NSPLIT : 256 / G_C;" in src["train_ops.cu"]


def narrow_slots(sm, B, Cin, Cout, k, stride, H, W):
    """k_conv_wgrad_r_det / k_conv_wgrad_g_det<1>: (slots k_sum_slices adds, output pixels per slot)."""
    Ho, Wo = (H + 2 * (k // 2) - k) // stride + 1, (W + 2 * (k // 2) - k) // stride + 1
    pairs = math.ceil(Cout / G_C) * math.ceil(Cin / G_C)
    items = B * math.ceil(Wo / 16) * math.ceil(Ho / 16)
    slices = max(1, min(math.ceil(sm * 8 / pairs), items))
    slots = slices * (WR_NSPLIT if k == 3 else 256 // G_C)
    return slots, B * Ho * Wo / slots


def _flushes(geo):
    return math.ceil(math.ceil(geo["n_tiles"] / geo["slices"]) / WG_FLUSH_TILES)


@pytestgpu
def test_chain_lengths_at_cfg4(dev):
    """The cfg4 cases of this module reach the long chains: >= 31 flushes added into one k_wgrad_tc_det slot (gru_zr),
    >= 1 792 k_dcn_wgrad_det slots summed by k_sum_slices, each 8x the pixels of a cfg2 slot in the narrow layers."""
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    rows = []
    for gate, cout in (("gru_zr", 128), ("gru_o", 64)):
        g2, g4 = wgrad_geometry(288, 128, cout, 3, 32, 32), wgrad_geometry(168, 128, cout, 3, 128, 128)
        rows.append((f"k_wgrad_tc_det {gate}: tiles per CTA -> flushes per slot (slots)",
                     f"{g2['tiles_per_cta']} -> {_flushes(g2)} ({g2['slices']})", f"{g4['tiles_per_cta']} -> {_flushes(g4)} ({g4['slices']})"))
        if gate == "gru_zr":
            assert _flushes(g4) >= 31, g4
        else:
            assert _flushes(g4) >= 16, g4
    B, C, H, W = t4.DCN4
    px2, px4 = 96 * 32 * 32, B * H * W
    slots2, slots4 = math.ceil(px2 / WG_PSL), math.ceil(px4 / WG_PSL)
    rows.append(("k_dcn_wgrad_det slots (MB of partials)", f"{slots2} ({slots2 * 64 * 64 * 9 * 4 / 1e6:.0f})",
                 f"{slots4} ({slots4 * 64 * 64 * 9 * 4 / 1e6:.0f})"))
    assert slots4 >= 1792
    rows.append(("k_dcn_bgrad_det pixels per thread (slots)", f"{math.ceil(px2 / (BG_BLOCKS * 4))} ({BG_BLOCKS * 4})",
                 f"{math.ceil(px4 / (BG_BLOCKS * 4))} ({BG_BLOCKS * 4})"))
    rows.append(("DCN fixed point: image H*W in 2^62 / (288 H W max)", f"{32 * 32}", f"{H * W} "
                 f"({int(math.log2(H * W / 1024))} bits less resolution)"))
    s2, p2 = narrow_slots(sm, 64, 2, 8, 3, 1, 256, 256)                   # head_2_8 at cfg2: 64 frames of 256²
    s4, p4 = narrow_slots(sm, t4.CONV4["head_2_8"][5], 2, 8, 3, 1, 1024, 1024)    # 32 frames of 1024²
    rows.append(("k_conv_wgrad_r_det head_2_8: slots, pixels per slot", f"{s2}, {p2:.0f}", f"{s4}, {p4:.0f}"))
    assert p4 >= 8 * p2
    print(f"\n[det4x] chain lengths on {torch.cuda.get_device_name(0)} ({sm} SMs): cfg2 | cfg4")
    for r in rows:
        print(f"[det4x]   {r[0]}: {r[1]} | {r[2]}")
    for name, c in t4.CONV4.items():
        Cin, Cout, k, stride, act, n, H_, W_, launches = c
        steps = launches if name.startswith("gru") else 1
        if train_branches(Cin, Cout, k, stride, act)[2] == "k_wgrad_tc":
            g = wgrad_geometry(n * steps, Cin, Cout, k, H_, W_)
            print(f"[det4x]   {name}: k_wgrad_tc_det {g['slices']} slots, {_flushes(g)} flushes per slot")
        else:
            s, p = narrow_slots(sm, n * steps, Cin, Cout, k, stride, H_, W_)
            print(f"[det4x]   {name}: k_conv_wgrad_*_det {s} slots of {p:.0f} pixels")


# ------------------------------------------------------------------------------------------------------------------
# 4. workspace guard (used by 2 and 3)
# ------------------------------------------------------------------------------------------------------------------
class _Guard:
    """Stands in for a workspace allocator: hands out the first nbytes of a buffer TAIL bytes longer, whose tail holds a
    seeded random pattern; check() asserts that no call wrote past the nbytes it was given."""
    TAIL = 4 << 20

    def __init__(self, dev):
        g = torch.Generator(device=dev).manual_seed(0x5e17)
        self.pattern = torch.randint(0, 256, (self.TAIL,), generator=g, device=dev, dtype=torch.uint8)
        self.bufs = []

    def __call__(self, nbytes, device):
        n = max(int(nbytes), 256)                                   # what train._ws / dcn_v2_ext._ws hand out
        buf = torch.empty((n + self.TAIL,), dtype=torch.uint8, device=device)
        buf[n:].copy_(self.pattern)
        self.bufs.append((buf, n))
        return buf[:n]

    def check(self, what):
        assert self.bufs, what
        bad = [n for buf, n in self.bufs if not torch.equal(buf[n:], self.pattern)]
        print(f"[det4x] {what}: {len(self.bufs)} workspaces, largest {max(n for _, n in self.bufs) / 2**20:.1f} MiB, "
              f"{len(bad)} written past their end")
        assert not bad, (what, bad)
        self.bufs.clear()


# ------------------------------------------------------------------------------------------------------------------
# 2. every cfg4 convolution in deterministic mode
# ------------------------------------------------------------------------------------------------------------------
@pytestgpu
@pytest.mark.parametrize("name", list(t4.CONV4))
def test_conv2d_cfg4_deterministic_vs_fp64(dev, cudnn_det, monkeypatch, name):
    """test_train_conv2d_cfg4_vs_fp64 in deterministic mode: y / dx / dw / db within TOL4 (dw through k_wgrad_tc_det or
    k_conv_wgrad_*_det and k_sum_slices, db through k_bias_grad_det), every backward call repeated bit for bit, and no
    workspace written past the size esr_conv2d_workspace_bytes_ex reported."""
    from esr_b200 import train
    guard = _Guard(dev)
    monkeypatch.setattr(train, "_ws", guard)
    rep = _Repeat(train._conv2d_backward_raw)
    monkeypatch.setattr(train, "_conv2d_backward_raw", rep)
    t4.test_train_conv2d_cfg4_vs_fp64(dev, name)
    guard.check(f"{name} workspaces")
    rep.again()
    guard.check(f"{name} workspaces of the repeated backward calls")
    print(f"[det4x] {name}: {len(rep.calls)} backward calls repeated bit for bit")
    rep.calls.clear()
    t4._free()


# ------------------------------------------------------------------------------------------------------------------
# 3. DCN backward at cfg4's counts in deterministic mode
# ------------------------------------------------------------------------------------------------------------------
@pytestgpu
@pytest.mark.parametrize("offsets", ["random", "lattice"])
def test_dcn_cfg4_deterministic_vs_fp64(dev, cudnn_det, monkeypatch, offsets):
    """test_dcn_cfg4_vs_fp64 in deterministic mode: the five gradients within TOL4, the backward repeated bit for bit,
    no workspace written past its reported size."""
    from esr_b200 import dcn_v2_ext
    guard = _Guard(dev)
    monkeypatch.setattr(dcn_v2_ext, "_ws", guard)
    rep = _Repeat(dcn_v2_ext.dcn_v2_backward)
    monkeypatch.setattr(dcn_v2_ext, "dcn_v2_backward", rep)
    t4.test_dcn_cfg4_vs_fp64(dev, offsets)
    guard.check(f"dcn_{offsets} workspaces")
    rep.again()
    guard.check(f"dcn_{offsets} workspaces of the repeated backward")
    rep.calls.clear()
    t4._free()


def colliding_offsets(gen, B, G, H, W, pts):
    """Offsets that pull every sample of every image onto the 2 x 2 pixel neighbourhood of one of `pts` (each sample
    picks a point, plus a jitter in [0, 0.4)), -> (offsets [B, G*18, H, W], picks [B, G, 9, H, W])."""
    dev = gen.device
    pick = torch.randint(0, len(pts), (B, G, 9, H, W), generator=gen, device=dev)
    jitter = 0.4 * torch.rand(B, G, 9, 2, H, W, generator=gen, device=dev)
    pts = torch.tensor(pts, device=dev)
    yy = torch.arange(H, device=dev).view(H, 1).float()
    xx = torch.arange(W, device=dev).view(1, W).float()
    off = torch.empty(B, G, 9, 2, H, W, device=dev)
    for kk in range(9):
        i, j = kk // 3, kk % 3
        off[:, :, kk, 0] = pts[pick[:, :, kk], 0] + jitter[:, :, kk, 0] - (yy - 1 + i)
        off[:, :, kk, 1] = pts[pick[:, :, kk], 1] + jitter[:, :, kk, 1] - (xx - 1 + j)
    return off.reshape(B, G * 18, H, W), pick


def dcn_grads64(x, w, off, m, go, G, chunk=4):
    """The five DCN gradients in float64 on x's device, a few images at a time, and the degraded ones: the column
    gradients from split weights and go without its lo plane (A_lo B_hi dropped), grad_weight from features without
    their lo plane.  -> (ref, deg) dicts keyed grad_input ... grad_bias."""
    B, C, H, W = x.shape
    w2 = w.reshape(C, C * 9)
    w2h, w2l = t4.split_dev(w2)
    w2s = w2h.double() + w2l.double()
    names = ["grad_input", "grad_offset", "grad_mask"]
    ref = {n: [] for n in names}
    deg = {n: [] for n in names}
    gw, gw_deg = (torch.zeros(C, C * 9, dtype=torch.float64, device=x.device) for _ in range(2))
    for i in range(0, B, chunk):
        sl = slice(i, i + chunk)
        leaves = [t[sl].double().requires_grad_() for t in (x, off, m)]
        cols = dcn_columns64(leaves[0], leaves[1], leaves[2], G)
        gcols = torch.einsum("ok,bohw->bkhw", w2.double(), go[sl].double()).view_as(cols)
        gcols_deg = torch.einsum("ok,bohw->bkhw", w2s, t4.split_dev(go[sl])[0].double()).view_as(cols)
        for n_, e_, d_ in zip(names, torch.autograd.grad(cols, leaves, gcols, retain_graph=True),
                              torch.autograd.grad(cols, leaves, gcols_deg)):
            ref[n_].append(e_)
            deg[n_].append(d_)
        gw += torch.einsum("bohw,bkhw->ok", go[sl].double(), cols.detach().flatten(1, 2))
        with torch.no_grad():
            cols_hi = dcn_columns64(t4.split_dev(x[sl])[0].double(), off[sl].double(), m[sl].double(), G)
        gw_deg += torch.einsum("bohw,bkhw->ok", go[sl].double(), cols_hi.flatten(1, 2))
        del leaves, cols, gcols, gcols_deg, cols_hi
    ref = {n: torch.cat(v, 0) for n, v in ref.items()}
    deg = {n: torch.cat(v, 0) for n, v in deg.items()}
    ref["grad_weight"], deg["grad_weight"] = gw.view(C, C, 3, 3), gw_deg.view(C, C, 3, 3)
    ref["grad_bias"], deg["grad_bias"] = go.double().sum((0, 2, 3)), None
    return ref, deg


DCN_NAMES = ["grad_input", "grad_offset", "grad_mask", "grad_weight", "grad_bias"]


@pytestgpu
def test_dcn_colliding_samples_cfg4_deterministic_vs_fp64(dev, cudnn_det, monkeypatch):
    """Every sample of each of the 56 images of 128² pulled onto the 2 x 2 neighbourhood of one of three points: each of
    those grad_input elements adds ~5e4 scattered values in int64 fixed point, whose scale leaves 4 bits less resolution
    than at cfg2's 32².  Bitwise repeatable, within TOL4 and no workspace written past its end; the default mode's
    fp32-atomic error on the same inputs is printed beside it."""
    from esr_b200 import dcn_v2_ext as ext
    B, C, H, W = t4.DCN4
    G = 8
    guard = _Guard(dev)
    monkeypatch.setattr(ext, "_ws", guard)
    gen = torch.Generator(device=dev).manual_seed(5)
    pts = [[3.25, 5.5], [61.5, 90.125], [120.25, 33.375]]         # + [0, 0.4): the same 2 x 2 corners per point
    off, pick = colliding_offsets(gen, B, G, H, W, pts)
    per_point = torch.bincount((torch.arange(B * G, device=dev).view(B, G, 1, 1, 1) * len(pts) + pick).flatten())
    x = t4._randn(gen, B, C, H, W)
    w = t4._randn(gen, C, C, 3, 3, scale=1 / 24)
    b = t4._randn(gen, C, scale=0.1)
    m = torch.rand(B, G * 9, H, W, generator=gen, device=dev)
    go = t4._randn(gen, B, C, H, W)
    args = (x, w, b, off, m, go, 3, 3, 1, 1, 1, 1, 1, 1, G)
    t0 = time.time()
    got = ext.dcn_v2_backward(*args)
    again = ext.dcn_v2_backward(*args)
    for n_, a, bb in zip(DCN_NAMES, got, again):
        assert _same_bits(a, bb), n_
    del again
    guard.check("dcn_collide workspaces")
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", False)
    atomics = ext.dcn_v2_backward(*args)
    torch.cuda.synchronize()
    t_gpu = time.time() - t0
    ref, deg = dcn_grads64(x, w, off, m, go, G)
    print(f"[det4x] dcn_collide: {B} x {C} x {H}x{W}, 8 groups, {len(pts)} points; up to {per_point.max().item()} "
          f"values scattered onto one grad_input element; GPU {t_gpu:.1f} s, float64 {time.time() - t0 - t_gpu:.1f} s")
    print("[det4x] dcn_collide, default mode (fp32 atomics) on the same inputs: "
          + ", ".join(f"{n_} {rel(a, ref[n_]):.2e}" for n_, a in zip(DCN_NAMES, atomics)))
    for n_, a in zip(DCN_NAMES, got):
        t4._check(f"dcn_collide.{n_}", f"dcn.{n_}", a, ref[n_], deg[n_],
                  "features without lo plane" if n_ == "grad_weight" else "A_lo B_hi dropped")
    del ref, deg, got, atomics
    t4._free()


# ------------------------------------------------------------------------------------------------------------------
# 5. the deterministic iteration at cfg3 and cfg4
# ------------------------------------------------------------------------------------------------------------------
def _host(state):
    return {k: [t.cpu() for t in v] if isinstance(v, list) else {n: t.cpu() for n, t in v.items()} if isinstance(v, dict)
            else v.cpu() for k, v in state.items()}


def _det_iteration(name, dev, graphed):
    """One deterministic iteration on bench.py's weights and inputs for workload `name`, from the initial state: a
    GraphedTrainStep captured (its warm-up rolled back) and replayed once, or one eager train_step.  -> host copy of
    _state() (loss, logging scalars, 68 gradients, parameters, Adam moments, step)."""
    from esr_b200 import train
    from esr_b200.model import DeepRecurrNet
    sd, frames, gt = t4.bench_inputs(name)
    net = DeepRecurrNet(inch=2, basech=8, num_frame=3)
    net.load_state_dict(sd)
    net = net.to(dev)
    opt = train.Adam(net.parameters(), lr=1e-3, weight_decay=1e-4, amsgrad=True)
    fd, gd = frames.to(dev), gt.to(dev)
    t4._free()
    torch.cuda.reset_peak_memory_stats(dev)
    t0 = time.time()
    step = None
    if graphed:
        step = train.GraphedTrainStep(net, opt, tuple(frames.shape), dev)
        assert step.deterministic and int(opt.step_dev.item()) == 0
        loss = step(fd, gd)
    else:
        loss = train.train_step(net, opt, fd, gd)
    torch.cuda.synchronize()
    assert int(opt.step_dev.item()) == 1
    out = _host(_state(net, opt, [loss]))
    print(f"[det4x] {name} deterministic {'GraphedTrainStep (capture + one replay)' if graphed else 'eager train_step'}: "
          f"{time.time() - t0:.1f} s, peak GPU memory {torch.cuda.max_memory_allocated(dev) / 2**30:.2f} GiB")
    del step, loss, opt, net, fd, gd
    t4._free()
    return out


def _as_compared(st):
    return st["losses"][0].item(), st["log"][0].item(), st["grads"]


@pytest.fixture(scope="module")
def cfg4_ref(dev):
    return t4._reference("cfg4", dev)


@pytestgpu
def test_deterministic_iteration_cfg4_vs_fp64_and_bitwise(dev, cudnn_det, cfg4_ref):
    """A deterministic GraphedTrainStep replay at cfg4 against the float64 reference (the bars of the default replay); a
    second capture from the same state and an eager deterministic train_step give the replay's bits: loss, logging
    scalars, all 68 gradients, parameters and the three Adam moments."""
    first = _det_iteration("cfg4", dev, graphed=True)
    t4._compare("cfg4 deterministic GraphedTrainStep", *_as_compared(first), cfg4_ref)
    _assert_same_state(first, _det_iteration("cfg4", dev, graphed=True))
    _assert_same_state(first, _det_iteration("cfg4", dev, graphed=False))


@pytestgpu
def test_deterministic_iteration_cfg3_eager_equals_replay(dev, cudnn_det):
    _assert_same_state(_det_iteration("cfg3", dev, graphed=False), _det_iteration("cfg3", dev, graphed=True))
