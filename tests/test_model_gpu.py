"""GPU parity of DeepRecurrNet.forward: CUDA plan (through the C ABI) vs the fp32 oracle and the fixtures produced
by the reference's own models/model.py.

Tolerance (BASELINE.json north_star: "within 1e-3 rel on fp32 count tensors"): max |got - want| <= 1e-3 * max |want|.
"""
import os

import numpy as np
import pytest
import torch

from oracle import model_ref

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REL = 1e-3


def _rel(got, want):
    return ((got - want).abs().max() / want.abs().max().clamp_min(1e-12)).item()


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda:0")


def _net(sd, dev):
    from esr_b200.model import DeepRecurrNet
    net = DeepRecurrNet(inch=2, basech=8, num_frame=3)
    net.load_state_dict(sd)
    return net.to(dev).eval()


@pytest.mark.parametrize("name", ["a", "b", "c", "d"])
def test_reference_fixtures(dev, name):
    from tests.test_oracle_model import golden_case
    g = np.load(os.path.join(ROOT, "tests", "golden", "model_golden.npz"))
    sd, frames, nwin = golden_case(g, name)
    net = _net(sd, dev)
    want = torch.from_numpy(g[f"{name}_out"])
    with torch.no_grad():
        net.reset_states()
        for w in range(nwin):
            got = net(frames[:, w:w + 3].contiguous().to(dev)).cpu()
            assert got.shape == want[w].shape
            assert _rel(got, want[w]) < REL, (name, w, _rel(got, want[w]))
        B, _, _, H, W = frames[:, :3].shape
        st = net.states(B, 3, H, W)[0].cpu()
        assert _rel(st[:, :4], torch.from_numpy(g[f"{name}_state_fwd"])) < REL
        # reset_states reproduces the first window exactly (run-to-run determinism of the plan)
        net.reset_states()
        again = net(frames[:, 0:3].contiguous().to(dev)).cpu()
        first = net  # noqa
    net.reset_states()
    with torch.no_grad():
        again2 = net(frames[:, 0:3].contiguous().to(dev)).cpu()
    assert torch.equal(again, again2)


@pytest.mark.parametrize("B,H,W,lam", [(1, 64, 64, 0.1), (2, 128, 128, 0.1), (1, 90, 160, 0.3), (3, 40, 72, 1.0)])
def test_vs_oracle_sequences(dev, B, H, W, lam):
    """4 windows with state carry, incl. the real NFS-syn 2x size 90x160 (pads to 96x160, SURVEY 8c)."""
    torch.set_num_threads(min(16, os.cpu_count() or 1))
    sd = model_ref.seeded_state_dict(5)
    g = torch.Generator().manual_seed(B * 1000 + H)
    frames = torch.poisson(torch.full((B, 6, 2, H, W), lam), generator=g)
    net, ora = _net(sd, dev), model_ref.OracleNet(sd)
    with torch.no_grad():
        for w in range(4):
            x = frames[:, w:w + 3].contiguous()
            want = ora(x)
            got = net(x.to(dev)).cpu()
            assert _rel(got, want) < REL, (w, _rel(got, want))
        for a, b in zip(net.states(B, 3, H, W), ora.states):
            assert _rel(a.cpu(), b) < REL


def test_frame_bank_windows_equal_explicit_windows(dev):
    sd = model_ref.seeded_state_dict(6)
    g = torch.Generator().manual_seed(77)
    B, L, H, W = 2, 5, 32, 48
    frames = torch.poisson(torch.full((B, L, 2, H, W), 0.2), generator=g).to(dev)
    n1, n2 = _net(sd, dev), _net(sd, dev)
    bank = frames.view(B * L, 2, H, W)
    with torch.no_grad():
        for w in range(L - 2):
            idx = torch.tensor([b * L + w + n for b in range(B) for n in range(3)], dtype=torch.int32, device=dev)
            assert torch.equal(n1(frames[:, w:w + 3].contiguous()), n2(bank, frame_index=idx))


@pytest.mark.parametrize("B,L,H,W", [(2, 5, 32, 48), (1, 8, 64, 64), (3, 4, 36, 44)])
def test_sequence_plan_equals_window_loop(dev, B, L, H, W):
    """forward_sequence (per-frame / state-independent layers batched over all windows) must reproduce the reference's
    loop of single-window forwards with carried state -- bit for bit, including the state left behind."""
    sd = model_ref.seeded_state_dict(8)
    g = torch.Generator().manual_seed(B * 31 + L)
    frames = torch.poisson(torch.full((B, L, 2, H, W), 0.3), generator=g).to(dev)
    n1, n2 = _net(sd, dev), _net(sd, dev)
    with torch.no_grad():
        for rep in range(2):                          # second pass starts from the carried state
            loop = torch.cat([n1(frames[:, w:w + 3].contiguous()) for w in range(L - 2)], 0)
            seq = n2.forward_sequence(frames)
            assert seq.shape == loop.shape
            assert torch.equal(seq, loop), (rep, (seq - loop).abs().max().item())
        for a, b in zip(n1.states(B, 3, H, W), n2.states(B, L, H, W)):
            assert torch.equal(a, b)


def _fused_vs_columns_vs_oracle(dev, sd, frames, monkeypatch):
    """forward_sequence with the fused DCN kernel == the columns path bit for bit, and within the bar of the oracle on the
    first and last sequence of the batch (the sequences of a batch are independent)."""
    import bench
    B, L = frames.shape[:2]
    n1 = _net(sd, dev)
    with torch.no_grad():
        fused = n1.forward_sequence(frames.to(dev))
        monkeypatch.setenv("ESR_DCN_COLUMNS", "1")
        n2 = _net(sd, dev)
        cols = n2.forward_sequence(frames.to(dev))
    assert torch.equal(fused, cols), (fused - cols).abs().max().item()
    torch.set_num_threads(bench.usable_cores())
    idx = sorted({0, B - 1})
    ora = model_ref.OracleNet(sd)
    got = fused.view(L - 2, B, *fused.shape[1:])[:, idx].cpu()
    for w in range(L - 2):
        want = ora(frames[idx, w:w + 3].contiguous())
        assert _rel(got[w], want) < REL, (w, _rel(got[w], want))


@pytest.mark.parametrize("B,L,H,W", [(1, 3, 16, 16), (2, 4, 36, 44), (1, 3, 72, 130), (8, 8, 256, 256), (1, 5, 16, 16), (2, 5, 36, 44),
                                     (1, 4, 72, 130)])
def test_fused_dcn_equals_columns_path(dev, B, L, H, W, monkeypatch):
    """The DCN kernel that samples straight into the swizzled wgmma operand tiles must give the same bits as the
    two-kernel path (columns tensor in HBM + 1x1 GEMM): same sampling arithmetic, same MMA order.  (8, 8, 256, 256) is
    the benchmark's cfg2 input: 96 DCN images of 32x32, several tiles per CTA."""
    sd = model_ref.seeded_state_dict(9)
    g = torch.Generator().manual_seed(L * 7 + H)
    frames = torch.poisson(torch.full((B, L, 2, H, W), 0.4), generator=g)
    _fused_vs_columns_vs_oracle(dev, sd, frames, monkeypatch)


def test_fused_dcn_lattice_offsets_on_the_borders(dev, monkeypatch):
    """conv_offset_mask with zero weights and a bias of lattice offsets (multiples of 1/8, exact in fp32): every pixel of a
    (group, tap) samples at the same offset, so integer offsets put samples exactly on -1, 0, H-1 and H (W-1, W) at the
    image edges, and the half / eighth offsets land just inside and outside them."""
    sd = model_ref.seeded_state_dict(10)
    g = torch.Generator().manual_seed(10)
    lattice = torch.tensor([-3.0, -2.0, -1.5, -1.0, -0.875, -0.5, -0.125, 0.0, 0.125, 0.5, 1.0, 1.125, 1.5, 2.0, 3.0])
    w = sd["spacetime_fuse.dcn.conv_offset_mask.weight"]
    b = sd["spacetime_fuse.dcn.conv_offset_mask.bias"].clone()
    b[:144] = lattice[torch.randint(0, len(lattice), (144,), generator=g)]
    sd["spacetime_fuse.dcn.conv_offset_mask.weight"] = torch.zeros_like(w)
    sd["spacetime_fuse.dcn.conv_offset_mask.bias"] = b
    frames = torch.poisson(torch.full((2, 4, 2, 64, 96), 0.4), generator=g)
    _fused_vs_columns_vs_oracle(dev, sd, frames, monkeypatch)


@pytest.mark.parametrize("scale", [1.0, 60.0])
def test_dcn_window_sampler_equals_gather_and_columns(dev, monkeypatch, scale):
    """The fused L2-gather sampler (default) vs the columns path: same bits, also when the learned offsets span many pixels
    (scale 60) and at ragged sizes."""
    sd = model_ref.seeded_state_dict(12)
    sd["spacetime_fuse.dcn.conv_offset_mask.weight"] = sd["spacetime_fuse.dcn.conv_offset_mask.weight"] * scale
    sd["spacetime_fuse.dcn.conv_offset_mask.bias"] = sd["spacetime_fuse.dcn.conv_offset_mask.bias"] + (0.0 if scale == 1.0 else 2.5)
    g = torch.Generator().manual_seed(3)
    frames = torch.poisson(torch.full((2, 4, 2, 72, 104), 0.4), generator=g).to(dev)
    outs = []
    for env in (None, "ESR_DCN_COLUMNS"):
        if env:
            monkeypatch.setenv(env, "1")
        with torch.no_grad():
            outs.append(_net(sd, dev).forward_sequence(frames))
        if env:
            monkeypatch.delenv(env)
    assert torch.equal(outs[0], outs[1])
    ora = model_ref.OracleNet(sd)
    want = torch.cat([ora(frames[:, w:w + 3].cpu()) for w in range(2)], 0)
    assert _rel(outs[0].cpu(), want) <= REL


@pytest.mark.parametrize("B,L,H,W", [(1, 3, 8, 8), (1, 4, 16, 24), (2, 3, 20, 300), (1, 5, 130, 70), (5, 3, 24, 24)])
def test_edge_shapes_vs_oracle(dev, B, L, H, W):
    """Tiny feature maps (1x1 at 8x8 input), very flat / odd sizes that need the CropSize pad, odd batch sizes: the TMA
    boxes then reach far outside the tensors and most tile rows are masked."""
    torch.set_num_threads(min(16, os.cpu_count() or 1))
    sd = model_ref.seeded_state_dict(9)
    g = torch.Generator().manual_seed(H * 1000 + W)
    frames = torch.poisson(torch.full((B, L, 2, H, W), 0.5), generator=g)
    net, ora = _net(sd, dev), model_ref.OracleNet(sd)
    with torch.no_grad():
        got = net.forward_sequence(frames.to(dev)).cpu()
        want = torch.cat([ora(frames[:, w:w + 3].contiguous()) for w in range(L - 2)], 0)
    assert got.shape == want.shape
    assert _rel(got, want) < REL, _rel(got, want)


def test_full_size_properties_cfg2(dev):
    """BASELINE.json configs[1] at full size (B=8, L=8, HR 256x256), where the CPU oracle would take minutes:
    size-independent properties instead -- (1) the sequence plan equals the reference's loop of single-window forwards
    bit for bit, (2) determinism across runs, (3) the batch is independent (a sample alone gives the same output),
    (4) outputs are non-negative (final ReLU) and finite."""
    sd = model_ref.seeded_state_dict(11)
    g = torch.Generator().manual_seed(4242)
    B, L, H, W = 8, 8, 256, 256
    frames = torch.poisson(torch.full((B, L, 2, H, W), 0.1), generator=g).to(dev)
    n1, n2, n3 = _net(sd, dev), _net(sd, dev), _net(sd, dev)
    with torch.no_grad():
        seq = n1.forward_sequence(frames)
        n1.reset_states()
        seq2 = n1.forward_sequence(frames)
        loop = torch.cat([n2(frames[:, w:w + 3].contiguous()) for w in range(L - 2)], 0)
        solo = n3.forward_sequence(frames[3:4].contiguous())
    assert torch.equal(seq, loop)
    assert torch.equal(seq, seq2)
    assert torch.equal(solo, seq.view(L - 2, B, 2, H, W)[:, 3])
    assert bool(torch.isfinite(seq).all()) and float(seq.min()) >= 0.0


# ---------------------------------------------------------------------------------------------------------------------
# Full-size parity on every configuration bench.py measures (VERDICT r1, "What's weak" 1): the fp32 oracle is run on the
# host cores over ALL windows of the sequence, with the ConvGRU state carried exactly as the reference's loop does
# (models/model.py:91-124, train_ours_cnt_seq.py:217-231), and every window output and both carried states must be within
# 1e-3 (max-norm relative, the north_star tolerance).
FULL = {
    # name: (B, L, LR, scale)  -- BASELINE.json configs[1..3], per-GPU batch as bench.py runs them
    "cfg2": (8, 8, (128, 128), 2),
    "cfg3": (4, 8, (128, 128), 4),
    "cfg4": (2, 16, (256, 256), 4),
}


def _bench_frames(B, L, lr, scale, dev, kind):
    """`events`: the bench's own input (bench.synth_events -> LR->HR lift + count scatter on the GPU);
    `poisson`: SURVEY 8d's synthetic count tensors, Poisson(0.1) per HR pixel and polarity."""
    hr = (lr[0] * scale, lr[1] * scale)
    if kind == "poisson":
        g = torch.Generator().manual_seed(B * 100 + L)
        return torch.poisson(torch.full((B, L, 2, hr[0], hr[1]), 0.1), generator=g).to(dev)
    import bench
    from esr_b200 import encodings as enc
    xs, ys, ps, off = bench.synth_events(B, L, lr, 100)
    bank = enc.encode_frames(xs.to(dev), ys.to(dev), ps.to(dev), off.to(dev), lr_size=lr, hr_size=hr,
                             n_max_frame=bench.EVENTS_PER_FRAME)
    return bank.view(B, L, 2, hr[0], hr[1])


def _weights(kind):
    import bench
    if kind == "bench":
        return bench.synth_weights(0)                       # what bench.py measures with
    if kind == "seeded":
        return model_ref.seeded_state_dict(3)
    # the reference's own initialisation (torch Conv2d defaults, orthogonal ConvGRU gates, models/submodules.py:489-494),
    # with a non-zero conv_offset_mask so that the deformable sampling is exercised
    from esr_b200.model import DeepRecurrNet
    torch.manual_seed(0)
    sd = {k: v.clone() for k, v in DeepRecurrNet(inch=2, basech=8, num_frame=3).state_dict().items()}
    g = torch.Generator().manual_seed(1)
    sd["spacetime_fuse.dcn.conv_offset_mask.weight"] = torch.randn(sd["spacetime_fuse.dcn.conv_offset_mask.weight"].shape, generator=g) * 0.01
    sd["spacetime_fuse.dcn.conv_offset_mask.bias"] = torch.randn(216, generator=g) * 0.3
    return sd


@pytest.mark.parametrize("weights", ["bench", "seeded", "refinit"])
@pytest.mark.parametrize("cfg,kind", [("cfg2", "events"), ("cfg2", "poisson"), ("cfg3", "events"), ("cfg4", "events")])
def test_full_size_vs_oracle(dev, cfg, kind, weights):
    import bench
    torch.set_num_threads(bench.usable_cores())
    B, L, lr, scale = FULL[cfg]
    H, W = lr[0] * scale, lr[1] * scale
    sd = _weights(weights)
    frames = _bench_frames(B, L, lr, scale, dev, kind)
    net, ora = _net(sd, dev), model_ref.OracleNet(sd)
    with torch.no_grad():
        got = net.forward_sequence(frames).cpu().view(L - 2, B, 2, H, W)
        st = [s.cpu() for s in net.states(B, L, H, W)]
        host = frames.cpu()
        worst = 0.0
        for w in range(L - 2):
            want = ora(host[:, w:w + 3].contiguous())
            assert float(want.abs().max()) > 0
            r = _rel(got[w], want)
            worst = max(worst, r)
            assert r < REL, (cfg, kind, weights, "window", w, r)
        for i, (a, b) in enumerate(zip(st, ora.states)):
            r = _rel(a, b)
            assert r < REL, (cfg, kind, weights, "state", i, r)
    print(f"[parity] {cfg}/{kind}/{weights}: worst window rel {worst:.2e}, states "
          f"{_rel(st[0], ora.states[0]):.2e} {_rel(st[1], ora.states[1]):.2e}")
