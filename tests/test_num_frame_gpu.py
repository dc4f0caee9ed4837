"""GPU: DeepRecurrNet at num_frame = 5, 7, 9 through every path -- the inference plan (against the reference's fixtures and
the fp32 oracle), its alternative paths bit for bit, dense_fusion.0's N-chunk k_conv_tc against float64, the training
operators and train_step / GraphedTrainStep against autograd through the oracle, the sequence reader and the pipeline.

Tolerances are those of num_frame = 3: 1e-3 max-norm relative for the plan (test_model_gpu.py), 3e-3 for whole-network
gradients (test_train_gpu.py), 4e-5 for k_conv_tc against float64 (test_tc_fp64_gpu.py)."""
import math
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import model_ref

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REL = 1e-3
OUT_FLOOR = 1e-2
SEED = 21             # weights whose outputs peak at 0.18 or more on the random inputs below (none is near all-zero)


def _rel(got, want):
    got, want = got.detach().float().cpu(), want.detach().float().cpu()
    return ((got - want).abs().max() / want.abs().max().clamp_min(1e-12)).item()


@pytest.fixture(scope="module")
def dev():
    torch.set_num_threads(min(16, os.cpu_count() or 1))
    return torch.device("cuda:0")


def _net(sd, N, dev, train=False):
    from esr_b200.model import DeepRecurrNet
    net = DeepRecurrNet(inch=2, basech=8, num_frame=N)
    net.load_state_dict(sd)
    net = net.to(dev)
    return net if train else net.eval()


def _poisson(shape, lam, seed):
    return torch.poisson(torch.full(shape, lam), generator=torch.Generator().manual_seed(seed))


# ------------------------------------------------------------------------------------------------- inference plan
@pytest.mark.parametrize("name", ["n5a", "n5b", "n7", "n9", "n5z"])
def test_reference_fixtures(dev, name):
    from tests.test_num_frame import golden_case
    g = np.load(os.path.join(ROOT, "tests", "golden", "model_nf_golden.npz"))
    sd, frames, nwin, N = golden_case(g, name)
    want = torch.from_numpy(g[f"{name}_out"])
    assert float(want.abs().max()) >= OUT_FLOOR
    net = _net(sd, N, dev)
    B, _, _, H, W = frames.shape
    with torch.no_grad():
        net.reset_states()
        for w in range(nwin):
            got = net(frames[:, w:w + N].contiguous().to(dev)).cpu()
            assert got.shape == want[w].shape
            assert _rel(got, want[w]) < REL, (name, w, _rel(got, want[w]))
        st = net.states(B, N, H, W)[0].cpu()
        assert _rel(st[:, :4], torch.from_numpy(g[f"{name}_state_fwd"])) < REL
    net2 = _net(sd, N, dev)
    with torch.no_grad():                                   # the same windows from one sequence plan
        seq = net2.forward_sequence(frames.to(dev)).cpu().view(nwin, B, 2, H, W)
    for w in range(nwin):
        assert _rel(seq[w], want[w]) < REL, (name, "sequence", w)


@pytest.mark.parametrize("N,B,H,W,lam", [(5, 1, 32, 32, 0.5), (5, 3, 36, 44, 1.0), (7, 2, 20, 28, 0.6), (9, 1, 42, 30, 1.0),
                                         (7, 3, 17, 23, 1.0)])
def test_vs_oracle_sequences(dev, N, B, H, W, lam):
    """Random sequences of N + 1 frames (two windows, state carried), sizes that are and are not multiples of 8."""
    sd = model_ref.seeded_state_dict(SEED, num_frame=N)
    frames = _poisson((B, N + 1, 2, H, W), lam, B * 1000 + H * 10 + N)
    net, ora = _net(sd, N, dev), model_ref.OracleNet(sd)
    with torch.no_grad():
        got = net.forward_sequence(frames.to(dev)).cpu().view(2, B, 2, H, W)
        for w in range(2):
            want = ora(frames[:, w:w + N].contiguous())
            assert float(want.abs().max()) >= OUT_FLOOR
            assert _rel(got[w], want) < REL, (w, _rel(got[w], want))
        for a, b in zip(net.states(B, N + 1, H, W), ora.states):
            assert _rel(a, b) < REL


@pytest.mark.parametrize("N,B,L,H,W", [(5, 2, 8, 32, 48), (7, 1, 9, 36, 44), (5, 3, 5, 24, 24)])
def test_sequence_plan_equals_window_loop_and_frame_bank(dev, N, B, L, H, W):
    """forward_sequence == the loop of single-window forwards == windows addressed in a frame bank, bit for bit, including
    the state left behind, over two passes (the second starts from the carried state)."""
    sd = model_ref.seeded_state_dict(SEED, num_frame=N)
    frames = _poisson((B, L, 2, H, W), 0.5, B * 31 + L).to(dev)
    bank = frames.view(B * L, 2, H, W)
    n1, n2, n3 = _net(sd, N, dev), _net(sd, N, dev), _net(sd, N, dev)
    with torch.no_grad():
        for rep in range(2):
            loop = torch.cat([n1(frames[:, w:w + N].contiguous()) for w in range(L - N + 1)], 0)
            idx = [torch.tensor([b * L + w + n for b in range(B) for n in range(N)], dtype=torch.int32, device=dev)
                   for w in range(L - N + 1)]
            banked = torch.cat([n3(bank, frame_index=i) for i in idx], 0)
            seq = n2.forward_sequence(frames)
            assert seq.shape == loop.shape == ((L - N + 1) * B, 2, H, W)
            assert float(loop.abs().max()) >= OUT_FLOOR
            assert torch.equal(seq, loop), (rep, (seq - loop).abs().max().item())
            assert torch.equal(banked, loop), rep
    for a, b in zip(n1.states(B, N, H, W), n2.states(B, L, H, W)):
        assert torch.equal(a, b)


@pytest.mark.parametrize("env", ["ESR_DCN_COLUMNS"])
@pytest.mark.parametrize("N,B,L,H,W", [(5, 2, 7, 36, 44), (7, 1, 9, 72, 40), (3, 2, 5, 20, 28), (9, 1, 10, 24, 16)])
def test_alternative_paths_are_bit_identical(dev, monkeypatch, env, N, B, L, H, W):
    """The two-kernel DCN path gives the default path's bits."""
    sd = model_ref.seeded_state_dict(SEED, num_frame=N)
    frames = _poisson((B, L, 2, H, W), 0.5, L * 11 + W).to(dev)
    with torch.no_grad():
        n1 = _net(sd, N, dev)
        ref = n1.forward_sequence(frames)
        monkeypatch.setenv(env, "1")
        n2 = _net(sd, N, dev)
        alt = n2.forward_sequence(frames)
    assert float(ref.abs().max()) >= OUT_FLOOR
    assert torch.equal(alt, ref), (alt - ref).abs().max().item()
    for a, b in zip(n1.states(B, L, H, W), n2.states(B, L, H, W)):
        assert torch.equal(a, b)


def test_full_size_n5_vs_oracle_and_workspace(dev):
    """num_frame = 5 at the benchmark's cfg2 input with the reference's SEQL (B = 8, L = 9, 256x256 HR): the first and the
    last sequence against the oracle over all five windows; the plan's workspace is esr_net_workspace_bytes and is all the
    device memory the plan takes besides the parameter blob and the output."""
    import bench
    from esr_b200 import _lib
    torch.set_num_threads(bench.usable_cores())
    N, B, L, H, W = 5, 8, 9, 256, 256
    sd = model_ref.seeded_state_dict(SEED, num_frame=N)
    frames = _poisson((B, L, 2, H, W), 0.1, 4243)
    net = _net(sd, N, dev)
    fd = frames.to(dev)
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated(dev)
    with torch.no_grad():
        got = net.forward_sequence(fd)
    torch.cuda.synchronize()
    used = torch.cuda.memory_allocated(dev) - before
    ws = _lib.lib().esr_net_workspace_bytes(B, N, L, H, W)
    plan = net._plans[(B, L, H, W)]
    assert plan.ws.numel() == ws > 0
    blob = net._blob.numel()
    assert blob == _lib.lib().esr_net_param_bytes_n(N)
    assert ws + blob + got.numel() * 4 <= used <= ws + blob + got.numel() * 4 + 3 * (2 << 20), (used, ws, blob)
    got = got.cpu().view(L - N + 1, B, 2, H, W)
    ora = model_ref.OracleNet(sd)
    for s in (0, B - 1):
        ora.reset_states()
        for w in range(L - N + 1):
            want = ora(frames[s:s + 1, w:w + N].contiguous())
            assert float(want.abs().max()) > 0
            assert _rel(got[w, s:s + 1], want) < REL, (s, w, _rel(got[w, s:s + 1], want))


# ------------------------------------------------------------------------------------------------- k_conv_tc vs float64
@pytest.mark.parametrize("chunks", [5, 7, 9])
def test_dense_fusion_chunked_conv_vs_fp64(dev, chunks):
    """dense_fusion.0's launch shape: one 64-channel source standing for chunks - 1 chunks (VB images apart, read through a
    permuting image map) plus a second source read through a repeating / permuting map, as ONE k_conv_tc launch, against
    float64 of the materialised concatenation.  >= 3 tiles per CTA and a tile count that is not a multiple of the grid."""
    from esr_b200 import layers as Lyr
    from tests.test_tc_fp64_gpu import (_check_images, _epilogue, _rand, assert_multi_tile, check, conv_geometry, emulations,
                                        product_terms)
    VB, H, W, cout = 100, 32, 32, 64
    g = torch.Generator().manual_seed(chunks * 977)
    geo = conv_geometry(VB, H, W, 64 * chunks, 9, cout)
    assert_multi_tile(geo)
    n_mid = 3 * VB
    fused = _rand(g, (chunks - 1) * VB, 64, H, W)                # k-major: neighbour k of window vb is image k * VB + vb
    mid = _rand(g, n_mid, 64, H, W)
    perm = torch.randperm(VB, generator=g)                       # permuting map of the chunked source
    mid_map = torch.randint(0, n_mid, (VB,), generator=g)
    w = _rand(g, cout, 64 * chunks, 3, 3, scale=1.0 / math.sqrt(64 * chunks * 9))
    b = _rand(g, cout, scale=0.1)
    s_f, s_m = Lyr.Split.from_nchw(fused.to(dev)), Lyr.Split.from_nchw(mid.to(dev))
    out = Lyr.Split(VB, cout, H, W, dev)
    Lyr.conv_tc([s_f, s_m], Lyr.pack_weight(w.to(dev)), Lyr.pad_bias(b.to(dev), cout), cout, act="relu",
                src_img=[perm, mid_map], n_img=VB, out=out, src_chunks=[chunks - 1, 0], chunk_img_step=[VB, 0])
    got = out.to_nchw().cpu()
    sel = torch.tensor(_check_images(VB, 12))
    xcat = torch.cat([fused[perm[sel] + k * VB] for k in range(chunks - 1)] + [mid[mid_map[sel]]], 1)
    conv = lambda a, bb: F.conv2d(a, bb, padding=1)              # noqa: E731
    ref = _epilogue(conv(xcat.double(), w.double()), b, "relu", 0, None, 0)
    deg = _epilogue(emulations(product_terms(conv, xcat, w))["drop_cross"], b, "relu", 0, None, 0)
    print(f"[tc64] dense_fusion chunks {chunks}: tiles {geo['n_tiles']}, grid {geo['grid']}, nkb {geo['nkb']}")
    check(f"dense_fusion_{chunks}chunks", "conv_split", got[sel], ref, deg)


def test_chunked_source_is_validated(dev):
    from esr_b200 import _lib
    from esr_b200 import layers as Lyr
    s = Lyr.Split(4, 128, 8, 8, dev)
    wp = torch.zeros(Lyr._lib.lib().esr_conv_weight_bytes(64, 256, 3), dtype=torch.uint8, device=dev)
    with pytest.raises(_lib.ESRError):                          # a stepped source must have 64 channels
        Lyr.conv_tc([s], wp, torch.zeros(64, device=dev), 64, n_img=2, out=Lyr.Split(2, 64, 8, 8, dev), src_chunks=[2],
                    chunk_img_step=[2])


# ------------------------------------------------------------------------------------------------- training
ACTS = {None: lambda v: v, "relu": torch.relu}


@pytest.mark.parametrize("B,Cin,H,W", [(2, 320, 20, 28), (1, 448, 17, 23), (1, 576, 16, 16)])
def test_dense_fusion_training_operator_vs_torch(dev, B, Cin, H, W):
    """esr_conv2d_forward / backward at dense_fusion.0's widths (num_frame 5, 7, 9)."""
    from esr_b200 import train
    g = torch.Generator().manual_seed(Cin + H)
    x = torch.randn(B, Cin, H, W, generator=g, requires_grad=True)
    w = (torch.randn(64, Cin, 3, 3, generator=g) / (Cin * 9) ** 0.5).requires_grad_()
    b = (0.1 * torch.randn(64, generator=g)).requires_grad_()
    want = torch.relu(F.conv2d(x, w, b, padding=1))
    dy = torch.randn(want.shape, generator=g)
    want.backward(dy)
    xg, wg, bg = (t.detach().to(dev).requires_grad_() for t in (x, w, b))
    got = train.conv2d(xg, wg, bg, 1, "relu")
    assert _rel(got, want) <= REL
    got.backward(dy.to(dev))
    assert _rel(xg.grad, x.grad) <= REL, "dx"
    assert _rel(wg.grad, w.grad) <= REL, "dw"
    assert _rel(bg.grad, b.grad) <= REL, "db"


def _oracle_sequence_loss(ref, frames, gt, N, mid, dcn_fn=model_ref.dcn_v2_forward):
    states, loss = None, 0
    for w in range(frames.shape[1] - N + 1):
        pred, states = model_ref.forward(ref, frames[:, w:w + N], states, dcn_fn=dcn_fn)
        loss = loss + F.mse_loss(pred, gt[:, w + mid])
    return loss


@pytest.mark.parametrize("N,B,L,H,W", [(5, 2, 7, 32, 32), (7, 1, 8, 32, 32)])
def test_sequence_gradients_vs_oracle_autograd(dev, N, B, L, H, W):
    """Sum over windows of MSE(pred, gt[window middle]) with the state carried: the loss and all 68 gradients of the batched
    training graph against float64 autograd through the oracle (DCN sample positions formed in fp32, as in
    test_train_gpu.py's cfg2 case)."""
    from esr_b200 import train
    from tests.test_train_gpu import _dcn_fp32_positions
    sd = model_ref.seeded_state_dict(SEED, num_frame=N)
    frames, gt = _poisson((B, L, 2, H, W), 0.3, 61 + N), _poisson((B, L, 2, H, W), 0.3, 62 + N)   # num_frame 3's rate
    mid = (N - 1) // 2
    ref = {k: v.double().requires_grad_() for k, v in sd.items()}
    loss_ref = _oracle_sequence_loss(ref, frames.double(), gt.double(), N, mid, dcn_fn=_dcn_fp32_positions)
    loss_ref.backward()
    net = _net(sd, N, dev, train=True)
    net.reset_states()
    fd, gd = frames.to(dev), gt.to(dev)
    pred = net(fd)                                               # all windows, window-major
    Wn = L - N + 1
    assert pred.shape == (Wn * B, 2, H, W)
    loss = sum(train.mse_loss(pred[w * B:(w + 1) * B], gd[:, w + mid]) for w in range(Wn))
    loss.backward()
    assert abs(loss.item() - loss_ref.item()) <= REL * abs(loss_ref.item())
    worst = {n: _rel(p.grad, ref[n].grad) for n, p in net.named_parameters()}
    assert len(worst) == 68
    top = sorted(worst.items(), key=lambda kv: -kv[1])[:3]
    print(f"[train N={N}] loss {loss.item():.6e} vs {loss_ref.item():.6e}; worst " + ", ".join(f"{k} {v:.2e}" for k, v in top))
    # pred_map.1's bias is one number: the sum of the gate gradient over every pixel of the N + 1 frame pairs of every window,
    # which nearly cancels, so its relative error is the largest (measured on an H100: 3.2e-3 at N = 5, 3.7e-3 at N = 7; every
    # other gradient <= 1.9e-3).  It gets 5e-3; the other 67 the whole-network bar of 3e-3.
    assert worst.pop("time_propagate.pred_map.1.conv2d.bias") <= 5 * REL
    bad = {k: v for k, v in worst.items() if v > 3 * REL}
    assert not bad, bad


def test_train_step_tracks_oracle_losses_n5(dev):
    """Four iterations of train_step at num_frame = 5 follow the oracle trained with torch.optim.Adam (amsgrad)."""
    from esr_b200 import train
    N = 5
    sd = model_ref.seeded_state_dict(SEED, num_frame=N)
    frames, gt = _poisson((2, 7, 2, 32, 32), 0.4, 72), _poisson((2, 7, 2, 32, 32), 0.4, 73)
    ref = {k: v.clone().requires_grad_() for k, v in sd.items()}
    opt_ref = torch.optim.Adam(list(ref.values()), lr=1e-3, weight_decay=1e-4, amsgrad=True)
    net = _net(sd, N, dev, train=True)
    opt = train.Adam(net.parameters(), lr=1e-3, weight_decay=1e-4, amsgrad=True)
    fd, gd = frames.to(dev), gt.to(dev)
    losses, losses_ref = [], []
    for _ in range(4):
        opt_ref.zero_grad()
        lr_ = _oracle_sequence_loss(ref, frames, gt, N, 2)
        lr_.backward()
        opt_ref.step()
        losses_ref.append(lr_.item())
        losses.append(train.train_step(net, opt, fd, gd).item())
    for a, b in zip(losses, losses_ref):
        assert abs(a - b) <= 1e-3 * abs(b), (losses, losses_ref)


def test_train_step_takes_num_frame_from_the_model(dev):
    """Without num_frame, train_step uses the model's windows and middle frame (2 at num_frame = 5); a value that disagrees
    with the model raises, the agreeing one is accepted."""
    from esr_b200 import _lib, train
    N, B, L, H, W = 5, 2, 7, 24, 32
    sd = model_ref.seeded_state_dict(SEED, num_frame=N)
    frames, gt = _poisson((B, L, 2, H, W), 0.4, 82).to(dev), _poisson((B, L, 2, H, W), 0.4, 83).to(dev)
    a, b = _net(sd, N, dev, train=True), _net(sd, N, dev, train=True)
    oa = train.Adam(a.parameters(), lr=1e-3)
    la = train.train_step(a, oa, frames, gt).item()
    b.reset_states()
    pred = b(frames).detach()
    Wn = L - N + 1
    sums = {m: sum(train.mse_loss(pred[w * B:(w + 1) * B], gt[:, w + m]).item() for w in range(Wn)) for m in (1, 2)}
    assert abs(la - sums[2]) <= 1e-5 * abs(sums[2]), (la, sums)
    assert abs(sums[1] - sums[2]) > 1e-3 * abs(sums[2])          # the middle frame matters at this data
    with pytest.raises(_lib.ESRError):
        train.train_step(a, oa, frames, gt, num_frame=3)
    with pytest.raises(_lib.ESRError):
        train.GraphedTrainStep(b, train.Adam(b.parameters(), lr=1e-3), (B, L, 2, H, W), dev, num_frame=3)
    train.train_step(a, oa, frames, gt, num_frame=5)


def test_graphed_train_step_equals_eager_n5(dev):
    from esr_b200 import train
    N = 5
    sd = model_ref.seeded_state_dict(SEED, num_frame=N)
    a, b = _net(sd, N, dev, train=True), _net(sd, N, dev, train=True)
    oa = train.Adam(a.parameters(), lr=1e-3, weight_decay=1e-4, amsgrad=True)
    ob = train.Adam(b.parameters(), lr=1e-3, weight_decay=1e-4, amsgrad=True)
    step_b = train.GraphedTrainStep(b, ob, (2, 6, 2, 32, 32), dev)
    assert int(ob.step_dev.item()) == 0
    for it in range(3):
        frames, gt = _poisson((2, 6, 2, 32, 32), 0.4, 100 + it), _poisson((2, 6, 2, 32, 32), 0.4, 200 + it)
        la = train.train_step(a, oa, frames.to(dev), gt.to(dev)).item()
        lb = step_b(frames.to(dev), gt.to(dev)).item()
        assert abs(la - lb) <= 1e-4 * abs(la), (it, la, lb)
    assert int(ob.step_dev.item()) == 3
    for (n, pa), (_, pb) in zip(a.named_parameters(), b.named_parameters()):
        assert torch.allclose(pa.detach(), pb.detach(), rtol=0, atol=3e-3), n


# ------------------------------------------------------------------------------------------------- loader and pipeline
def test_sequence_reader_seqn5_feeds_the_model(dev, tmp_path):
    """SequenceReader with `seqn: 5` yields L - 4 windows; running them through a num_frame = 5 model one after another (state
    carried) equals forward_sequence on the batch's bank."""
    from esr_b200 import eventstore as es
    from tests.test_augment_gpu import _store
    store, cfg = _store("pause_noaug", tmp_path)
    cfg["sequence"]["seqn"] = 5
    cfg["sequence"]["pause"]["enabled"] = False
    cfg["data_augment"]["enabled"] = False
    rd = es.SequenceReader(store, cfg)
    wins = rd.load_batch([0, 2, 1])
    L = rd.L
    assert rd.num_frame == 5 and len(wins) == L - 4 >= 2
    sd = model_ref.seeded_state_dict(SEED, num_frame=5)
    n1, n2 = _net(sd, 5, dev), _net(sd, 5, dev)
    with torch.no_grad():
        loop = torch.cat([n1(w["inp_scaled_cnt"].contiguous()) for w in wins], 0)
        seq = n2.forward_sequence(wins[0]["bank"]["inp_scaled_cnt"])
    assert float(loop.abs().max()) > 0
    assert torch.equal(seq, loop)


def test_pipeline_runs_a_num_frame_5_model(dev):
    from esr_b200.expand import expand
    from esr_b200.pipeline import EventSRPipeline
    from tests.test_pipeline_gpu import _events
    B, L, lr, scale, n = 2, 7, (32, 40), 2, 300
    net = _net(model_ref.seeded_state_dict(SEED, num_frame=5), 5, dev)
    pipe = EventSRPipeline(net, B, L, lr, scale, dev)
    assert len(pipe.window_index) == L - 4
    batch = _events(B, L, lr, n, 3)
    sr, ev = pipe.run_device(*[t.to(dev) for t in batch], n)
    assert sr.shape == ((L - 4) * B, 2, lr[0] * scale, lr[1] * scale)
    with torch.no_grad():
        net.reset_states()
        want = net.forward_sequence(pipe.bank.view(B, L, 2, lr[0] * scale, lr[1] * scale))
    assert torch.equal(sr, want)
    assert torch.equal(ev, expand(want, 0, 0))
    pipe.sequence_plan = False                                   # the reference's loop of frame-bank windows
    with torch.no_grad():
        assert torch.equal(pipe._windows(), want)
    host = pipe.run_host(*batch, n)
    assert torch.equal(host, ev.cpu())
    with pytest.raises(ValueError):
        EventSRPipeline(net, B, 4, lr, scale, dev)
