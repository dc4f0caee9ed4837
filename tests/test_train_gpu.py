"""GPU parity of the training-step operators (SURVEY.md 8a row 17): esr_conv2d_forward/backward, esr_mse_loss,
esr_adam_step and the differentiable window forward, against torch CPU fp32 autograd of the same maths (for the whole
network: autograd through the oracle restatement of models/model.py).

Tolerance: max |got - want| <= 1e-3 * max |want| per tensor (BASELINE.json north_star's fp32 bar), a little wider for
whole-network gradients where it says so.
"""
import pytest
import torch
import torch.nn.functional as F

from oracle import model_ref

pytestmark = pytest.mark.gpu
REL = 1e-3
torch.set_num_threads(min(16, torch.get_num_threads()))


def _rel(got, want):
    return ((got.cpu() - want).abs().max() / want.abs().max().clamp_min(1e-20)).item()


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda:0")


ACTS = {None: lambda v: v, "relu": torch.relu, "sigmoid": torch.sigmoid, "tanh": torch.tanh}

CONV_CASES = [
    # B, Cin, Cout, k, stride, act, H, W
    (2, 64, 64, 3, 1, "relu", 20, 28),          # tensor-core forward, dx and dw
    (1, 128, 64, 3, 1, "sigmoid", 17, 23),      # ConvGRU gates (ragged tile edges)
    (2, 128, 64, 3, 1, "tanh", 16, 16),
    (1, 192, 192, 3, 1, None, 16, 24),          # local_fusion residual convs
    (1, 192, 64, 3, 1, None, 12, 40),
    (2, 64, 216, 3, 1, None, 16, 16),           # conv_offset_mask: Cout not a multiple of 64 -> CUDA-core dx
    (2, 64, 1, 3, 1, "sigmoid", 20, 20),        # pred_map[1], attens[0]
    (2, 64, 2, 1, 1, "sigmoid", 20, 20),        # STFusion.kernel (1x1)
    (2, 128, 64, 1, 1, "relu", 20, 20),         # global_fusion (1x1)
    (2, 64, 32, 3, 1, "relu", 24, 24),          # recons[0]
    (2, 2, 8, 3, 1, "relu", 40, 56),            # head
    (2, 8, 16, 3, 2, "relu", 40, 56),           # encoder, stride 2
    (2, 16, 32, 3, 2, "relu", 20, 28),
    (1, 32, 64, 3, 2, "relu", 18, 26),
    (2, 32, 16, 3, 1, "relu", 33, 47),          # recons[1] (odd sizes)
    (2, 16, 8, 3, 1, "relu", 40, 40),
    (3, 8, 2, 3, 1, "relu", 31, 17),            # tail
    (1, 32, 1, 3, 1, "sigmoid", 24, 24),        # attens[1]
    (2, 16, 8, 3, 1, "relu", 40, 150),          # wider than one 64-pixel register tile (halo columns between tiles)
    (1, 32, 16, 3, 1, None, 70, 130),
    (1, 8, 2, 3, 1, "relu", 20, 64),            # exactly one tile wide
    (1, 64, 32, 3, 1, "relu", 20, 70),          # Cout 32: g padded to 64 channels for the tensor-core dx / dw
    (2, 16, 8, 3, 1, "relu", 40, 50),           # more narrow layers whose dw runs on k_conv_wgrad_r
    (1, 32, 16, 3, 1, "relu", 33, 47),
    (1, 8, 16, 3, 2, "relu", 33, 45),
    (1, 2, 8, 3, 1, "relu", 20, 36),
]


@pytest.mark.parametrize("B,Cin,Cout,k,stride,act,H,W", CONV_CASES)
def test_conv2d_forward_backward_vs_torch(dev, B, Cin, Cout, k, stride, act, H, W):
    from esr_b200 import train
    g = torch.Generator().manual_seed(Cin * 1000 + Cout * 7 + H)
    x = torch.randn(B, Cin, H, W, generator=g, requires_grad=True)
    w = (torch.randn(Cout, Cin, k, k, generator=g) / (Cin * k * k) ** 0.5).requires_grad_()
    b = (0.1 * torch.randn(Cout, generator=g)).requires_grad_()
    want = ACTS[act](F.conv2d(x, w, b, stride=stride, padding=k // 2))
    dy = torch.randn(want.shape, generator=g)
    want.backward(dy)
    xg, wg, bg = (t.detach().to(dev).requires_grad_() for t in (x, w, b))
    got = train.conv2d(xg, wg, bg, stride, act)
    assert got.shape == want.shape
    assert _rel(got.detach(), want.detach()) <= REL
    got.backward(dy.to(dev))
    assert _rel(xg.grad, x.grad) <= REL, "dx"
    assert _rel(wg.grad, w.grad) <= REL, "dw"
    assert _rel(bg.grad, b.grad) <= REL, "db"


def test_conv2d_first_layer_needs_no_dx(dev):
    from esr_b200 import train
    x = torch.randn(1, 2, 16, 16, device=dev)
    w = torch.randn(8, 2, 3, 3, device=dev, requires_grad=True)
    b = torch.zeros(8, device=dev, requires_grad=True)
    train.conv2d(x, w, b, 1, "relu").sum().backward()
    assert w.grad is not None and b.grad is not None


@pytest.mark.parametrize("shape", [(2, 3, 8, 8), (1, 5, 7, 13), (3, 2, 1, 9), (2, 16, 33, 20)])
def test_upsample2x_forward_backward_vs_torch(dev, shape):
    from esr_b200 import train
    g = torch.Generator().manual_seed(sum(shape))
    x = torch.randn(shape, generator=g, requires_grad=True)
    want = F.interpolate(x, scale_factor=2, mode="bilinear", align_corners=False)
    dy = torch.randn(want.shape, generator=g)
    want.backward(dy)
    xg = x.detach().to(dev).requires_grad_()
    got = train.upsample2x(xg)
    assert _rel(got.detach(), want.detach()) <= 1e-6
    got.backward(dy.to(dev))
    assert _rel(xg.grad, x.grad) <= 1e-6


def test_mse_loss_and_adam_vs_torch(dev):
    from esr_b200 import train
    g = torch.Generator().manual_seed(5)
    p0, t0 = torch.randn(3, 2, 33, 17, generator=g), torch.randn(3, 2, 33, 17, generator=g)
    pr = p0.clone().requires_grad_()
    want = F.mse_loss(pr, t0)
    want.backward()
    pg = p0.to(dev).requires_grad_()
    got = train.mse_loss(pg, t0.to(dev))
    (3.0 * got).backward()
    assert abs(got.item() - want.item()) <= 1e-6 * abs(want.item()) + 1e-9
    assert _rel(pg.grad, 3.0 * pr.grad) <= 1e-6
    # Adam(lr 1e-3, weight_decay 1e-4, amsgrad) = config/train_ours_enfssyn.yml optimizer
    shapes = [(8, 2, 3, 3), (8,), (64, 128, 3, 3), (5,)]
    ref = [torch.randn(s, generator=g).requires_grad_() for s in shapes]
    mine = [r.detach().clone().to(dev).requires_grad_() for r in ref]
    o_ref = torch.optim.Adam(ref, lr=1e-3, weight_decay=1e-4, amsgrad=True)
    o_mine = train.Adam(mine, lr=1e-3, weight_decay=1e-4, amsgrad=True)
    for step in range(6):
        o_mine.zero_grad()
        for r, m in zip(ref, mine):
            gr = torch.randn(r.shape, generator=g) * (0.1 if step % 2 else 10.0)
            r.grad = gr.clone()
            m.grad.copy_(gr.to(dev))
        o_ref.step()
        o_mine.step()
        for r, m in zip(ref, mine):
            assert torch.allclose(m.detach().cpu(), r.detach(), rtol=2e-6, atol=2e-7), step


def _frames(B, L, H, W, seed, lam=0.3):
    g = torch.Generator().manual_seed(seed)
    return torch.poisson(torch.full((B, L, 2, H, W), lam), generator=g), torch.poisson(torch.full((B, L, 2, H, W), lam), generator=g)


def _net(sd, dev):
    from esr_b200.model import DeepRecurrNet
    net = DeepRecurrNet(inch=2, basech=8, num_frame=3)
    net.load_state_dict(sd)
    return net.to(dev)


def test_training_forward_matches_inference_plan(dev):
    """The differentiable composition and the fused no_grad plan are the same function (incl. the carried state)."""
    sd = model_ref.seeded_state_dict(21)
    frames, _ = _frames(2, 5, 36, 44, 3)
    frames = frames.to(dev)
    a, b = _net(sd, dev), _net(sd, dev)
    for w in range(3):
        with torch.no_grad():
            want = a(frames[:, w:w + 3].contiguous())
        got = b(frames[:, w:w + 3])
        assert got.requires_grad
        assert _rel(got.detach().cpu(), want.cpu()) <= REL, w


@pytest.mark.parametrize("B,L,H,W", [(1, 4, 32, 32), (2, 5, 24, 40), (1, 3, 20, 28)])
def test_sequence_gradients_vs_oracle_autograd(dev, B, L, H, W):
    """Loss = sum over windows of MSE(pred, gt[mid]) with the ConvGRU state carried (train_ours_cnt_seq.py:209-232):
    loss value and all 68 parameter gradients vs autograd through the oracle on the CPU."""
    from esr_b200 import train
    sd = model_ref.seeded_state_dict(31 + L)
    frames, gt = _frames(B, L, H, W, 11 + H)
    ref = {k: v.clone().requires_grad_() for k, v in sd.items()}
    states, loss_ref = None, 0
    for w in range(L - 2):
        pred, states = model_ref.forward(ref, frames[:, w:w + 3], states)
        loss_ref = loss_ref + F.mse_loss(pred, gt[:, w + 1])
    loss_ref.backward()

    net = _net(sd, dev)
    net.reset_states()
    fd, gd = frames.to(dev), gt.to(dev)
    loss = 0
    for w in range(L - 2):
        loss = loss + train.mse_loss(net(fd[:, w:w + 3]), gd[:, w + 1])
    loss.backward()
    assert abs(loss.item() - loss_ref.item()) <= REL * abs(loss_ref.item())
    worst = {}
    for name, p in net.named_parameters():
        want = ref[name].grad
        assert p.grad is not None, name
        worst[name] = _rel(p.grad, want)
    bad = {k: v for k, v in worst.items() if v > 3 * REL}
    assert not bad, bad


def test_train_step_tracks_oracle_losses(dev):
    """Four full iterations (zero_grad, reset_states, windows, backward, Adam amsgrad): the loss trajectory follows the
    oracle trained with torch.optim.Adam step for step."""
    from esr_b200 import train
    sd = model_ref.seeded_state_dict(41)
    frames, gt = _frames(2, 5, 32, 32, 77)
    ref = {k: v.clone().requires_grad_() for k, v in sd.items()}
    opt_ref = torch.optim.Adam(list(ref.values()), lr=1e-3, weight_decay=1e-4, amsgrad=True)
    net = _net(sd, dev)
    opt = train.Adam(net.parameters(), lr=1e-3, weight_decay=1e-4, amsgrad=True)
    fd, gd = frames.to(dev), gt.to(dev)
    losses, losses_ref = [], []
    for it in range(4):
        opt_ref.zero_grad()
        states, lr_ = None, 0
        for w in range(3):
            pred, states = model_ref.forward(ref, frames[:, w:w + 3], states)
            lr_ = lr_ + F.mse_loss(pred, gt[:, w + 1])
        lr_.backward()
        opt_ref.step()
        losses_ref.append(lr_.item())
        losses.append(train.train_step(net, opt, fd, gd).item())
    for a, b in zip(losses, losses_ref):
        assert abs(a - b) <= 1e-3 * abs(b), (losses, losses_ref)
    # the inference plan sees the updated parameters (cached blob repacked after the in-place optimizer step)
    with torch.no_grad():
        net.reset_states()
        out = net(fd[:, 0:3].contiguous())
        want, _ = model_ref.forward({k: v.detach() for k, v in ref.items()}, frames[:, 0:3], None)
    assert _rel(out.cpu(), want) <= 2e-2


def test_batched_sequence_graph_equals_window_loop(dev):
    """forward over BxLx... with gradients on = the reference's loop of single-window forwards with carried state:
    same predictions, same loss, same gradients (up to fp32 summation order)."""
    from esr_b200 import train
    sd = model_ref.seeded_state_dict(51)
    frames, gt = _frames(2, 5, 24, 32, 9)
    fd, gd = frames.to(dev), gt.to(dev)
    a, b = _net(sd, dev), _net(sd, dev)
    loss_a, preds = 0, []
    for w in range(3):
        p = a(fd[:, w:w + 3])
        preds.append(p)
        loss_a = loss_a + train.mse_loss(p, gd[:, w + 1])
    loss_a.backward()
    pb = b(fd)
    assert pb.shape == (6, 2, 24, 32)
    loss_b = 3 * train.mse_loss(pb, gd[:, 1:4].transpose(0, 1).reshape(pb.shape))
    loss_b.backward()
    assert _rel(pb.detach(), torch.cat(preds, 0).detach().cpu()) <= 1e-5
    assert abs(loss_a.item() - loss_b.item()) <= 1e-5 * abs(loss_a.item())
    for (n, pa), (_, pbb) in zip(a.named_parameters(), b.named_parameters()):
        assert _rel(pbb.grad, pa.grad.cpu()) <= 1e-3, n
    for sa, sb in zip(a._train_states, b._train_states):
        assert _rel(sb.detach(), sa.detach().cpu()) <= 1e-5


def test_graphed_train_step_equals_eager(dev):
    """The CUDA-graph replay of the whole iteration (forward, backward, Adam with the device-side step counter) follows the
    eager iterations."""
    from esr_b200 import train
    sd = model_ref.seeded_state_dict(61)
    a, b = _net(sd, dev), _net(sd, dev)
    oa = train.Adam(a.parameters(), lr=1e-3, weight_decay=1e-4, amsgrad=True)
    ob = train.Adam(b.parameters(), lr=1e-3, weight_decay=1e-4, amsgrad=True)
    step_b = train.GraphedTrainStep(b, ob, (2, 4, 2, 32, 32), dev)
    assert int(ob.step_dev.item()) == 0                        # the warm-up iterations were rolled back
    for it in range(3):
        frames, gt = _frames(2, 4, 32, 32, 100 + it)
        la = train.train_step(a, oa, frames.to(dev), gt.to(dev)).item()
        lb = step_b(frames.to(dev), gt.to(dev)).item()
        assert abs(la - lb) <= 1e-4 * abs(la), (it, la, lb)
    assert int(ob.step_dev.item()) == 3
    for (n, pa), (_, pb) in zip(a.named_parameters(), b.named_parameters()):
        assert torch.allclose(pa.detach(), pb.detach(), rtol=0, atol=3e-3), n     # Adam normalises: +-lr per step at most


def _dcn_fp32_positions(inp, weight, bias, offset, mask, dg):
    """The oracle's DCNv2 in float64, with the sample positions formed in fp32 as the kernels (and the reference's CUDA
    code) form them: otherwise positions near integers floor differently and the offset gradient jumps by O(1) there."""
    from tests.test_tc_fp64_gpu import dcn_columns64
    cols = dcn_columns64(inp, offset, mask, dg)
    return torch.einsum("ok,bkhw->bohw", weight.reshape(weight.shape[0], -1), cols.flatten(1, 2)) + bias.view(1, -1, 1, 1)


def test_train_step_cfg2_size_vs_fp64_oracle_and_graph_replay(dev):
    """One train_step at the benchmark's cfg2 input (B=8, L=8, 256x256: 144 feature images of 32x32, the deferred ConvGRU
    weight gradients over 288 images): loss and all 68 parameter gradients against float64 autograd through the oracle.
    The samples are independent and the loss is a batch mean, so the reference is accumulated one sequence at a time:
    (1/B) sum_b grad(sum over windows of MSE(pred_bw, gt_bw)).  Then two iterations of the CUDA-graph replay follow the
    eager train_step."""
    import bench
    from esr_b200 import train
    torch.set_num_threads(bench.usable_cores())
    B, L, H, W = 8, 8, 256, 256
    sd = model_ref.seeded_state_dict(81)
    frames, gt = _frames(B, L, H, W, 83, lam=0.1)
    fd, gd = frames.to(dev), gt.to(dev)
    a = _net(sd, dev)
    oa = train.Adam(a.parameters(), lr=1e-3, weight_decay=1e-4, amsgrad=True)
    la = [train.train_step(a, oa, fd, gd).item()]
    grads = {n: p.grad.detach().cpu().clone() for n, p in a.named_parameters()}

    ref = {k: v.double().requires_grad_() for k, v in sd.items()}
    loss_ref = 0.0
    for s in range(B):
        states, ls = None, 0
        for w in range(L - 2):
            pred, states = model_ref.forward(ref, frames[s:s + 1, w:w + 3].double(), states, dcn_fn=_dcn_fp32_positions)
            ls = ls + F.mse_loss(pred, gt[s:s + 1, w + 1].double())
        (ls / B).backward()
        loss_ref += ls.item() / B
    assert abs(la[0] - loss_ref) <= REL * abs(loss_ref), (la[0], loss_ref)
    worst = {n: _rel(grads[n], ref[n].grad) for n in grads}
    top = sorted(worst.items(), key=lambda kv: -kv[1])[:4]
    print(f"[train cfg2] loss {la[0]:.6e} vs {loss_ref:.6e}; worst gradients " + ", ".join(f"{k} {v:.2e}" for k, v in top))
    assert len(worst) == 68
    # whole-network bar (as in test_sequence_gradients_vs_oracle_autograd): the fp32 forward and the fp64 oracle disagree on
    # the ReLU decisions of near-zero outputs, and where a layer's bias / weight gradient sums nearly cancel (convblock.0:
    # measured 1.03e-3 on its weight, 6.2e-4 on its bias, a plain fp32 sum) the few flipped pixels show up at that level
    bad = {k: v for k, v in worst.items() if v > 3 * REL}
    assert not bad, bad

    b = _net(sd, dev)
    ob = train.Adam(b.parameters(), lr=1e-3, weight_decay=1e-4, amsgrad=True)
    step_b = train.GraphedTrainStep(b, ob, (B, L, 2, H, W), dev)
    lb = [step_b(fd, gd).item()]
    f2, g2 = _frames(B, L, H, W, 84, lam=0.1)
    la.append(train.train_step(a, oa, f2.to(dev), g2.to(dev)).item())
    lb.append(step_b(f2.to(dev), g2.to(dev)).item())
    for it in range(2):
        assert abs(la[it] - lb[it]) <= 1e-4 * abs(la[it]), (it, la, lb)
    assert int(ob.step_dev.item()) == 2
    for (n, pa), (_, pb) in zip(a.named_parameters(), b.named_parameters()):
        assert torch.allclose(pa.detach(), pb.detach(), rtol=0, atol=3e-3), n


def test_deferred_gru_weight_gradients_equal_per_step(dev):
    """train_step batches the ConvGRU weight gradients of all steps into one launch per gate; same gradients as the
    per-step path."""
    from esr_b200 import train
    sd = model_ref.seeded_state_dict(71)
    frames, gt = _frames(2, 5, 24, 24, 13)
    fd, gd = frames.to(dev), gt.to(dev)
    a, b = _net(sd, dev), _net(sd, dev)
    target = gd[:, 1:4].transpose(0, 1).reshape(6, 2, 24, 24)
    (3 * train.mse_loss(a(fd), target)).backward()
    with train._defer_weight_grads() as d:
        (3 * train.mse_loss(b(fd), target)).backward()
        assert b.time_propagate.lstm.recurrent_block.out_gate.weight.grad is None     # not produced by backward itself
        d.flush()
    for (n, pa), (_, pb) in zip(a.named_parameters(), b.named_parameters()):
        assert pb.grad is not None, n
        assert _rel(pb.grad, pa.grad.cpu()) <= 1e-4, n


def test_adam_follows_a_torch_lr_scheduler_also_inside_the_graph(dev):
    """train_ours_cnt_seq.py:784 attaches a torch lr_scheduler to the optimizer: esr_b200.train.Adam is a torch.optim.Optimizer
    whose hyper-parameters are read from device memory by the update kernel, so StepLR changes reach eager steps AND replays of a
    captured iteration (ADVICE r1: by-value lr was frozen into the graph)."""
    from esr_b200 import train
    g = torch.Generator().manual_seed(11)
    shapes = [(16, 8, 3, 3), (16,), (7,)]
    ref = [torch.randn(s, generator=g).requires_grad_() for s in shapes]
    mine = [r.detach().clone().to(dev).requires_grad_() for r in ref]
    o_ref = torch.optim.Adam(ref, lr=1e-2, weight_decay=1e-4, amsgrad=True)
    o_mine = train.Adam(mine, lr=1e-2, weight_decay=1e-4, amsgrad=True)
    s_ref = torch.optim.lr_scheduler.StepLR(o_ref, step_size=2, gamma=0.1)
    s_mine = torch.optim.lr_scheduler.StepLR(o_mine, step_size=2, gamma=0.1)
    grads = [[torch.randn(s, generator=g) for s in shapes] for _ in range(6)]
    static = [torch.zeros(s, device=dev) for s in shapes]
    graph = None
    for step in range(6):
        for r, m, gr, st in zip(ref, mine, grads[step], static):
            r.grad = gr.clone()
            st.copy_(gr.to(dev))
        if step < 2:                                   # eager
            for m, st in zip(mine, static):
                m.grad.copy_(st)
            o_mine.step()
        else:                                          # the same update replayed from a CUDA graph captured at step 2
            if graph is None:
                o_mine.upload_hyper()
                keep = [t.clone() for t in (o_mine.flat, o_mine.exp_avg, o_mine.exp_avg_sq, o_mine.max_exp_avg_sq, o_mine.step_dev)]
                side = torch.cuda.Stream(dev)
                side.wait_stream(torch.cuda.current_stream(dev))
                graph = torch.cuda.CUDAGraph()
                with torch.cuda.stream(side):
                    for m, st in zip(mine, static):
                        m.grad.copy_(st)
                    o_mine.step()
                torch.cuda.current_stream(dev).wait_stream(side)
                for dst, src in zip((o_mine.flat, o_mine.exp_avg, o_mine.exp_avg_sq, o_mine.max_exp_avg_sq, o_mine.step_dev), keep):
                    dst.copy_(src)
                with torch.cuda.graph(graph):
                    for m, st in zip(mine, static):
                        m.grad.copy_(st)
                    o_mine.step()
                for dst, src in zip((o_mine.flat, o_mine.exp_avg, o_mine.exp_avg_sq, o_mine.max_exp_avg_sq, o_mine.step_dev), keep):
                    dst.copy_(src)
            o_mine.upload_hyper()
            graph.replay()
        o_ref.step()
        s_ref.step()
        s_mine.step()
        assert o_mine.param_groups[0]["lr"] == pytest.approx(o_ref.param_groups[0]["lr"])
        for r, m in zip(ref, mine):
            assert torch.allclose(m.detach().cpu(), r.detach(), rtol=3e-6, atol=3e-7), step
    assert o_ref.param_groups[0]["lr"] == pytest.approx(1e-5)


def test_logging_scalars_ride_in_the_gradient_bucket(dev):
    """SURVEY 8f rank 4: the two scalars the trainer logs (train_ours_cnt_seq.py:238-239: last-window MSE, summed loss) sit at the
    tail of the flat exchange buffer, so the iteration's single all-reduce covers them (no reduce_tensor barriers)."""
    from esr_b200 import train
    sd = model_ref.seeded_state_dict(2)
    frames, gt = _frames(2, 5, 16, 24, 91)
    net = _net(sd, dev)
    opt = train.Adam(net.parameters(), lr=1e-3, weight_decay=1e-4, amsgrad=True)
    seen = {}

    def fake_allreduce(buf):
        seen["n"] = buf.numel()
        seen["log"] = buf[-2:].clone()
        buf[-2:] *= 0.5                                # what an average with a rank holding zeros would do

    loss = train.train_step(net, opt, frames.to(dev), gt.to(dev), all_reduce=fake_allreduce)
    assert seen["n"] == 1813120 + 2 and opt.exchange.data_ptr() == opt.flat_grad.data_ptr()
    assert seen["log"][1].item() == pytest.approx(loss.item(), rel=1e-6)
    # last-window MSE against the oracle's prediction of that window
    ora = model_ref.OracleNet(sd)
    outs = [ora(frames[:, w:w + 3].contiguous()) for w in range(3)]
    want_last = F.mse_loss(outs[-1], gt[:, 3]).item()
    assert seen["log"][0].item() == pytest.approx(want_last, rel=2e-3)
    assert opt.log[1].item() == pytest.approx(0.5 * loss.item(), rel=1e-6)
