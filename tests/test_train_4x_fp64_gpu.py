"""The training step against float64 at the benchmark's 4x configurations: cfg3 (B 4, L 8, 512²) and cfg4 (B 2, L 16, 1024²).

The training kernels change shape with the problem size: k_wgrad_tc's slice split and tiles per CTA, the CUDA-core weight
gradients and bias sums over 28-32 full-resolution images, DCN backward over 56 images of 128², k_mse over 58.7 M elements and
k_adam's grid-stride loop over the whole 1 813 120-parameter buffer (3.5 passes of its 2048 x 256 grid).  This module checks
each of them at cfg4's counts, and the whole iteration bench.py times at cfg3 and cfg4.

  1. launch table: train.forward_sequence at cfg4 on the `meta` device, with the operators replaced by recorders, yields
     exactly the convolution, DCN, upsample and ConvGRU launches of CONV4 / DCN4 / UP4 / GRU4 (CPU test);
  2. every convolution of that table through train.conv2d (the ConvGRU gates through _defer_weight_grads, 42 steps of 4
     images), y / dx / dw / db, and the DCN forward and its five gradients, at cfg4's counts;
  3. esr_mse_loss(_ex) at cfg4's prediction size, esr_adam_step_dev on the full flat buffer, the upsample backward and the
     ConvGRU element-wise operators;
  4. one replay of train.GraphedTrainStep on bench.py's own weights and inputs at cfg3 and cfg4: loss, all 68 gradients and
     the last-window MSE against float64 autograd through the oracle, and at cfg3 two eager deterministic steps.

Norm and rule are those of tests/test_tc_fp64_gpu.py: err = max|got - ref64| / max|ref64| <= TOL and TOL <= err(degraded) / 4.
The float64 references of this module run on the GPU (torch's own float64 kernels): the layer references would take minutes
per case on the host at these sizes.  The split of an fp32 operand into bf16 hi + lo uses torch's round-to-nearest-even
conversion on the device, which `test_split_dev_is_split` ties to the bit-level `split` of the other modules.
TOL is about 4x the error measured on an H100 (DESIGN.md 3 lists the measurements).
"""
import gc
import math
import time
from collections import Counter

import pytest
import torch
import torch.nn.functional as F

from oracle import model_ref
from tests.test_small_conv_fp64_gpu import _taps, train_branches
from tests.test_tc_fp64_gpu import (ACT64, _act_grad, _check_images, _lattice_offsets, check, dcn_columns64, rel, split,
                                    wgrad_geometry)

pytestgpu = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------------------------
# helpers (any device)
# ------------------------------------------------------------------------------------------------------------------
def split_dev(x):
    """split() on x's own device: hi = bf16(x), lo = bf16(x - hi), as fp32 tensors (torch's conversion rounds to nearest
    even, as bf16_rne does)."""
    x = x.detach().float()
    hi = x.to(torch.bfloat16).float()
    return hi, (x - hi).to(torch.bfloat16).float()


def drop_cross(op, a, b):
    """op(A_hi, B_hi) + op(A_hi, B_lo) in float64 (the split product without A_lo B_hi) for a bilinear op."""
    ah = split_dev(a)[0].double()
    bh, bl = split_dev(b)
    return op(ah, bh.double() + bl.double())


def bf16_dev(x):
    return x.detach().float().to(torch.bfloat16).double()


def wgrad64(x, g, k, stride, chunk=4):
    """dw[co, ci, ky, kx] = sum over images and output pixels of g * the shifted, strided x, in float64, tap by tap and
    a few images at a time (no im2col: at 1024² that would be several GB)."""
    co, ci = g.shape[1], x.shape[1]
    dw = torch.zeros(co, ci, k, k, dtype=torch.float64, device=x.device)
    for i in range(0, x.shape[0], chunk):
        gi = g[i:i + chunk].double()
        for t, xs in enumerate(_taps(x[i:i + chunk].double(), k, stride, k // 2)):
            dw[:, :, t // k, t % k] += torch.einsum("nohw,nchw->oc", gi, xs)
    return dw


def adam64(p, grads, lrs, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-4):
    """torch.optim.Adam(amsgrad=True) restated in float64: -> (param, exp_avg, exp_avg_sq, max_exp_avg_sq) after one step
    per (gradient, lr)."""
    b1, b2 = betas
    p = p.double().clone()
    m, v, vmax = torch.zeros_like(p), torch.zeros_like(p), torch.zeros_like(p)
    for t, (g, lr) in enumerate(zip(grads, lrs), 1):
        g = g.double() + weight_decay * p
        m = b1 * m + (1 - b1) * g
        v = b2 * v + (1 - b2) * g * g
        vmax = torch.maximum(vmax, v)
        p = p - lr / (1 - b1 ** t) * m / (vmax.sqrt() / math.sqrt(1 - b2 ** t) + eps)
    return p, m, v, vmax


def oracle_step64(sd, frames, gt, dev, ckpt=True):
    """The training iteration's loss, last-window MSE and parameter gradients in float64 on `dev`:
    (1/B) sum_b grad sum_w MSE(pred_bw, gt_b,w+1), model_ref.forward one sample at a time with the ConvGRU state carried
    across windows, DCN sample positions formed in fp32 as the kernels form them.  ckpt: each window under
    torch.utils.checkpoint, so only window boundaries stay alive between the forward and the backward."""
    from torch.utils.checkpoint import checkpoint
    from tests.test_train_gpu import _dcn_fp32_positions
    ref = {k: v.detach().to(dev, torch.float64).requires_grad_() for k, v in sd.items()}
    B, L = frames.shape[:2]

    def window(inp, states):
        return model_ref.forward(ref, inp, states, dcn_fn=_dcn_fp32_positions)

    loss, last = 0.0, 0.0
    for s in range(B):
        fs, gs = frames[s:s + 1].to(dev, torch.float64), gt[s:s + 1].to(dev, torch.float64)
        states, ls = None, 0
        for w in range(L - 2):
            inp = fs[:, w:w + 3]
            pred, states = checkpoint(window, inp, states, use_reentrant=False) if ckpt else window(inp, states)
            mse = F.mse_loss(pred, gs[:, w + 1])
            ls = ls + mse
        last += mse.item() / B
        (ls / B).backward()
        loss += ls.item() / B
        del states, ls, pred, mse
    return loss, last, {k: v.grad.detach() for k, v in ref.items()}


# ------------------------------------------------------------------------------------------------------------------
# 1. the launch table of train.forward_sequence at the benchmark's 4x shapes (CPU)
# ------------------------------------------------------------------------------------------------------------------
def enumerate_launches(monkeypatch, B, L, H, W):
    """Counter of the operator launches of train.forward_sequence for frames BxLx2xHxW, on the `meta` device:
    ("conv", Cin, Cout, k, stride, act, n_img, H, W), ("dcn", n_img, C, H, W), ("up", n_img, C, H, W) (input shape),
    ("gru_hr" | "gru_blend", n_img, C, H, W)."""
    from esr_b200 import train
    from esr_b200.model import DeepRecurrNet
    seen = Counter()

    def conv(x, w, b, stride=1, act=None, defer=None):
        Cout, Cin, k, _ = w.shape
        n, _, H_, W_ = x.shape
        seen[("conv", Cin, Cout, k, int(stride), act, n, H_, W_)] += 1
        Ho, Wo = (H_ + 2 * (k // 2) - k) // stride + 1, (W_ + 2 * (k // 2) - k) // stride + 1
        return torch.empty(n, Cout, Ho, Wo, device=x.device)

    def dcn(inp, offset, mask, weight, bias, dg=8):
        seen[("dcn",) + tuple(inp.shape)] += 1
        return torch.empty_like(inp)

    def up(x):
        seen[("up",) + tuple(x.shape)] += 1
        n, C, H_, W_ = x.shape
        return torch.empty(n, C, 2 * H_, 2 * W_, device=x.device)

    class Hr:
        @staticmethod
        def apply(h, zr):
            seen[("gru_hr",) + tuple(h.shape)] += 1
            return torch.empty_like(h)

    class Blend:
        @staticmethod
        def apply(h, zr, o):
            seen[("gru_blend",) + tuple(h.shape)] += 1
            return torch.empty_like(h)

    for name, fake in (("conv2d", conv), ("dcn_v2", dcn), ("upsample2x", up), ("_GruHRFn", Hr), ("_GruBlendFn", Blend)):
        monkeypatch.setattr(train, name, fake)
    model = DeepRecurrNet(inch=2, basech=8, num_frame=3).to("meta")
    train.forward_sequence(model, torch.empty(B, L, 2, H, W, device="meta"))
    return seen


# cfg4 (B 2, L 16, 1024²: 32 frames, 14 windows, 84 window slots of 128² features, 28 decoder images)
# id: (Cin, Cout, k, stride, act, images per launch, H, W, launches: the ConvGRU steps, deferred), input size H x W
CONV4 = {
    "head_2_8": (2, 8, 3, 1, "relu", 32, 1024, 1024, 1),
    "enc0_8_16_s2": (8, 16, 3, 2, "relu", 32, 1024, 1024, 1),
    "enc1_16_32_s2": (16, 32, 3, 2, "relu", 32, 512, 512, 1),
    "enc2_32_64_s2": (32, 64, 3, 2, "relu", 32, 256, 256, 1),
    "pred_map0_128_64": (128, 64, 3, 1, "relu", 62, 128, 128, 1),
    "pred_map1_64_1": (64, 1, 3, 1, "sigmoid", 62, 128, 128, 1),
    "local_fusion_conv1_192_192": (192, 192, 3, 1, "relu", 84, 128, 128, 1),
    "local_fusion_conv2_192_192": (192, 192, 3, 1, None, 84, 128, 128, 1),
    "local_fusion1_192_64": (192, 64, 3, 1, None, 84, 128, 128, 1),
    "lstm_conv_64_64": (64, 64, 3, 1, "relu", 84, 128, 128, 1),
    "gru_zr_128_128": (128, 128, 3, 1, "sigmoid", 4, 128, 128, 42),
    "gru_o_128_64": (128, 64, 3, 1, "tanh", 4, 128, 128, 42),
    "global_fusion_128_64_1x1": (128, 64, 1, 1, "relu", 84, 128, 128, 1),
    "stf_128_64": (128, 64, 3, 1, "relu", 56, 128, 128, 3),          # offset[0], convblock[0], dcn_fusion[0]
    "stf_64_64": (64, 64, 3, 1, None, 56, 128, 128, 3),              # offset[1], convblock[1], dcn_fusion[1]
    "offset_mask_64_216": (64, 216, 3, 1, None, 56, 128, 128, 1),
    "kernel_64_2_1x1": (64, 2, 1, 1, "sigmoid", 56, 128, 128, 1),
    "dense_fusion0_192_64": (192, 64, 3, 1, "relu", 28, 128, 128, 1),
    "dense_fusion1_64_64": (64, 64, 3, 1, None, 28, 128, 128, 1),
    "atten0_64_1": (64, 1, 3, 1, "sigmoid", 32, 128, 128, 1),
    "recon0_64_32": (64, 32, 3, 1, "relu", 28, 256, 256, 1),
    "atten1_32_1": (32, 1, 3, 1, "sigmoid", 32, 256, 256, 1),
    "recon1_32_16": (32, 16, 3, 1, "relu", 28, 512, 512, 1),
    "atten2_16_1": (16, 1, 3, 1, "sigmoid", 32, 512, 512, 1),
    "recon2_16_8": (16, 8, 3, 1, "relu", 28, 1024, 1024, 1),
    "tail_8_2": (8, 2, 3, 1, "relu", 28, 1024, 1024, 1),
}
DCN4 = (56, 64, 128, 128)
UP4 = [(28, 64, 128, 128), (28, 32, 256, 256), (28, 16, 512, 512)]
GRU4 = ((4, 64, 128, 128), 42)


def test_launch_table_is_the_networks_at_cfg4(monkeypatch):
    seen = enumerate_launches(monkeypatch, 2, 16, 1024, 1024)
    want = Counter({("conv",) + c[:8]: c[8] for c in CONV4.values()})
    want[("dcn",) + DCN4] = 1
    for s in UP4:
        want[("up",) + s] = 1
    want[("gru_hr",) + GRU4[0]] = want[("gru_blend",) + GRU4[0]] = GRU4[1]
    assert seen == want
    assert len(seen) == 32 and len(CONV4) == 26
    # cfg3 (B 4, L 8, 512²) runs the same layers at other counts
    seen3 = enumerate_launches(monkeypatch, 4, 8, 512, 512)
    assert {k[:6] for k in seen3 if k[0] == "conv"} == {k[:6] for k in seen if k[0] == "conv"}
    assert len(seen3) == 32


def test_split_dev_is_split():
    g = torch.Generator().manual_seed(7)
    x = torch.randn(1 << 16, generator=g) * torch.exp2(torch.randint(-30, 30, (1 << 16,), generator=g).float())
    for a, b in zip(split_dev(x), split(x)):
        assert torch.equal(a, b)


def test_adam64_is_torch_adam():
    """The float64 restatement follows torch.optim.Adam(amsgrad, weight_decay) in float64, lr changed between steps."""
    g = torch.Generator().manual_seed(9)
    p0 = torch.randn(1000, generator=g, dtype=torch.float64)
    grads = [torch.randn(1000, generator=g, dtype=torch.float64) * (10.0 if t % 2 == 0 else 0.1) for t in range(6)]
    lrs = [1e-3, 1e-3, 5e-4, 5e-4, 2e-3, 1e-4]
    p = p0.clone().requires_grad_()
    opt = torch.optim.Adam([p], lr=lrs[0], weight_decay=1e-4, amsgrad=True, foreach=False)
    for gr, lr in zip(grads, lrs):
        opt.param_groups[0]["lr"] = lr
        p.grad = gr.clone()
        opt.step()
    mine = adam64(p0, grads, lrs)
    st = opt.state[p]
    for got, want in zip(mine, (p.detach(), st["exp_avg"], st["exp_avg_sq"], st["max_exp_avg_sq"])):
        assert (got - want).abs().max().item() <= 1e-15 * want.abs().max().item()


def test_checkpointed_oracle_equals_unwrapped():
    """Each window under torch.utils.checkpoint gives the unwrapped oracle's loss and gradients bit for bit."""
    g = torch.Generator().manual_seed(5)
    frames = torch.poisson(torch.full((2, 4, 2, 16, 24), 0.3), generator=g)
    gt = torch.poisson(torch.full((2, 4, 2, 16, 24), 0.3), generator=g)
    sd = model_ref.seeded_state_dict(3)
    a = oracle_step64(sd, frames, gt, "cpu", ckpt=True)
    b = oracle_step64(sd, frames, gt, "cpu", ckpt=False)
    assert a[0] == b[0] and a[1] == b[1]
    assert all(torch.equal(a[2][k], b[2][k]) for k in sd)


# ------------------------------------------------------------------------------------------------------------------
# GPU cases
# ------------------------------------------------------------------------------------------------------------------
# TOL per (kernel, output): measured max err at cfg4's counts on one H100 80GB HBM3 (700 W power limit) x ~4 (DESIGN.md 3)
TOL4 = {
    "k_conv_tc.y": 1e-4,            # measured 2.5e-5 (ConvGRU candidate, tanh)
    "k_conv_mma.y": 4.5e-5,         # 1.1e-5
    "k_conv_tc.dx": 4e-5,           # 9.6e-6
    "k_conv_mma.dx": 4.5e-5,        # 1.1e-5
    "k_conv_dgrad_s2.dx": 2e-6,     # 4.8e-7
    "k_conv_dgrad_g<1>.dx": 5e-7,   # 1.2e-7
    "k_wgrad_tc.dw": 7e-5,          # 1.7e-5 (6.3e-4 before the accumulators were flushed every 32 tiles)
    "k_conv_wgrad_r.dw": 1.5e-5,    # 3.7e-6
    "k_conv_wgrad_g<1>.dw": 5e-6,   # 1.2e-6
    "db": 9e-6,                     # 2.2e-6: fp32 sums over up to 32 x 1024² pixels
    "dcn.out": 3.5e-5,              # 8.9e-6
    "dcn.grad_input": 2e-5,         # 5.0e-6
    "dcn.grad_offset": 2.2e-5,      # 5.5e-6
    "dcn.grad_mask": 2.5e-5,        # 6.1e-6
    "dcn.grad_weight": 1.6e-5,      # 3.9e-6
    "dcn.grad_bias": 7e-6,          # 1.8e-6
    "mse.loss": 1.1e-6,             # 2.7e-7
    "mse.grad": 4e-7,               # 1.0e-7
    "adam.param": 8.5e-5,           # 2.1e-5: the parameters' own fp32 rounding against updates of ~1e-3
    # 1.3e-5: the kernel reads beta2 as fp32 (0.99900001), so its 1 - beta2 is 1.3e-5 below torch's; the bias correction
    # uses the same beta2, so the step itself is unaffected (adam.param)
    "adam.moments": 5.5e-5,
    "up2.dx": 5.5e-7,               # 1.3e-7
    "gru": 3.5e-7,                  # 8.6e-8
}


def _check(name, kind, got, ref, deg=None, deg_is=None):
    check(name, kind, got, ref, deg, deg_is or "", tol=TOL4[kind])


@pytest.fixture(scope="module")
def dev():
    import bench
    torch.set_num_threads(bench.usable_cores())
    return torch.device("cuda:0")


def _free():
    gc.collect()
    torch.cuda.empty_cache()


def _randn(gen, *shape, scale=1.0):
    return torch.randn(*shape, generator=gen, device=gen.device) * scale


@pytestgpu
@pytest.mark.parametrize("name", list(CONV4))
def test_train_conv2d_cfg4_vs_fp64(dev, name):
    """train.conv2d forward and backward at one cfg4 launch's counts; the ConvGRU gates as train_step runs them: 42 steps
    of 4 images, dw / db flushed once over all 168 images.  y and dx on a spread of images, dw and db over all of them."""
    from esr_b200 import train
    Cin, Cout, k, stride, act, n, H, W, launches = CONV4[name]
    steps = launches if name.startswith("gru") else 1
    B = n * steps
    k_fwd, k_dx, k_dw = train_branches(Cin, Cout, k, stride, act)
    geo = wgrad_geometry(B, Cin, Cout, k, H, W) if k_dw == "k_wgrad_tc" else None
    if name.startswith("gru"):
        cfg2 = wgrad_geometry(288, Cin, Cout, k, 32, 32)                   # the same gate at cfg2: 18 steps of 16 images
        assert k_dw == "k_wgrad_tc" and geo["tiles_per_cta"] >= 9 * cfg2["tiles_per_cta"], (geo, cfg2)
    need_dx = Cin != 2                                                         # the frames need no gradient
    t0 = time.time()
    gen = torch.Generator(device=dev).manual_seed(sum(map(ord, name)))
    x = _randn(gen, B, Cin, H, W)
    w = _randn(gen, Cout, Cin, k, k, scale=1.0 / math.sqrt(Cin * k * k))
    b = _randn(gen, Cout, scale=0.1)
    pad = k // 2
    Ho, Wo = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
    dy = _randn(gen, B, Cout, Ho, Wo)

    xg, wg, bg = x.clone().requires_grad_(need_dx), w.clone().requires_grad_(), b.clone().requires_grad_()
    if steps > 1:
        sunk = {}
        with train._defer_weight_grads() as d:
            y = torch.cat([train.conv2d(xg[i * n:(i + 1) * n], wg, bg, stride, act,
                                        defer=("k", lambda dw_, db_: sunk.update(dw=dw_, db=db_))) for i in range(steps)], 0)
            y.backward(dy)
            assert wg.grad is None
            d.flush()
        dw_got, db_got = sunk["dw"], sunk["db"]
    else:
        y = train.conv2d(xg, wg, bg, stride, act)
        y.backward(dy)
        dw_got, db_got = wg.grad, bg.grad
    y_got, dx_got = y.detach(), xg.grad
    del y, xg
    torch.cuda.synchronize()
    t_gpu = time.time() - t0

    sel = torch.tensor(_check_images(B, 3), device=dev)
    xs = x[sel]
    conv = lambda a, bb: F.conv2d(a, bb, stride=stride, padding=pad)                                     # noqa: E731
    b64 = b.double().view(1, -1, 1, 1)
    y64 = ACT64[act](conv(xs.double(), w.double()) + b64)
    if k_fwd in ("k_conv_tc", "k_conv_mma"):
        y_deg, y_is = ACT64[act](drop_cross(conv, xs, w) + b64), "A_lo B_hi dropped"
    else:
        y_deg, y_is = ACT64[act](conv(bf16_dev(xs), w.double()) + b64), "x rounded to bf16"
    # the backward on the y it is handed (the forward's output): g = dy * act'(y) in fp32, as the kernels form it
    g32 = dy * _act_grad(y_got, act)
    g64 = dy.double() * _act_grad(y_got.double(), act)
    db64 = g64.sum((0, 2, 3))
    dw64 = wgrad64(x, g64, k, stride)
    del g64
    if k_dw == "k_wgrad_tc" and geo["a_is_x"]:                           # M side = x: A = x, B = g
        dw_deg, dw_is = _wgrad_drop_cross(x, g32, k, stride, a_is_x=True), "A_lo B_hi dropped"
    elif k_dw == "k_wgrad_tc":                                           # M side = g: A = g, B = x
        dw_deg, dw_is = _wgrad_drop_cross(x, g32, k, stride, a_is_x=False), "A_lo B_hi dropped"
    else:
        dw_deg, dw_is = wgrad64(split_dev(x)[0], g32, k, stride), "x rounded to bf16"
    geo_s = "" if geo is None else (f", wgrad tiles {geo['n_tiles']}, slices {geo['slices']}, >= {geo['tiles_per_cta']} tiles "
                                    f"per CTA, M side {'x' if geo['a_is_x'] else 'g'} ({geo['m_ch']} ch)")
    print(f"[train4x] {name}: {Cin}->{Cout} k{k} s{stride} {act}, {steps} x {n} x {H}x{W}: forward {k_fwd}, dx "
          f"{k_dx if need_dx else '-'}, dw {k_dw}{geo_s}; images checked for y / dx {len(sel)}/{B}; GPU {t_gpu:.1f} s")
    _check(f"{name}.y", f"{k_fwd}.y", y_got[sel], y64, y_deg, y_is)
    if need_dx:
        dxop = lambda gg, bb: torch.nn.grad.conv2d_input((len(sel), Cin, H, W), bb, gg, stride=stride, padding=pad)  # noqa: E731
        gs64 = dy[sel].double() * _act_grad(y_got[sel].double(), act)
        dx64 = dxop(gs64, w.double())
        if k_dx in ("k_conv_tc", "k_conv_mma"):
            dx_deg, dx_is = drop_cross(dxop, g32[sel], w), "A_lo B_hi dropped"
        else:
            dx_deg, dx_is = dxop(bf16_dev(g32[sel]), w.double()), "g rounded to bf16"
        _check(f"{name}.dx", f"{k_dx}.dx", dx_got[sel], dx64, dx_deg, dx_is)
    _check(f"{name}.dw", f"{k_dw}.dw", dw_got, dw64, dw_deg, dw_is)
    _check(f"{name}.db", "db", db_got, db64)
    print(f"[train4x] {name}: total {time.time() - t0:.1f} s")
    del x, dy, y_got, dx_got, g32
    _free()


def _wgrad_drop_cross(x, g32, k, stride, a_is_x):
    """k_wgrad_tc without A_lo B_hi: A = x, B = g (a_is_x) or A = g, B = x; = A_hi (B_hi + B_lo) in float64."""
    xh, xl = split_dev(x)
    gh, gl = split_dev(g32)
    if a_is_x:
        return wgrad64(xh, gh.double() + gl.double(), k, stride)
    return wgrad64(xh.double() + xl.double(), gh, k, stride)


@pytestgpu
@pytest.mark.parametrize("offsets", ["random", "lattice"])
def test_dcn_cfg4_vs_fp64(dev, offsets):
    """Forward and the five gradients of `_ext.dcn_v2_forward / backward` (64 -> 64, 8 groups) on cfg4's 56 images of 128²,
    with random offsets and with offsets that land on and around the borders."""
    from esr_b200 import dcn_v2_ext as ext
    B, C, H, W = DCN4
    G = 8
    t0 = time.time()
    gen = torch.Generator(device=dev).manual_seed(56 + len(offsets))
    if offsets == "random":
        off = _randn(gen, B, G * 18, H, W, scale=2.0)
    else:
        off = _lattice_offsets(torch.Generator().manual_seed(57), B, G, H, W).to(dev)
    x = _randn(gen, B, C, H, W)
    w = _randn(gen, C, C, 3, 3, scale=1 / 24)
    b = _randn(gen, C, scale=0.1)
    m = torch.rand(B, G * 9, H, W, generator=gen, device=dev)
    go = _randn(gen, B, C, H, W)
    out_got = ext.dcn_v2_forward(x, w, b, off, m, 3, 3, 1, 1, 1, 1, 1, 1, G)
    grads_got = ext.dcn_v2_backward(x, w, b, off, m, go, 3, 3, 1, 1, 1, 1, 1, 1, G)
    torch.cuda.synchronize()
    t_gpu = time.time() - t0

    w2 = w.reshape(C, C * 9)
    w2h, w2l = split_dev(w2)
    w2s = w2h.double() + w2l.double()                                    # B operand of the degraded products
    b64 = b.double().view(1, -1, 1, 1)
    names = ["grad_input", "grad_offset", "grad_mask"]
    ref = {k: [] for k in ["out", "out_deg"] + names + [n + "_deg" for n in names]}
    gw, gw_deg = (torch.zeros(C, C * 9, dtype=torch.float64, device=dev) for _ in range(2))
    for i in range(0, B, 4):                                             # bounded memory: chunks of images
        sl = slice(i, i + 4)
        leaves = [t[sl].double().requires_grad_() for t in (x, off, m)]
        cols = dcn_columns64(leaves[0], leaves[1], leaves[2], G)
        cflat = cols.detach().flatten(1, 2)
        ref["out"].append(torch.einsum("ok,bkhw->bohw", w2.double(), cflat) + b64)
        ref["out_deg"].append(torch.einsum("ok,bkhw->bohw", w2s, split_dev(cflat.float())[0].double()) + b64)
        gcols = torch.einsum("ok,bohw->bkhw", w2.double(), go[sl].double()).view_as(cols)
        gcols_deg = torch.einsum("ok,bohw->bkhw", w2s, split_dev(go[sl])[0].double()).view_as(cols)
        exact = torch.autograd.grad(cols, leaves, gcols, retain_graph=True)
        degr = torch.autograd.grad(cols, leaves, gcols_deg)
        for n_, e_, d_ in zip(names, exact, degr):
            ref[n_].append(e_)
            ref[n_ + "_deg"].append(d_)
        gw += torch.einsum("bohw,bkhw->ok", go[sl].double(), cflat)
        with torch.no_grad():                                            # features read without their lo plane
            cols_hi = dcn_columns64(split_dev(x[sl])[0].double(), off[sl].double(), m[sl].double(), G)
        gw_deg += torch.einsum("bohw,bkhw->ok", go[sl].double(), cols_hi.flatten(1, 2))
        del leaves, cols, cflat, gcols, gcols_deg, exact, degr, cols_hi
    cat = {k: torch.cat(v, 0) for k, v in ref.items()}
    del ref
    print(f"[train4x] dcn_{offsets}: {B} x {C} x {H}x{W}, 8 groups; GPU {t_gpu:.1f} s, float64 {time.time() - t0 - t_gpu:.1f} s")
    _check(f"dcn_{offsets}.out", "dcn.out", out_got, cat["out"], cat["out_deg"], "A_lo B_hi dropped")
    for n_, got in zip(names, grads_got[:3]):
        _check(f"dcn_{offsets}.{n_}", f"dcn.{n_}", got, cat[n_], cat[n_ + "_deg"], "A_lo B_hi dropped")
    _check(f"dcn_{offsets}.grad_weight", "dcn.grad_weight", grads_got[3], gw.view(C, C, 3, 3), gw_deg.view(C, C, 3, 3),
           "features without lo plane")
    _check(f"dcn_{offsets}.grad_bias", "dcn.grad_bias", grads_got[4], go.double().sum((0, 2, 3)))
    del cat
    _free()


# ------------------------------------------------------------------------------------------------------------------
# 3. the training step's own kernels at the benchmark's sizes
# ------------------------------------------------------------------------------------------------------------------
@pytestgpu
@pytest.mark.parametrize("mode", ["default", "deterministic"])
def test_mse_loss_cfg4_vs_fp64(dev, mode):
    """esr_mse_loss_ex over cfg4's prediction (14 windows x 2 samples x 2 x 1024²): the loss and 2 d / n * scale per element.
    The degraded loss drops the grid-stride loop's last pass (58 720 256 is exactly 224 passes of its 1024 x 256 grid)."""
    from esr_b200 import _lib, train
    n = 28 * 2 * 1024 * 1024
    scale = 14.0
    gen = torch.Generator(device=dev).manual_seed(58)
    pred, tgt = _randn(gen, n), torch.poisson(torch.full((n,), 0.1, device=dev), generator=gen)
    loss, grad = torch.empty(1, device=dev), torch.empty_like(pred)
    L = _lib.lib()
    flags = _lib.DETERMINISTIC if mode == "deterministic" else 0
    nbytes = L.esr_mse_loss_workspace_bytes_ex(n, flags)
    assert (nbytes == 4096) == (mode == "deterministic")                 # one partial per block of the 1024
    ws = train._ws(nbytes, dev)
    _lib.check(L.esr_mse_loss_ex(_lib.ptr(pred), _lib.ptr(tgt), n, _lib.ptr(loss), _lib.ptr(grad), scale, flags, _lib.ptr(ws),
                                 nbytes, _lib.stream_ptr()), "esr_mse_loss_ex")
    d = pred.double() - tgt.double()
    loss64 = (d * d).mean()
    stride = 1024 * 256
    assert n % stride == 0 and n // stride == 224
    loss_deg = (d[:n - stride] * d[:n - stride]).sum() / n
    print(f"[train4x] mse_{mode}: n {n}, loss {loss.item():.7e} vs {loss64.item():.7e}")
    _check(f"mse_{mode}.loss", "mse.loss", loss, loss64.view(1), loss_deg.view(1), "last grid-stride pass dropped")
    _check(f"mse_{mode}.grad", "mse.grad", grad, 2.0 * d / n * scale)


@pytestgpu
def test_adam_full_buffer_vs_fp64(dev):
    """esr_adam_step_dev on the network's whole flat buffer (1 813 120 parameters: 3.5 passes of the 2048 x 256 grid), six
    amsgrad steps with weight decay, gradients alternating between x10 and x0.1, lr changed through `hyper` between steps,
    against the float64 restatement of torch.optim.Adam.  The degraded kernel ran the grid-stride loop's first pass only."""
    import bench
    from esr_b200 import train
    from esr_b200.model import DeepRecurrNet
    net = DeepRecurrNet(inch=2, basech=8, num_frame=3)
    net.load_state_dict(bench.synth_weights(0))
    net = net.to(dev)
    opt = train.Adam(net.parameters(), lr=1e-3, weight_decay=1e-4, amsgrad=True)
    n = opt.flat.numel()
    assert n == 1813120 and n > 3 * 2048 * 256
    p0 = opt.flat.clone()
    gen = torch.Generator(device=dev).manual_seed(1813)
    grads = [_randn(gen, n, scale=10.0 if t % 2 == 0 else 0.1) for t in range(6)]
    lrs = [1e-3, 1e-3, 5e-4, 5e-4, 2e-3, 1e-4]
    for gr, lr in zip(grads, lrs):
        opt.param_groups[0]["lr"] = lr
        opt.flat_grad.copy_(gr)
        opt.step()
    assert int(opt.step_dev.item()) == 6
    p64, m64, v64, vmax64 = adam64(p0, grads, lrs)
    upd64 = p64 - p0.double()
    upd_deg = upd64.clone()
    upd_deg[2048 * 256:] = 0
    _check("adam.update", "adam.param", opt.flat.double() - p0.double(), upd64, upd_deg, "first grid-stride pass only")
    for nm, got, want in (("exp_avg", opt.exp_avg, m64), ("exp_avg_sq", opt.exp_avg_sq, v64), ("max_exp_avg_sq", opt.max_exp_avg_sq, vmax64)):
        _check(f"adam.{nm}", "adam.moments", got, want)


@pytestgpu
@pytest.mark.parametrize("shape", UP4)
def test_upsample2x_backward_cfg4_vs_fp64(dev, shape):
    from esr_b200 import train
    gen = torch.Generator(device=dev).manual_seed(sum(shape))
    n, C, H, W = shape
    x = _randn(gen, *shape).requires_grad_()
    dy = _randn(gen, n, C, 2 * H, 2 * W)
    train.upsample2x(x).backward(dy)
    x64 = x.detach().double().requires_grad_()
    F.interpolate(x64, scale_factor=2, mode="bilinear", align_corners=False).backward(dy.double())
    xd = x.detach().double().requires_grad_()
    F.interpolate(xd, scale_factor=2, mode="bilinear", align_corners=False).backward(bf16_dev(dy))
    _check(f"up2_bwd_{n}x{C}x{H}x{W}", "up2.dx", x.grad, x64.grad, xd.grad, "dy rounded to bf16")
    del x, dy, x64, xd
    _free()


@pytestgpu
@pytest.mark.parametrize("shape", [GRU4[0], (3, 64, 13, 7)])
def test_gru_ops_vs_fp64(dev, shape):
    """esr_gru_hr / esr_gru_blend and their backwards on 2B images of the cfg4 ConvGRU step (1 M elements per image: 16
    grid-stride passes), and on a chw (64 x 13 x 7) that is not a multiple of 256."""
    from esr_b200 import train
    gen = torch.Generator(device=dev).manual_seed(sum(shape) + 1)
    B, C, H, W = shape
    h = _randn(gen, B, C, H, W).requires_grad_()
    zr = torch.sigmoid(_randn(gen, B, 2 * C, H, W)).requires_grad_()
    o = torch.tanh(_randn(gen, B, C, H, W)).requires_grad_()
    g1, g2 = _randn(gen, B, C, H, W), _randn(gen, B, C, H, W)
    hr = train._GruHRFn.apply(h, zr)
    hr.backward(g1)
    hr_grads = (h.grad.clone(), zr.grad.clone())
    h.grad = zr.grad = None
    hn = train._GruBlendFn.apply(h, zr, o)
    hn.backward(g2)
    assert bool((hr_grads[1][:, :C] == 0).all()) and bool((zr.grad[:, C:] == 0).all())   # the other gate's half: zero
    h64, zr64, o64 = (t.detach().double().requires_grad_() for t in (h, zr, o))
    z64, r64 = zr64[:, :C], zr64[:, C:]
    hr64 = h64 * r64
    hr64.backward(g1.double())
    sid = "x".join(map(str, shape))
    _check(f"gru_hr_{sid}", "gru", hr, hr64)
    _check(f"gru_hr_{sid}.dh", "gru", hr_grads[0], h64.grad)
    _check(f"gru_hr_{sid}.dzr", "gru", hr_grads[1], zr64.grad)
    h64.grad = zr64.grad = None
    hn64 = h64 * (1 - z64) + o64 * z64
    hn64.backward(g2.double())
    _check(f"gru_blend_{sid}", "gru", hn, hn64)
    for nm, got, want in (("dh", h.grad, h64.grad), ("dzr", zr.grad, zr64.grad), ("do", o.grad, o64.grad)):
        _check(f"gru_blend_{sid}.{nm}", "gru", got, want)


# ------------------------------------------------------------------------------------------------------------------
# 4. the iteration bench.py times, as a whole, at cfg3 and cfg4
# ------------------------------------------------------------------------------------------------------------------
REL = 1e-3          # loss and last-window MSE (BASELINE.json's fp32 bar)
GRAD_REL = 3e-3     # whole-network gradients, the bar of test_train_gpu's cfg2 iteration (ReLU decisions near zero)


def bench_inputs(name):
    """bench.py's measure_training inputs for workload `name` (rank 0): synth_weights(0), frames then gt from seed 200."""
    import bench
    wl = bench.WORKLOADS[name]
    B, L, H, W = wl["B"], wl["L"], wl["lr"][0] * wl["scale"], wl["lr"][1] * wl["scale"]
    g = torch.Generator().manual_seed(200)
    frames = torch.poisson(torch.full((B, L, 2, H, W), 0.1), generator=g)
    gt = torch.poisson(torch.full((B, L, 2, H, W), 0.1), generator=g)
    return bench.synth_weights(0), frames, gt


def _reference(name, dev):
    sd, frames, gt = bench_inputs(name)
    _free()
    torch.cuda.reset_peak_memory_stats(dev)
    t0 = time.time()
    loss, last, grads = oracle_step64(sd, frames, gt, dev)
    torch.cuda.synchronize()
    print(f"[train4x] {name} float64 reference: {time.time() - t0:.1f} s, peak GPU memory "
          f"{torch.cuda.max_memory_allocated(dev) / 2**30:.2f} GiB")
    grads = {k: v.cpu() for k, v in grads.items()}
    _free()
    return loss, last, grads


@pytest.fixture(scope="module")
def cfg3_ref(dev):
    return _reference("cfg3", dev)


def _compare(tag, loss, last, grads, ref):
    loss_ref, last_ref, g_ref = ref
    worst = {n: rel(grads[n], g_ref[n]) for n in g_ref}
    top = sorted(worst.items(), key=lambda kv: -kv[1])[:4]
    print(f"[train4x] {tag}: loss {loss:.7e} vs {loss_ref:.7e} ({abs(loss - loss_ref) / abs(loss_ref):.1e}), last-window MSE "
          f"{last:.7e} vs {last_ref:.7e}; worst gradients " + ", ".join(f"{k} {v:.2e}" for k, v in top))
    assert len(worst) == 68 and set(grads) == set(g_ref)
    assert abs(loss - loss_ref) <= REL * abs(loss_ref), (loss, loss_ref)
    assert abs(last - last_ref) <= REL * abs(last_ref), (last, last_ref)
    bad = {k: v for k, v in worst.items() if v > GRAD_REL}
    assert not bad, bad


def _graphed_step(name, dev):
    """One replay of GraphedTrainStep as measure_training builds it: (loss, last-window MSE, gradients at the initial weights).
    The warm-up iterations are rolled back and Adam does not touch flat_grad, so after the replay it holds the gradient of
    the first iteration."""
    from esr_b200 import train
    from esr_b200.model import DeepRecurrNet
    sd, frames, gt = bench_inputs(name)
    net = DeepRecurrNet(inch=2, basech=8, num_frame=3)
    net.load_state_dict(sd)
    net = net.to(dev)
    opt = train.Adam(net.parameters(), lr=1e-3, weight_decay=1e-4, amsgrad=True)
    t0 = time.time()
    step = train.GraphedTrainStep(net, opt, tuple(frames.shape), dev)
    assert int(opt.step_dev.item()) == 0
    loss = step(frames.to(dev), gt.to(dev)).item()
    assert int(opt.step_dev.item()) == 1
    out = (loss, opt.log[0].item(), {n: p.grad.detach().cpu().clone() for n, p in net.named_parameters()})
    print(f"[train4x] {name} GraphedTrainStep (capture + one replay): {time.time() - t0:.1f} s, peak GPU memory "
          f"{torch.cuda.max_memory_allocated(dev) / 2**30:.2f} GiB")
    del step, opt, net
    _free()
    return out


@pytestgpu
def test_float64_gpu_reference_equals_host_oracle(dev):
    g = torch.Generator().manual_seed(15)
    frames = torch.poisson(torch.full((1, 5, 2, 32, 48), 0.3), generator=g)
    gt = torch.poisson(torch.full((1, 5, 2, 32, 48), 0.3), generator=g)
    sd = model_ref.seeded_state_dict(16)
    a = oracle_step64(sd, frames, gt, dev)
    b = oracle_step64(sd, frames, gt, "cpu", ckpt=False)
    assert abs(a[0] - b[0]) <= 1e-10 * abs(b[0]) and abs(a[1] - b[1]) <= 1e-10 * abs(b[1])
    worst = max(rel(a[2][k], b[2][k]) for k in sd)
    print(f"[train4x] float64 GPU reference vs host oracle: worst gradient {worst:.1e}")
    assert worst <= 1e-10


@pytestgpu
def test_graphed_train_step_cfg3_vs_fp64(dev, cfg3_ref):
    torch.cuda.reset_peak_memory_stats(dev)
    _compare("cfg3 GraphedTrainStep", *_graphed_step("cfg3", dev), cfg3_ref)


@pytestgpu
def test_deterministic_train_step_cfg3_bitwise_and_vs_fp64(dev, cfg3_ref, monkeypatch):
    """Two eager train_steps under torch.use_deterministic_algorithms(True) from the same state: bitwise equal loss and
    gradients, and within the bars of the graphed step against the same float64 reference."""
    from esr_b200 import train
    from esr_b200.model import DeepRecurrNet
    monkeypatch.setenv("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    sd, frames, gt = bench_inputs("cfg3")
    fd, gd = frames.to(dev), gt.to(dev)
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        runs = []
        for _ in range(2):
            net = DeepRecurrNet(inch=2, basech=8, num_frame=3)
            net.load_state_dict(sd)
            net = net.to(dev)
            opt = train.Adam(net.parameters(), lr=1e-3, weight_decay=1e-4, amsgrad=True)
            loss = train.train_step(net, opt, fd, gd).item()
            runs.append((loss, opt.log[0].item(), {n: p.grad.detach().cpu().clone() for n, p in net.named_parameters()}))
            del net, opt
            _free()
    finally:
        torch.use_deterministic_algorithms(prev)
    assert runs[0][0] == runs[1][0] and runs[0][1] == runs[1][1]
    assert all(torch.equal(runs[0][2][k], runs[1][2][k]) for k in runs[0][2])
    _compare("cfg3 deterministic train_step", *runs[0], cfg3_ref)


@pytestgpu
def test_graphed_train_step_cfg4_vs_fp64(dev):
    torch.cuda.reset_peak_memory_stats(dev)
    got = _graphed_step("cfg4", dev)
    _compare("cfg4 GraphedTrainStep", *got, _reference("cfg4", dev))
