"""The small-channel and narrow-output convolutions against float64, layer by layer, on every kernel family that runs them.

esr_conv_small (through esr_b200.layers.conv_small) runs one launch of the network's plan on a chosen path:
  mma     k_conv_mma (mma.sync, split bf16 operands: head+enc0, enc1, enc2, atten1/2, recons[1/2], tail)
  ffma    k_conv_direct, the fp32 FFMA twins (ESR_DIRECT_FFMA=1 in the network)
  narrow  k_conv_narrow (the 1x1 spatial-attention kernel)
The reference is float64 on the exact values the kernel reads (the split input's hi + lo, the fp32 weights), with the fused
head, the bilinear x2 and CropSize stated as model_ref.forward computes them.  Every case asserts err <= TOL and
TOL <= err(degraded) / 4, where the degraded kernel is, for mma, the same product without A_lo B_hi (emulated on the kernel's
operands) and, for ffma / narrow, one that reads the input without its lo plane (the head's fp32 input: rounded to bf16).
Outputs are pre-filled with a sentinel: images >= n_img must keep it, and every output element below n_img is written;
the tail's cropped output must be the uncropped output's window, bit for bit.
TOL is about 4x the error measured on an H100 (DESIGN.md 3 lists the measurements).

The training part runs train.conv2d at every narrow (Cin, Cout, stride, act) of the network, at cfg2's training counts and
at ragged sizes, and checks y, dx, dw and db against float64 the same way (degraded: a lost cross term for the mma.sync /
wgmma kernels, bf16-rounded x or g for the fp32 FFMA kernels).  train_branches restates the rule (conv2d_paths of
train_ops.cu) that picks the forward, dx and dw kernels; a CPU test asserts that the cases cover every branch, and a GPU test
profiles the ragged cases and three wide layers, in default and deterministic mode, and asserts that the kernels launched
are exactly the ones train_branches names.  Another asserts that a workspace one byte short of the reported size is refused
before anything is launched.

The last part runs forward_sequence and one training window in subprocesses under the process-wide switches
(ESR_DIRECT_FFMA, ESR_DCN_COLUMNS, ESR_TRAIN_NO_MMA), which are read once per process.
"""
import math
import os
import subprocess
import sys
import textwrap

import pytest
import torch
import torch.nn.functional as F

from oracle import model_ref
from tests.test_tc_fp64_gpu import ACT64, _act_grad, _check_images, bf16_rne, check, emulations, product_terms, rel, split

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# ------------------------------------------------------------------------------------------------------------------
# float64 reference helpers (CPU)
# ------------------------------------------------------------------------------------------------------------------


def crop_size(H, W):
    """CropSize of the network input: ((pad_top, pad_bottom, pad_left, pad_right), (crop_top, crop_left)).  The input is
    zero-padded to multiples of 8 (ceil on top / left), the tail's output is cut back to H x W from (crop_top, crop_left)."""
    Hc, Wc = (H + 7) // 8 * 8, (W + 7) // 8 * 8
    return ((Hc - H + 1) // 2, (Hc - H) // 2, (Wc - W + 1) // 2, (Wc - W) // 2), (Hc // 2 - H // 2, Wc // 2 - W // 2)


def _taps(x, k, stride, pad):
    """[n, C, H, W] -> the k*k shifted (and strided) views of the zero-padded x, tap-major (ky, kx)."""
    H, W = x.shape[-2:]
    xp = F.pad(x, (pad, pad, pad, pad))
    Ho, Wo = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
    return [xp[..., ky:ky + stride * (Ho - 1) + 1:stride, kx:kx + stride * (Wo - 1) + 1:stride]
            for ky in range(k) for kx in range(k)]


def conv64(x, w, b, stride=1):
    """Convolution as a sum over taps of per-pixel channel contractions (what the kernels compute), pad k // 2."""
    k = w.shape[-1]
    taps = _taps(x, k, stride, k // 2)
    out = b.to(x.dtype).view(1, -1, 1, 1).expand(x.shape[0], -1, *taps[0].shape[-2:]).clone()
    for t, xs in enumerate(taps):
        out += torch.einsum("nchw,oc->nohw", xs, w[:, :, t // k, t % k].to(x.dtype))
    return out


def head64(x, wh, bh, pads):
    """The fused head: relu(head conv) on the CropSize-padded frame (zero outside the input image)."""
    pt, pb, pl, pr = pads
    xp = torch.zeros(*x.shape[:2], x.shape[2] + pt + pb, x.shape[3] + pl + pr, dtype=x.dtype)
    xp[..., pt:pt + x.shape[2], pl:pl + x.shape[3]] = x
    return torch.relu(conv64(xp, wh, bh))


def up2_64(x):
    """Bilinear x2, align_corners=False, as ATen states it: src = max(0, (dst + 0.5) / 2 - 0.5), neighbour index clamped,
    h0 * (w0 * v00 + w1 * v01) + h1 * (w0 * v10 + w1 * v11)."""
    H, W = x.shape[-2:]

    def axis(n):
        f = ((torch.arange(2 * n, dtype=torch.float64) + 0.5) * 0.5 - 0.5).clamp_min(0)
        i0 = f.floor().long()
        return i0, (i0 + 1).clamp_max(n - 1), f - i0
    y0, y1, ly = axis(H)
    x0, x1, lx = axis(W)
    ly, lx = ly.view(-1, 1), lx.view(1, -1)
    r0, r1 = x[..., y0, :], x[..., y1, :]
    return (1 - ly) * ((1 - lx) * r0[..., x0] + lx * r0[..., x1]) + ly * ((1 - lx) * r1[..., x0] + lx * r1[..., x1])


# ------------------------------------------------------------------------------------------------------------------
# CPU tests of the helpers
# ------------------------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("H,W", [(90, 160), (37, 45), (33, 31), (64, 64), (12, 30), (1, 7), (15, 9)])
def test_crop_size_is_model_ref_pad_and_crop(H, W, monkeypatch):
    """model_ref.forward's own CropSize: the frame the head sees and the window the tail's output is cut to."""
    pads, (ct, cl) = crop_size(H, W)
    seen = {}
    real_conv = model_ref._conv

    def spy(sd, name, x, **kw):
        if name == "head.conv2d":
            seen["head_in"] = x.clone()
        if name == "tail.conv2d":                    # the padded-frame coordinates in place of the tail's output
            n, _, Hc, Wc = x.shape
            return torch.arange(Hc * Wc, dtype=x.dtype).view(1, 1, Hc, Wc).expand(n, 2, Hc, Wc)
        return real_conv(sd, name, x, **kw)
    monkeypatch.setattr(model_ref, "_conv", spy)
    g = torch.Generator().manual_seed(H * 100 + W)
    inp = torch.rand(1, 3, 2, H, W, generator=g) + 0.5
    out, _ = model_ref.forward(model_ref.seeded_state_dict(1), inp)
    Hc, Wc = H + pads[0] + pads[1], W + pads[2] + pads[3]
    assert Hc % 8 == 0 and Wc % 8 == 0 and Hc - H < 8 and Wc - W < 8
    assert torch.equal(seen["head_in"], F.pad(inp.view(3, 2, H, W), (pads[2], pads[3], pads[0], pads[1])))
    assert out.shape == (1, 2, H, W)
    assert out[0, 0, 0, 0].item() == ct * Wc + cl                                   # the crop window's corner
    assert torch.equal(out[0, 0], torch.arange(Hc * Wc, dtype=out.dtype).view(Hc, Wc)[ct:ct + H, cl:cl + W])


def test_unequal_pads_cover_every_remainder():
    rems = set()
    for H, W in [(37, 45), (33, 31), (90, 163), (12, 30)]:
        (pt, pb, pl, pr), _ = crop_size(H, W)
        rems |= {H % 8, W % 8}
        if H % 2:
            assert pt == pb + 1
        if W % 2:
            assert pl == pr + 1
    assert rems >= set(range(1, 8))


@pytest.mark.parametrize("shape,stride", [((2, 8, 17, 23), 2), ((2, 8, 16, 16), 2), ((1, 16, 9, 14), 1), ((3, 2, 5, 4), 1)])
def test_conv64_is_torch_conv2d(shape, stride):
    g = torch.Generator().manual_seed(sum(shape))
    x = torch.randn(shape, generator=g, dtype=torch.float64)
    w = torch.randn(5, shape[1], 3, 3, generator=g, dtype=torch.float64)
    b = torch.randn(5, generator=g, dtype=torch.float64)
    ref = F.conv2d(x, w, b, stride=stride, padding=1)
    assert (conv64(x, w, b, stride) - ref).abs().max().item() < 1e-12
    w1 = torch.randn(2, shape[1], 1, 1, generator=g, dtype=torch.float64)
    assert (conv64(x, w1, b[:2]) - F.conv2d(x, w1, b[:2])).abs().max().item() < 1e-12


@pytest.mark.parametrize("H,W", [(37, 45), (33, 31), (8, 16), (3, 5)])
def test_fused_head_is_pad_then_conv(H, W):
    g = torch.Generator().manual_seed(H + W)
    x = torch.randn(2, 2, H, W, generator=g, dtype=torch.float64)
    wh = torch.randn(8, 2, 3, 3, generator=g, dtype=torch.float64)
    bh = torch.randn(8, generator=g, dtype=torch.float64)
    pads, _ = crop_size(H, W)
    ref = torch.relu(F.conv2d(F.pad(x, (pads[2], pads[3], pads[0], pads[1])), wh, bh, padding=1))
    assert (head64(x, wh, bh, pads) - ref).abs().max().item() < 1e-12


@pytest.mark.parametrize("shape", [(2, 3, 8, 8), (1, 5, 7, 13), (3, 2, 1, 9), (1, 4, 2, 1)])
def test_up2_is_aten_bilinear(shape):
    x = torch.randn(shape, generator=torch.Generator().manual_seed(sum(shape)), dtype=torch.float64)
    ref = F.interpolate(x, scale_factor=2, mode="bilinear", align_corners=False)
    assert (up2_64(x) - ref).abs().max().item() < 1e-12


# ------------------------------------------------------------------------------------------------------------------
# the layer-level entry: which (kind, path) pairs run
# ------------------------------------------------------------------------------------------------------------------
# kind: (Cin, Cout, k, stride, bilinear x2 first, activation, paths the network runs it on)
LAYERS = {
    "head_enc0": (8, 16, 3, 2, False, "relu", ("mma", "ffma")),
    "enc1": (16, 32, 3, 2, False, "relu", ("mma", "ffma")),
    "enc2": (32, 64, 3, 2, False, "relu", ("mma", "ffma")),
    "att32": (32, 1, 3, 1, False, "sigmoid", ("mma", "ffma")),
    "att16": (16, 1, 3, 1, False, "sigmoid", ("mma", "ffma")),
    "recon1": (32, 16, 3, 1, True, "relu", ("mma", "ffma")),
    "recon2": (16, 8, 3, 1, True, "relu", ("mma", "ffma")),
    "tail": (8, 2, 3, 1, False, "relu", ("mma", "ffma")),
    "spatial_kernel": (64, 2, 1, 1, False, "sigmoid", ("narrow",)),
}


def test_conv_small_refuses_pairs_the_plan_never_runs():
    """esr_conv_small_workspace_bytes is 0 for a (kind, path) the network never runs, and the call refuses it
    (ESR_EUNSUPPORTED) before touching the device."""
    import ctypes
    from esr_b200 import _lib, build
    from esr_b200 import layers as Lyr
    build.build()
    assert set(Lyr.SMALL_KINDS) == set(LAYERS)
    for kind, spec in LAYERS.items():
        for path in Lyr.SMALL_PATHS:
            assert Lyr.conv_small_supported(kind, path) == (path in spec[6]), (kind, path)
            if path not in spec[6]:
                d = _lib.ConvSmallDesc()
                d.kind, d.path = Lyr.SMALL_KINDS[kind], Lyr.SMALL_PATHS[path]
                assert _lib.lib().esr_conv_small(ctypes.byref(d), None) == -4, (kind, path)


# ------------------------------------------------------------------------------------------------------------------
# GPU cases
# ------------------------------------------------------------------------------------------------------------------
# TOL per (path, output): measured max err on one H100 80GB HBM3 x ~4 (DESIGN.md 3 lists the measurements)
TOL = {
    ("mma", "split"): 4.5e-5,     # k_conv_mma, split-bf16 output (the hi + lo storage itself carries ~2^-17 relative)
    ("mma", "f32"): 2e-5,         # k_conv_mma, fp32 output (attention maps, tail)
    ("ffma", "split"): 3e-5,      # k_conv_direct
    ("ffma", "f32"): 1.5e-6,
    ("narrow", "f32"): 1.5e-6,    # k_conv_narrow
}



# id: (kind, n_img, H_in, W_in, extras).  H_in x W_in is the layer's input: the network frame for head_enc0 (padded by
# CropSize), the conv input otherwise (half the output for recon1 / recon2, the padded frame for the tail).
#   extras: in_n (input images; in_img then repeats and permutes), crop (H, W of the network frame: the tail's window),
#           check (images compared with float64)
SMALL_CASES = {
    # cfg2 (B 8, L 8, 256 x 256, N 3): 64 frames, 48 decoder images, features 32 x 32
    "head_enc0_cfg2": ("head_enc0", 64, 256, 256, dict(check=3)),
    "enc1_cfg2": ("enc1", 64, 128, 128, dict(check=4)),
    "enc2_cfg2": ("enc2", 64, 64, 64, dict(check=6)),
    "att32_cfg2": ("att32", 64, 64, 64, dict(check=6)),
    "att16_cfg2": ("att16", 64, 128, 128, dict(check=4)),
    "recon1_cfg2": ("recon1", 48, 64, 64, dict(check=3)),
    "recon2_cfg2": ("recon2", 48, 128, 128, dict(check=2)),
    "tail_cfg2": ("tail", 48, 256, 256, dict(check=3)),
    "spatial_kernel_cfg2": ("spatial_kernel", 96, 32, 32, dict(check=8)),
    # CropSize with unequal pads (H % 8, W % 8 over 1..7), odd stride-2 inputs, tiles straddling the edge
    "head_enc0_37x45": ("head_enc0", 6, 37, 45, dict(in_n=4)),
    "head_enc0_33x31": ("head_enc0", 5, 33, 31, {}),
    "head_enc0_90x163": ("head_enc0", 3, 90, 163, {}),
    "head_enc0_12x30": ("head_enc0", 4, 12, 30, dict(in_n=9)),
    "enc1_37x45": ("enc1", 9, 37, 45, dict(in_n=5)),
    "enc1_5x7": ("enc1", 3, 5, 7, {}),
    "enc2_19x23": ("enc2", 7, 19, 23, dict(in_n=11)),
    "enc2_3x3": ("enc2", 2, 3, 3, {}),
    "att32_19x45": ("att32", 6, 19, 45, dict(in_n=4)),
    "att32_3x5": ("att32", 2, 3, 5, {}),
    "att16_37x21": ("att16", 5, 37, 21, dict(in_n=8)),
    "recon1_10x21": ("recon1", 4, 10, 21, dict(in_n=3)),
    "recon1_3x5": ("recon1", 2, 3, 5, {}),
    "recon2_19x23": ("recon2", 3, 19, 23, {}),
    "tail_37x45": ("tail", 5, 40, 48, dict(crop=(37, 45))),
    "tail_33x31": ("tail", 4, 40, 32, dict(crop=(33, 31))),
    "tail_90x163": ("tail", 2, 96, 168, dict(crop=(90, 163))),
    "tail_5x9": ("tail", 3, 8, 16, dict(crop=(5, 9))),
    "tail_19x27": ("tail", 3, 24, 32, dict(crop=(19, 27))),
    "head_enc0_17x23": ("head_enc0", 3, 17, 23, dict(in_n=2)),
    "enc1_11x13": ("enc1", 5, 11, 13, dict(in_n=3)),
    "enc2_7x9": ("enc2", 3, 7, 9, {}),
    "att32_33x17": ("att32", 4, 33, 17, dict(in_n=6)),
    "att16_5x3": ("att16", 2, 5, 3, {}),
    "recon1_7x11": ("recon1", 3, 7, 11, dict(in_n=5)),
    "recon2_5x9": ("recon2", 2, 5, 9, dict(in_n=4)),
    "spatial_kernel_11x19": ("spatial_kernel", 6, 11, 19, dict(in_n=9)),
    "spatial_kernel_5x7": ("spatial_kernel", 3, 5, 7, {}),
}
PARAMS = [(c, p) for c, v in SMALL_CASES.items() for p in LAYERS[v[0]][6]]
SENTINEL = -3.0


@pytest.fixture(scope="module")
def dev():
    import bench
    torch.set_num_threads(bench.usable_cores())
    return torch.device("cuda:0")


def _in_img(g, n_img, in_n):
    """Output image -> input image: every input at least once where possible, repeated and out of order."""
    idx = torch.cat([torch.randperm(in_n, generator=g), torch.randint(0, in_n, (max(0, n_img - in_n),), generator=g)])
    return idx[torch.randperm(len(idx), generator=g)][:n_img]


@pytest.mark.gpu
@pytest.mark.parametrize("case,path", PARAMS)
def test_small_conv_vs_fp64(dev, case, path):
    from esr_b200 import layers as Lyr
    kind, n_img, H, W, ex = SMALL_CASES[case]
    cin, cout, k, stride, ups, act, _ = LAYERS[kind]
    head = kind == "head_enc0"
    g = torch.Generator().manual_seed(sum(map(ord, case)))
    in_n = ex.get("in_n", n_img)
    in_img = _in_img(g, n_img, in_n) if "in_n" in ex else None
    w = torch.randn(cout, cin, k, k, generator=g) / math.sqrt(cin * k * k)
    b = torch.randn(cout, generator=g) * 0.1
    pads = (0, 0, 0, 0)
    if head:
        pads, _ = crop_size(H, W)
        x = torch.poisson(torch.full((in_n, 2, H, W), 0.5), generator=g) * torch.rand(in_n, 2, H, W, generator=g)
        wh, bh = torch.randn(8, 2, 3, 3, generator=g) / math.sqrt(18), torch.randn(8, generator=g) * 0.1
    else:
        x = torch.randn(in_n, cin, H, W, generator=g)
    Hc, Wc = H + pads[0] + pads[1], W + pads[2] + pads[3]
    Ho, Wo = (2 * Hc, 2 * Wc) if ups else (((Hc - 1) // 2 + 1, (Wc - 1) // 2 + 1) if stride == 2 else (Hc, Wc))

    # ---- the GPU launch, outputs pre-filled with a sentinel and two images more than written
    xin = x.to(dev) if head else Lyr.Split.from_nchw(x.to(dev))
    kw = dict(in_img=in_img, pads=pads)
    if head:
        kw["head"] = (wh.to(dev), bh.to(dev))
    crop = None
    if cout >= 8:
        out = Lyr.Split(n_img + 2, cout, Ho, Wo, dev)
        out.buf.fill_(SENTINEL)
        Lyr.conv_small(kind, path, xin, w.to(dev), b.to(dev), n_img, out=out, **kw)
        assert bool((out.buf[:, n_img:] == SENTINEL).all()), "images >= n_img written"
        assert bool((out.buf[0, :n_img] != SENTINEL).all()), "output not fully written"   # relu: hi >= 0
        got_all = out.to_nchw()[:n_img].cpu()
        out_kind = "split"
    else:
        if kind == "tail":
            ch, cw = ex.get("crop", (Hc, Wc))
            _, crop = crop_size(ch, cw)
            o32 = torch.full((n_img + 2, cout, ch, cw), SENTINEL, device=dev)
            kw["crop"] = crop
        else:
            o32 = torch.full((n_img + 2, Ho, Wo, cout), SENTINEL, device=dev)
        Lyr.conv_small(kind, path, xin, w.to(dev), b.to(dev), n_img, out_f32=o32, **kw)
        assert bool((o32[n_img:] == SENTINEL).all()), "images >= n_img written"
        assert bool((o32[:n_img] != SENTINEL).all()), "output not fully written"
        got_all = (o32 if kind == "tail" else o32.permute(0, 3, 1, 2))[:n_img].cpu()
        out_kind = "f32"
        if crop is not None and (ch, cw) != (Hc, Wc):
            # the crop window and nothing else: the cropped output is the uncropped one's window, bit for bit
            full = torch.full((n_img, cout, Hc, Wc), SENTINEL, device=dev)
            Lyr.conv_small(kind, path, xin, w.to(dev), b.to(dev), n_img, out_f32=full, in_img=in_img, crop=(0, 0))
            assert torch.equal(o32[:n_img], full[..., crop[0]:crop[0] + ch, crop[1]:crop[1] + cw])

    # ---- float64 on what the kernel reads, for a spread of output images
    sel = torch.tensor(_check_images(n_img, ex.get("check", 12)))
    src = sel if in_img is None else in_img[sel]
    b64 = b.double()
    fin = lambda acc: ACT64[act](acc)                                                    # noqa: E731
    if head:
        xs = x[src]
        convin = head64(xs.double(), wh.double(), bh.double(), pads)
        if path == "mma":                                        # the encoder's A operand: the head output, split
            convin_deg_a = convin.float()
        else:                                                    # the head fed bf16-rounded input
            convin_deg = head64(bf16_rne(xs).double(), wh.double(), bh.double(), pads)
    else:
        hi, lo = split(x[src])
        xv, xv_hi = hi.double() + lo.double(), hi.double()
        if ups:
            xv, xv_hi = up2_64(xv), up2_64(xv_hi)
        convin = xv
        if path == "mma":
            convin_deg_a = xv.float()
        else:
            convin_deg = xv_hi
    ref = fin(conv64(convin, w.double(), b64, stride))
    if path == "mma":
        terms = product_terms(lambda a_, w_: conv64(a_, w_, torch.zeros(cout, dtype=torch.float64), stride), convin_deg_a, w)
        deg = fin(emulations(terms)["drop_cross"] + b64.view(1, -1, 1, 1))
        deg_is = "A_lo B_hi dropped"
    else:
        deg = fin(conv64(convin_deg, w.double(), b64, stride))
        deg_is = "input without lo plane" if not head else "input rounded to bf16"
    if crop is not None:
        ch, cw = got_all.shape[-2:]
        ref, deg = (t[..., crop[0]:crop[0] + ch, crop[1]:crop[1] + cw] for t in (ref, deg))
    print(f"[small64] {case} / {path}: {kind} {cin}->{cout} s{stride}{' up2' if ups else ''}, input {H}x{W} "
          f"(pads {pads}), output {tuple(got_all.shape[-2:])}, images checked {len(sel)}/{n_img}")
    check(f"{case}.{path}", f"{path}_{out_kind}", got_all[sel], ref, deg, deg_is, tol=TOL[(path, out_kind)])


# ------------------------------------------------------------------------------------------------------------------
# training: train.conv2d at every narrow layer of the network, on every dispatch branch of esr_conv2d_forward / backward
# ------------------------------------------------------------------------------------------------------------------
# The dispatch rule of train_ops.cu, restated: tc_fwd_ok, tc_dgrad_ok and the (Cin, Cout, stride) instantiations of
# conv_mma_nchw (the MMA_CASE list of mma_conv.cu; a CPU test keeps the two in step).
MMA_CASES = {(2, 8, 1), (32, 16, 1), (16, 8, 1), (8, 2, 1), (32, 1, 1), (16, 1, 1), (16, 32, 1), (8, 16, 1), (1, 32, 1),
             (1, 16, 1), (1, 64, 1), (8, 16, 2), (16, 32, 2), (32, 64, 2)}


def tc_fwd_ok(cin, cout, k, s):
    return s == 1 and cin % 64 == 0 and cout <= 256


def tc_dgrad_ok(cin, cout, k, s):
    return s == 1 and 32 <= cout <= 256 and cin <= 256


def train_branches(cin, cout, k, s, act, no_mma=False):
    """(forward, dx, dw) kernels esr_conv2d_forward / esr_conv2d_backward launch for this layer (no_mma: under
    ESR_TRAIN_NO_MMA)."""
    if tc_fwd_ok(cin, cout, k, s):
        fwd = "k_conv_tc"
    elif k == 3 and (cin, cout, s) in MMA_CASES and act != "tanh" and not no_mma:
        fwd = "k_conv_mma"
    else:
        fwd = "k_conv_fwd_r" if k == 3 and s == 1 else f"k_conv_fwd_g<{k}>"
    tcd = tc_dgrad_ok(cin, cout, k, s)
    if tcd:
        dx = "k_conv_tc"
    elif k == 3 and s == 1:
        dx = "k_conv_mma" if (cout, cin, 1) in MMA_CASES and not no_mma else "k_conv_fwd_r"
    else:
        dx = "k_conv_dgrad_s2" if k == 3 else f"k_conv_dgrad_g<{k}>"
    if tcd and cin % 64 == 0:
        dw = "k_wgrad_tc"
    elif k == 3:
        dw = "k_conv_wgrad_r"
    else:
        dw = f"k_conv_wgrad_g<{k}>"
    return fwd, dx, dw


# id: (Cin, Cout, k, stride, act, B, H, W, the (forward, dx, dw) branches the case covers, extras)
#   extras: check (images compared with float64 for y and dx; dw and db sum over all)
MMA, R, S2 = "k_conv_mma", "k_conv_wgrad_r", "k_conv_dgrad_s2"
TRAIN_NARROW = {
    # cfg2 training counts: B * L = 64 frames at 256 x 256 (encoder, attention maps), 48 decoder images
    "head_2_8_cfg2": (2, 8, 3, 1, "relu", 64, 256, 256, (MMA, MMA, R), dict(check=2)),
    "enc0_8_16_s2_cfg2": (8, 16, 3, 2, "relu", 64, 256, 256, (MMA, S2, R), dict(check=2)),
    "enc1_16_32_s2_cfg2": (16, 32, 3, 2, "relu", 64, 128, 128, (MMA, S2, R), dict(check=3)),
    "enc2_32_64_s2_cfg2": (32, 64, 3, 2, "relu", 64, 64, 64, (MMA, S2, R), dict(check=4)),
    "recon1_32_16_cfg2": (32, 16, 3, 1, "relu", 48, 128, 128, (MMA, MMA, R), dict(check=3)),
    "recon2_16_8_cfg2": (16, 8, 3, 1, "relu", 48, 256, 256, (MMA, MMA, R), dict(check=2)),
    "tail_8_2_cfg2": (8, 2, 3, 1, "relu", 48, 256, 256, (MMA, MMA, R), dict(check=2)),
    "att1_32_1_cfg2": (32, 1, 3, 1, "sigmoid", 64, 64, 64, (MMA, MMA, R), dict(check=4)),
    "att2_16_1_cfg2": (16, 1, 3, 1, "sigmoid", 64, 128, 128, (MMA, MMA, R), dict(check=3)),
    "att0_64_1_cfg2": (64, 1, 3, 1, "sigmoid", 64, 32, 32, ("k_conv_tc", MMA, R), dict(check=6)),
    "kernel_64_2_1x1_cfg2": (64, 2, 1, 1, "sigmoid", 96, 32, 32, ("k_conv_tc", "k_conv_dgrad_g<1>", "k_conv_wgrad_g<1>"),
                             dict(check=6)),
    # ragged sizes: tiles straddling the edge, odd stride-2 inputs, images smaller than a tile
    "head_2_8_37x45": (2, 8, 3, 1, "relu", 3, 37, 45, (MMA, MMA, R), {}),
    "enc0_8_16_s2_33x31": (8, 16, 3, 2, "relu", 3, 33, 31, (MMA, S2, R), {}),
    "enc1_16_32_s2_19x23": (16, 32, 3, 2, "relu", 4, 19, 23, (MMA, S2, R), {}),
    "enc2_32_64_s2_9x13": (32, 64, 3, 2, "relu", 5, 9, 13, (MMA, S2, R), {}),
    "recon1_32_16_21x37": (32, 16, 3, 1, "relu", 3, 21, 37, (MMA, MMA, R), {}),
    "recon2_16_8_19x23": (16, 8, 3, 1, "relu", 4, 19, 23, (MMA, MMA, R), {}),
    "tail_8_2_11x45": (8, 2, 3, 1, "relu", 3, 11, 45, (MMA, MMA, R), {}),
    "att1_32_1_13x7": (32, 1, 3, 1, "sigmoid", 4, 13, 7, (MMA, MMA, R), {}),
    "att2_16_1_5x9": (16, 1, 3, 1, "sigmoid", 3, 5, 9, (MMA, MMA, R), {}),
    "pm1_64_1_13x21": (64, 1, 3, 1, "sigmoid", 5, 13, 21, ("k_conv_tc", MMA, R), {}),
    "kernel_64_2_1x1_11x19": (64, 2, 1, 1, "sigmoid", 4, 11, 19, ("k_conv_tc", "k_conv_dgrad_g<1>", "k_conv_wgrad_g<1>"), {}),
    # the fallbacks: tanh has no mma instantiation (k_conv_fwd_r at stride 1, k_conv_fwd_g<3> at stride 2)
    "recon2_16_8_tanh_19x23": (16, 8, 3, 1, "tanh", 4, 19, 23, ("k_conv_fwd_r", MMA, R), {}),
    "enc0_8_16_s2_tanh_17x21": (8, 16, 3, 2, "tanh", 3, 17, 21, ("k_conv_fwd_g<3>", S2, R), {}),
    # more ragged sizes of the layers whose weight gradient runs on k_conv_wgrad_r
    "head_2_8_17x9": (2, 8, 3, 1, "relu", 2, 17, 9, (MMA, MMA, R), {}),
    "enc1_16_32_s2_21x17": (16, 32, 3, 2, "relu", 3, 21, 17, (MMA, S2, R), {}),
    "recon1_32_16_9x13": (32, 16, 3, 1, "relu", 2, 9, 13, (MMA, MMA, R), {}),
}
# TOL per kernel (y, dx, dw) and for the bias gradient: measured max err on one H100 80GB HBM3 x ~4 (DESIGN.md 3)
TRAIN_TOL = {
    "k_conv_mma": 4e-5,           # forward and stride-1 dx, split products (measured 1.0e-5)
    "k_conv_tc": 2e-5,            # the 64-channel forwards on wgmma (4.8e-6)
    "k_conv_fwd_r": 3e-6,         # fp32 FFMA kernels (7.2e-7)
    "k_conv_fwd_g<3>": 2.5e-6,    # (5.3e-7)
    "k_conv_dgrad_s2": 2e-6,      # (4.3e-7)
    "k_conv_dgrad_g<1>": 7e-7,    # (1.6e-7)
    "k_conv_wgrad_r": 1e-5,       # (2.4e-6)
    "k_conv_wgrad_g<1>": 7e-6,    # (1.8e-6)
    "db": 2e-6,                   # fp32 sums, no product term (5.1e-7)
}
BRANCHES = {"k_conv_mma", "k_conv_fwd_r", "k_conv_dgrad_s2", "k_conv_dgrad_g<1>", "k_conv_wgrad_g<1>", "k_conv_wgrad_r"}
NARROW_LAYERS = {(2, 8, 3, 1), (8, 16, 3, 2), (16, 32, 3, 2), (32, 64, 3, 2), (32, 16, 3, 1), (16, 8, 3, 1), (8, 2, 3, 1),
                 (32, 1, 3, 1), (16, 1, 3, 1), (64, 1, 3, 1), (64, 2, 1, 1)}


def test_train_cases_cover_every_layer_and_branch():
    import re
    src = open(os.path.join(ROOT, "esr_b200", "csrc", "mma_conv.cu")).read()
    listed = {tuple(int(v) for v in m) for m in re.findall(r"MMA_CASE\((\d+), (\d+), (\d+), \d+, \d+\)", src)}
    assert listed == MMA_CASES                                          # the restated rule follows conv_mma_nchw
    covered = set()
    for name, (cin, cout, k, s, act, B, H, W, claims, ex) in TRAIN_NARROW.items():
        assert train_branches(cin, cout, k, s, act) == claims, name
        covered |= set(claims)
    assert covered >= BRANCHES
    assert {c[:4] for c in TRAIN_NARROW.values()} == NARROW_LAYERS
    for lay in NARROW_LAYERS:                                           # each layer at cfg2's counts and at a ragged size
        assert any(c[:4] == lay and c[5] >= 48 for c in TRAIN_NARROW.values()), lay
        assert any(c[:4] == lay and c[5] < 12 and (c[6] % 16 or c[7] % 16) for c in TRAIN_NARROW.values()), lay


def _wgrad64s(x, g, k, stride, chunk=4):
    """dw[co, ci, ky, kx] = sum over images and output pixels of g * the strided, shifted x, in float64."""
    co, ci = g.shape[1], x.shape[1]
    dw = torch.zeros(co, ci * k * k, dtype=torch.float64)
    for i in range(0, x.shape[0], chunk):
        cols = F.unfold(x[i:i + chunk].double(), k, padding=k // 2, stride=stride)     # [n, ci*k*k, Ho*Wo]
        dw += torch.einsum("npl,nql->pq", g[i:i + chunk].double().flatten(2), cols)
    return dw.view(co, ci, k, k)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(TRAIN_NARROW))
def test_train_narrow_conv2d_vs_fp64(dev, name):
    from esr_b200 import train
    cin, cout, k, stride, act, B, H, W, (k_fwd, k_dx, k_dw), ex = TRAIN_NARROW[name]
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    x = torch.randn(B, cin, H, W, generator=g)
    w = torch.randn(cout, cin, k, k, generator=g) / math.sqrt(cin * k * k)
    b = torch.randn(cout, generator=g) * 0.1
    pad = k // 2
    Ho, Wo = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
    dy = torch.randn(B, cout, Ho, Wo, generator=g)
    xg, wg, bg = (t.to(dev).requires_grad_() for t in (x, w, b))
    y = train.conv2d(xg, wg, bg, stride, act)
    y.backward(dy.to(dev))
    y_got, dx_got, dw_got, db_got = y.detach().cpu(), xg.grad.cpu(), wg.grad.cpu(), bg.grad.cpu()

    sel = torch.tensor(_check_images(B, ex.get("check", 12)))
    conv = lambda a, bb: F.conv2d(a, bb, stride=stride, padding=pad)                   # noqa: E731
    dxop = lambda gg, bb: torch.nn.grad.conv2d_input((len(sel), cin, H, W), bb, gg, stride=stride, padding=pad)  # noqa: E731
    b64 = b.double().view(1, -1, 1, 1)
    xs = x[sel]
    y64 = ACT64[act](conv(xs.double(), w.double()) + b64)
    # the backward on the y it is handed (the forward's output), as the kernels see it: g = dy * act'(y) in fp32
    g64 = dy.double() * _act_grad(y_got.double(), act)
    g32 = dy * _act_grad(y_got, act)
    dx64 = dxop(g64[sel], w.double())
    dw64 = _wgrad64s(x, g64, k, stride)
    # degraded kernels: a lost A_lo B_hi cross term for the split products (k_conv_mma: A = x / g, k_conv_tc likewise),
    # bf16-rounded x / g for the fp32 FFMA kernels
    if k_fwd in ("k_conv_mma", "k_conv_tc"):
        y_deg, y_is = ACT64[act](emulations(product_terms(conv, xs, w))["drop_cross"] + b64), "A_lo B_hi dropped"
    else:
        y_deg, y_is = ACT64[act](conv(bf16_rne(xs).double(), w.double()) + b64), "x rounded to bf16"
    if k_dx == "k_conv_mma":
        dx_deg, dx_is = emulations(product_terms(dxop, g32[sel], w))["drop_cross"], "A_lo B_hi dropped"
    else:
        dx_deg, dx_is = dxop(bf16_rne(g32[sel]).double(), w.double()), "g rounded to bf16"
    dw_deg, dw_is = _wgrad64s(bf16_rne(x), g64, k, stride), "x rounded to bf16"
    print(f"[train64] {name}: {cin}->{cout} k{k} s{stride} {act}, {B} x {H}x{W}: forward {k_fwd}, dx {k_dx}, dw {k_dw}, "
          f"images checked for y / dx {len(sel)}/{B}")
    check(f"{name}.y", k_fwd, y_got[sel], y64, y_deg, y_is, tol=TRAIN_TOL[k_fwd])
    check(f"{name}.dx", k_dx, dx_got[sel], dx64, dx_deg, dx_is, tol=TRAIN_TOL[k_dx])
    check(f"{name}.dw", k_dw, dw_got, dw64, dw_deg, dw_is, tol=TRAIN_TOL[k_dw])
    check(f"{name}.db", "db", db_got, g64.sum((0, 2, 3)), None, tol=TRAIN_TOL["db"])


# ------------------------------------------------------------------------------------------------------------------
# the kernels train_branches names are the ones that run
# ------------------------------------------------------------------------------------------------------------------
CONV_KERNELS = {"k_conv_tc", "k_conv_mma", "k_conv_fwd_r", "k_conv_fwd_g", "k_conv_dgrad_s2", "k_conv_dgrad_g", "k_wgrad_tc",
                "k_wgrad_tc_det", "k_conv_wgrad_r", "k_conv_wgrad_r_det", "k_conv_wgrad_g", "k_conv_wgrad_g_det", "k_sum_slices"}
# the ragged cases of TRAIN_NARROW, and small-count versions of three tensor-core layers of test_train_4x_fp64_gpu.CONV4
# (offset_mask: g padded from 216 to 256 channels): (Cin, Cout, k, stride, act, B, H, W)
LAUNCH_CASES = {
    **{n: c[:8] for n, c in TRAIN_NARROW.items() if not n.endswith("_cfg2")},
    "gru_zr_128_128": (128, 128, 3, 1, "sigmoid", 2, 19, 23),
    "offset_mask_64_216": (64, 216, 3, 1, None, 2, 13, 21),
    "global_fusion_128_64_1x1": (128, 64, 1, 1, "relu", 2, 11, 19),
}


def _conv_kernel(name):
    """Profiler kernel name (demangled or not) -> its name in train_branches, None for kernels outside CONV_KERNELS."""
    import re
    m = re.search(r"(?:^|[^a-z_])(k_[a-z0-9_]+)(?:<(\d+)|ILi(\d+)E)?", name)
    if not m or m.group(1) not in CONV_KERNELS:
        return None
    return f"{m.group(1)}<{m.group(2) or m.group(3)}>" if m.group(1).endswith(("_g", "_g_det")) else m.group(1)


def expected_kernels(cin, cout, k, s, act, det, no_mma=False):
    """[forward, backward]: the sorted convolution kernels of one train.conv2d forward and of its backward.  Deterministic
    mode: dw on its _det kernel, then k_sum_slices (which also sums the bias partials)."""
    fwd, dx, dw = train_branches(cin, cout, k, s, act, no_mma)
    if det:
        dw = dw.replace("<", "_det<") if "<" in dw else dw + "_det"
    return [[fwd], sorted({dx, dw} | ({"k_sum_slices"} if det else set()))]


def profiled_conv_kernels(cin, cout, k, s, act, B, H, W, det):
    """Runs train.conv2d forward, then backward (dx, dw, db) under torch.profiler (CUDA activity), after one unprofiled run:
    their kernels as expected_kernels lists them.  A spin kernel between the two marks where the backward starts."""
    from torch.profiler import ProfilerActivity, profile
    from esr_b200 import train
    g = torch.Generator().manual_seed(B * H * W + cin)
    x = torch.randn(B, cin, H, W, generator=g).cuda().requires_grad_()
    w = (torch.randn(cout, cin, k, k, generator=g) / math.sqrt(cin * k * k)).cuda().requires_grad_()
    b = (torch.randn(cout, generator=g) * 0.1).cuda().requires_grad_()
    Ho, Wo = (H + 2 * (k // 2) - k) // s + 1, (W + 2 * (k // 2) - k) // s + 1
    dy = torch.randn(B, cout, Ho, Wo, generator=g).cuda()
    prev = torch.backends.cudnn.deterministic
    torch.backends.cudnn.deterministic = det
    try:
        train.conv2d(x, w, b, s, act).backward(dy)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            y = train.conv2d(x, w, b, s, act)
            torch.cuda._sleep(1000)
            y.backward(dy)
            torch.cuda.synchronize()
    finally:
        torch.backends.cudnn.deterministic = prev
    names = [e.name for e in sorted(prof.events(), key=lambda e: e.time_range.start)
             if e.device_type == torch.autograd.DeviceType.CUDA]
    cut = [i for i, n in enumerate(names) if "spin_kernel" in n]
    assert len(cut) == 1, names
    return [sorted({_conv_kernel(n) for n in part} - {None}) for part in (names[:cut[0]], names[cut[0] + 1:])]


@pytest.mark.gpu
@pytest.mark.parametrize("det", [False, True], ids=["default", "deterministic"])
@pytest.mark.parametrize("name", list(LAUNCH_CASES))
def test_train_launches_the_claimed_kernels(dev, name, det):
    cin, cout, k, s, act, B, H, W = LAUNCH_CASES[name]
    got = profiled_conv_kernels(cin, cout, k, s, act, B, H, W, det)
    print(f"[launch] {name} {'deterministic' if det else 'default'}: forward {got[0]}, backward {got[1]}")
    want = expected_kernels(cin, cout, k, s, act, det)
    assert got == want, (name, got, want)


_LAUNCHES = """
    import sys, torch
    from tests.test_small_conv_fp64_gpu import LAUNCH_CASES, profiled_conv_kernels
    torch.save(profiled_conv_kernels(*LAUNCH_CASES["{name}"], det=False), sys.argv[1])
"""


@pytest.mark.gpu
def test_train_no_mma_launches_the_claimed_kernels(tmp_path):
    """Under ESR_TRAIN_NO_MMA the stride-1 dx of a narrow layer runs k_conv_fwd_r on rotated weights: the one row of the
    rule that default mode does not reach at the network's shapes."""
    name = "recon1_32_16_21x37"
    got = _run(_LAUNCHES.format(name=name), tmp_path / "launches.pt", ("ESR_TRAIN_NO_MMA",))
    want = expected_kernels(*LAUNCH_CASES[name][:5], det=False, no_mma=True)
    print(f"[launch] {name} ESR_TRAIN_NO_MMA: forward {got[0]}, backward {got[1]}")
    assert "k_conv_fwd_r" in want[1] and got == want


@pytest.mark.gpu
@pytest.mark.parametrize("layer", ["tc_64_64", "mma_head_2_8"])
def test_short_workspace_is_refused(dev, layer):
    """esr_conv2d_forward and esr_conv2d_backward_ex (default and deterministic) with one byte less workspace than
    esr_conv2d_workspace_bytes_ex reports, and the mma layer's forward with less than its weight image: each call returns
    an error and launches nothing, and the outputs keep their sentinel.  With the reported size the same calls run."""
    from esr_b200 import _lib
    L, ptr = _lib.lib(), _lib.ptr
    cin, cout, k, s, act = {"tc_64_64": (64, 64, 3, 1, 1), "mma_head_2_8": (2, 8, 3, 1, 1)}[layer]
    B, H, W = 2, 13, 21
    g = torch.Generator(device=dev).manual_seed(7)
    x, w, b = torch.randn(B, cin, H, W, generator=g, device=dev), torch.randn(cout, cin, k, k, generator=g, device=dev), \
        torch.randn(cout, generator=g, device=dev)
    y_in, dy = torch.rand(B, cout, H, W, generator=g, device=dev), torch.randn(B, cout, H, W, generator=g, device=dev)
    y, dx, dw, db = (torch.full(t.shape, SENTINEL, device=dev) for t in (y_in, x, w, b))

    def forward(ws, n):
        return L.esr_conv2d_forward(ptr(x), ptr(w), ptr(b), B, cin, H, W, cout, k, s, act, ptr(y), None, ptr(ws), n,
                                    _lib.stream_ptr())

    def backward(ws, n, flags):
        return L.esr_conv2d_backward_ex(ptr(x), None, ptr(w), ptr(y_in), ptr(dy), B, cin, H, W, cout, k, s, act, ptr(dx), ptr(dw),
                                        ptr(db), flags, ptr(ws), n, _lib.stream_ptr())
    calls = []
    for flags in (0, _lib.DETERMINISTIC):
        n = L.esr_conv2d_workspace_bytes_ex(B, cin, H, W, cout, k, s, flags)
        ws = torch.empty((n,), dtype=torch.uint8, device=dev)
        calls.append((f"backward flags={flags}", lambda ws=ws, n=n, f=flags: backward(ws, n - 1, f), lambda ws=ws, n=n, f=flags: backward(ws, n, f)))
        if flags == 0:
            calls.append(("forward", lambda ws=ws, n=n: forward(ws, n - 1), lambda ws=ws, n=n: forward(ws, n)))
            if layer == "mma_head_2_8":                    # below the mma weight image (2 x 9 x 8 x 16 bf16 = 4.5 KiB)
                calls.append(("forward, 256 bytes", lambda ws=ws: forward(ws, 256), None))
    for what, short, _ in calls:
        torch.cuda.synchronize()
        before = L.esr_launch_count()
        rc = short()
        torch.cuda.synchronize()
        assert rc != 0, what
        assert L.esr_launch_count() == before, what
        assert "workspace" in L.esr_last_error().decode(), what
    for t in (y, dx, dw, db):
        assert bool((t == SENTINEL).all())
    for what, _, full in calls:                           # the reported size is enough
        if full is not None:
            before = L.esr_launch_count()
            assert full() == 0, what
            assert L.esr_launch_count() > before, what
    torch.cuda.synchronize()
    assert not bool((y == SENTINEL).any()) and not bool((dw == SENTINEL).any())


# ------------------------------------------------------------------------------------------------------------------
# the process-wide switches, end to end, in subprocesses
# ------------------------------------------------------------------------------------------------------------------
REL = 1e-3
# id: (switches set to 1, num_frame, max-norm relative distance of the switched plan from the default plan: about 4x what an
# H100 measured; 0 = bit-identical)
SWITCHED = {
    "ESR_DIRECT_FFMA": (("ESR_DIRECT_FFMA",), 3, 2e-4),                              # measured 5.3e-5
    "ESR_DCN_COLUMNS": (("ESR_DCN_COLUMNS",), 3, 0.0),
    "ESR_DIRECT_FFMA+ESR_DCN_COLUMNS": (("ESR_DIRECT_FFMA", "ESR_DCN_COLUMNS"), 3, 2e-4),   # 5.3e-5
    "ESR_DIRECT_FFMA-N5": (("ESR_DIRECT_FFMA",), 5, 2e-4),                           # 4.8e-5
    "ESR_DCN_COLUMNS-N5": (("ESR_DCN_COLUMNS",), 5, 0.0),
}
_SWITCHES = ("ESR_DIRECT_FFMA", "ESR_DCN_COLUMNS", "ESR_TRAIN_NO_MMA")
B_, H_, W_ = 2, 37, 45


def _run(code, out, switches=()):
    env = {k: v for k, v in os.environ.items() if k not in _SWITCHES}
    env["PYTHONPATH"] = ROOT
    for sw in switches:
        env[sw] = "1"
    r = subprocess.run([sys.executable, "-c", textwrap.dedent(code), str(out)], capture_output=True, text=True, timeout=900,
                       cwd=ROOT, env=env)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    return torch.load(out)


_FORWARD = """
    import sys, torch
    from oracle import model_ref
    from esr_b200.model import DeepRecurrNet
    N = {N}
    g = torch.Generator().manual_seed(41)
    frames = torch.poisson(torch.full(({B}, N + 2, 2, {H}, {W}), 0.3), generator=g).cuda()
    net = DeepRecurrNet(inch=2, basech=8, num_frame=N)
    net.load_state_dict(model_ref.seeded_state_dict(12, num_frame=N))
    net = net.cuda().eval()
    with torch.no_grad():
        out = torch.cat([net.forward_sequence(frames) for _ in range(2)]).cpu()      # second call: carried state
    torch.save(out, sys.argv[1])
"""


@pytest.fixture(scope="module")
def default_plans(tmp_path_factory):
    """num_frame -> (directory, the default plan's output, the oracle's), computed on first use."""
    d, plans = tmp_path_factory.mktemp("switches"), {}

    def get(N):
        if N not in plans:
            out = _run(_FORWARD.format(N=N, B=B_, H=H_, W=W_), d / f"default_n{N}.pt")
            ora = model_ref.OracleNet(model_ref.seeded_state_dict(12, num_frame=N))
            g = torch.Generator().manual_seed(41)
            frames = torch.poisson(torch.full((B_, N + 2, 2, H_, W_), 0.3), generator=g)
            with torch.no_grad():
                want = torch.cat([ora(frames[:, w:w + N].contiguous()) for _ in range(2) for w in range(3)])
            plans[N] = (d, out, want)
        return plans[N]
    return get


@pytest.mark.gpu
@pytest.mark.parametrize("switch", list(SWITCHED))
def test_switched_plan_vs_oracle_and_default(default_plans, switch):
    switches, N, tol = SWITCHED[switch]
    d, base, want = default_plans(N)
    assert rel(base, want) <= REL, rel(base, want)
    got = _run(_FORWARD.format(N=N, B=B_, H=H_, W=W_), d / f"{switch}.pt", switches)
    e_ora, e_def = rel(got, want), rel(got, base)
    print(f"[switch] {switch}: vs oracle {e_ora:.2e} (default {rel(base, want):.2e}), vs default {e_def:.2e}, TOL {tol:.1e}")
    assert e_ora <= REL, e_ora
    if tol == 0.0:
        assert torch.equal(got, base)
    else:
        assert 0.0 < e_def <= tol, e_def                                   # the switch did change the kernels


_TRAIN = """
    import sys, torch
    from oracle import model_ref
    from esr_b200 import train
    from esr_b200.model import DeepRecurrNet
    g = torch.Generator().manual_seed(35)
    frames = torch.poisson(torch.full((2, 5, 2, 24, 40), 0.3), generator=g)
    gt = torch.poisson(torch.full((2, 5, 2, 24, 40), 0.3), generator=g)
    net = DeepRecurrNet(inch=2, basech=8, num_frame=3)
    net.load_state_dict(model_ref.seeded_state_dict(36))
    net = net.cuda()
    net.reset_states()
    fd, gd = frames.cuda(), gt.cuda()
    loss = 0
    for w in range(3):
        loss = loss + train.mse_loss(net(fd[:, w:w + 3]), gd[:, w + 1])
    loss.backward()
    torch.save(dict(loss=loss.item(), frames=frames, gt=gt, grads={n: p.grad.cpu() for n, p in net.named_parameters()}),
               sys.argv[1])
"""


@pytest.mark.gpu
def test_train_no_mma_window_vs_oracle_autograd(tmp_path):
    """ESR_TRAIN_NO_MMA=1 (the narrow training convolutions on the FFMA kernels): three windows' loss and all parameter
    gradients vs autograd through the oracle, on the inputs and with the bars of
    test_train_gpu.test_sequence_gradients_vs_oracle_autograd (B 2, L 5, 24 x 40); the default plan runs beside it."""
    base = _run(_TRAIN, tmp_path / "default.pt")
    r = _run(_TRAIN, tmp_path / "no_mma.pt", ("ESR_TRAIN_NO_MMA",))
    ref = {k: v.clone().requires_grad_() for k, v in model_ref.seeded_state_dict(36).items()}
    states, loss_ref = None, 0
    for w in range(3):
        pred, states = model_ref.forward(ref, r["frames"][:, w:w + 3], states)
        loss_ref = loss_ref + F.mse_loss(pred, r["gt"][:, w + 1])
    loss_ref.backward()
    worst = {n: rel(gd, ref[n].grad) for n, gd in r["grads"].items()}
    worst_base = {n: rel(gd, ref[n].grad) for n, gd in base["grads"].items()}
    print(f"[switch] ESR_TRAIN_NO_MMA: loss {r['loss']:.6e} (default {base['loss']:.6e}, oracle {loss_ref.item():.6e}), "
          f"worst gradient {max(worst.values()):.2e} (default {max(worst_base.values()):.2e})")
    assert abs(r["loss"] - loss_ref.item()) <= REL * abs(loss_ref.item())
    assert len(worst) == len(ref)
    assert any(not torch.equal(r["grads"][n], base["grads"][n]) for n in ref)          # the switch did change the kernels
    bad = {k: v for k, v in worst.items() if v > 3 * REL}
    assert not bad, bad
