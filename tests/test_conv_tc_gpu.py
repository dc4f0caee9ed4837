"""GPU: the wgmma implicit-GEMM convolution (through the C ABI) against torch fp32 conv2d on the CPU.
Floating point => tolerance: 1e-4 relative to the output's max magnitude (the 3-pass split-bf16 product carries
~2^-17 relative operand error; the path-level budget from BASELINE.json is 1e-3)."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
TOL = 1e-4


def _rel(got, want):
    return ((got - want).abs().max() / want.abs().max().clamp_min(1e-6)).item()


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda:0")


@pytest.mark.parametrize("H,W,n_img", [(16, 16, 2), (32, 32, 3), (12, 20, 2), (8, 8, 1), (64, 64, 1)])
def test_conv3x3_64_64_relu(dev, H, W, n_img):
    from esr_b200 import layers as L
    g = torch.Generator().manual_seed(H * 100 + W)
    x = torch.randn(n_img, 64, H, W, generator=g)
    w = torch.randn(64, 64, 3, 3, generator=g) / 24
    b = torch.randn(64, generator=g) * 0.1
    want = F.relu(F.conv2d(x, w, b, padding=1))
    xs = L.Split.from_nchw(x.to(dev))
    out = L.Split(n_img, 64, H, W, dev)
    L.conv_tc([xs], L.pack_weight(w.to(dev)), L.pad_bias(b.to(dev), 64), 64, act="relu", out=out)
    got = out.to_nchw().cpu()
    assert _rel(got, want) < TOL, _rel(got, want)
    # the layout conversion itself is (nearly) lossless
    assert _rel(xs.to_nchw().cpu(), x) < 1e-5


def test_concat_sources_with_image_maps_and_post_residual(dev):
    from esr_b200 import layers as L
    g = torch.Generator().manual_seed(7)
    H, W = 16, 24
    fa = torch.randn(5, 64, H, W, generator=g)
    fb = torch.randn(4, 64, H, W, generator=g)
    ia = torch.tensor([0, 0, 3, 4, 2, 1])
    ib = torch.tensor([1, 0, 3, 2, 2, 0])
    ir = torch.tensor([4, 3, 2, 1, 0, 0])
    w = torch.randn(64, 128, 3, 3, generator=g) / 34
    b = torch.randn(64, generator=g) * 0.1
    want = F.relu(F.conv2d(torch.cat([fa[ia], fb[ib]], 1), w, b, padding=1)) + fa[ir]
    out = L.Split(6, 64, H, W, dev)
    sa, sb = L.Split.from_nchw(fa.to(dev)), L.Split.from_nchw(fb.to(dev))
    L.conv_tc([sa, sb], L.pack_weight(w.to(dev)), L.pad_bias(b.to(dev), 64), 64, act="relu", src_img=[ia, ib], n_img=6,
              res=sa, res_mode=2, res_img=ir, out=out)
    assert _rel(out.to_nchw().cpu(), want) < TOL


def test_192_to_192_pre_residual_and_channel_offset(dev):
    from esr_b200 import layers as L
    g = torch.Generator().manual_seed(9)
    H, W, n = 16, 16, 2
    x = torch.randn(n, 192, H, W, generator=g)
    w = torch.randn(192, 192, 3, 3, generator=g) / 42
    b = torch.randn(192, generator=g) * 0.1
    want = F.relu(F.conv2d(x, w, b, padding=1) + x)
    xs = L.Split.from_nchw(x.to(dev))
    out = L.Split(n, 256, H, W, dev)
    L.conv_tc([xs], L.pack_weight(w.to(dev)), L.pad_bias(b.to(dev), 192), 192, act="relu", res=xs, res_mode=1, out=out,
              out_coff=64)
    got = out.to_nchw().cpu()
    assert _rel(got[:, 64:], want) < TOL
    assert got[:, :64].abs().max().item() == 0.0


def test_narrow_outputs_fp32(dev):
    from esr_b200 import layers as L
    g = torch.Generator().manual_seed(11)
    H, W, n = 20, 12, 3
    x = torch.randn(n, 64, H, W, generator=g)
    xs = L.Split.from_nchw(x.to(dev))
    # Cout = 1, sigmoid (pred_map.1 / attens)
    w = torch.randn(1, 64, 3, 3, generator=g) / 24
    b = torch.randn(1, generator=g)
    o32 = torch.zeros(n, H, W, 1, device=dev)
    L.conv_tc([xs], L.pack_weight(w.to(dev)), L.pad_bias(b.to(dev), 1), 1, act="sigmoid", out_f32=o32)
    want = torch.sigmoid(F.conv2d(x, w, b, padding=1))
    assert _rel(o32.permute(0, 3, 1, 2).cpu(), want) < TOL
    # Cout = 216: raw offsets for channels < 144, sigmoid mask above (DCN_sep.conv_offset_mask)
    w = torch.randn(216, 64, 3, 3, generator=g) / 24
    b = torch.randn(216, generator=g)
    o32 = torch.zeros(n, H, W, 216, device=dev)
    L.conv_tc([xs], L.pack_weight(w.to(dev)), L.pad_bias(b.to(dev), 216), 216, act="sigmoid", act_from=144, out_f32=o32)
    raw = F.conv2d(x, w, b, padding=1)
    want = torch.cat([raw[:, :144], torch.sigmoid(raw[:, 144:])], 1)
    assert _rel(o32.permute(0, 3, 1, 2).cpu(), want) < TOL


def test_conv1x1_two_sources(dev):
    from esr_b200 import layers as L
    g = torch.Generator().manual_seed(13)
    H, W, n = 16, 16, 4
    a, c = torch.randn(n, 64, H, W, generator=g), torch.randn(n, 64, H, W, generator=g)
    w = torch.randn(64, 128, 1, 1, generator=g) / 11
    b = torch.randn(64, generator=g) * 0.1
    want = F.relu(F.conv2d(torch.cat([a, c], 1), w, b))
    out = L.Split(n, 64, H, W, dev)
    L.conv_tc([L.Split.from_nchw(a.to(dev)), L.Split.from_nchw(c.to(dev))], L.pack_weight(w.to(dev)),
              L.pad_bias(b.to(dev), 64), 64, ntaps=1, act="relu", out=out)
    assert _rel(out.to_nchw().cpu(), want) < TOL


def test_convgru_step(dev):
    """ConvGRU (models/submodules.py:496-514) as two fused launches."""
    from esr_b200 import layers as L
    g = torch.Generator().manual_seed(17)
    H, W, n = 16, 16, 2
    x, h = torch.randn(n, 64, H, W, generator=g), torch.randn(n, 64, H, W, generator=g) * 0.5
    wu, wr, wo = (torch.randn(64, 128, 3, 3, generator=g) / 34 for _ in range(3))
    bu, br, bo = (torch.randn(64, generator=g) * 0.1 for _ in range(3))
    xh = torch.cat([x, h], 1)
    z = torch.sigmoid(F.conv2d(xh, wu, bu, padding=1))
    r = torch.sigmoid(F.conv2d(xh, wr, br, padding=1))
    o = torch.tanh(F.conv2d(torch.cat([x, h * r], 1), wo, bo, padding=1))
    want = h * (1 - z) + o * z
    xs, hs = L.Split.from_nchw(x.to(dev)), L.Split.from_nchw(h.to(dev))
    rh, hn = L.Split(n, 64, H, W, dev), L.Split(n, 64, H, W, dev)
    zb = torch.zeros(n, H, W, 64, device=dev)
    bias_zr = torch.cat([bu, br]).to(dev)
    L.conv_tc([xs, hs], L.pack_weight(wu.to(dev), wr.to(dev)), bias_zr, 128, epi_mode=1, h_prev=hs, z_buf=zb, out=rh)
    assert _rel(zb.permute(0, 3, 1, 2).cpu(), z) < TOL
    assert _rel(rh.to_nchw().cpu(), h * r) < TOL
    L.conv_tc([xs, rh], L.pack_weight(wo.to(dev)), L.pad_bias(bo.to(dev), 64), 64, epi_mode=2, h_prev=hs, z_buf=zb, out=hn)
    assert _rel(hn.to_nchw().cpu(), want) < TOL
