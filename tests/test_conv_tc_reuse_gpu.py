"""k_conv_tc with one A box per (64-channel chunk, dx) shared by the three dy taps, and separate A / B rings, against float64.

The kernel loads a TW x (TH + 2) box per (chunk, dx) and reads its three dy taps at row offsets 0, TW and 2 TW; a 1x1 layer
loads the tile itself.  K-blocks run in the order (chunk, dx, dy).  The A ring holds one box per slot and the B ring one tap's
weights per slot; both carry their positions across tiles.  The cases below pin the regimes that layout creates: each ring
wrapping across tiles (K-blocks per tile not a multiple of either depth), a K loop shorter than the ring, halo boxes that
start above the image and end below it (H < TH, W < 8), image maps, the stepped (dense_fusion.0) source, both GRU
epilogues and the benchmark's layer shapes.  Norm, emulation and tolerances are those of test_tc_fp64_gpu.py.
"""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

STG_BYTES = (63 * 68 + 64) * 4          # one warpgroup's epilogue staging tile (TC_STG_BYTES)


def smem_bytes(npad, a_box, na, nb):
    return 1024 + na * (a_box + 16) + nb * (2 * npad * 128 + 16) + 2 * STG_BYTES


def rings(npad, a_box, taps, cap):
    """Ring depths (A boxes, B slots), by the rule of tc_rings (tc_conv.cu)."""
    na, nb = 2, 2
    if smem_bytes(npad, a_box, na, nb) > cap:
        na = 1
    assert smem_bytes(npad, a_box, na, nb) <= cap
    while True:
        a_can = na < 4 and smem_bytes(npad, a_box, na + 1, nb) <= cap
        b_can = nb < 9 and smem_bytes(npad, a_box, na, nb + 1) <= cap
        if a_can and (not b_can or (na - 1) * taps < nb - 1):
            na += 1
        elif b_can:
            nb += 1
        else:
            return na, nb


def conv_geometry(n_img, H, W, cin_total, ntaps, cout):
    """Launch geometry of k_conv_tc, by the rule of conv_tc_prepare / launch_np (tc_conv.cu): one CTA per SM."""
    p = torch.cuda.get_device_properties(0)
    sm, cap = p.multi_processor_count, getattr(p, "shared_memory_per_block_optin", 232448)
    TW = 16 if W >= 12 else 8
    TH = 128 // TW
    taps = 3 if ntaps == 9 else 1
    a_box = 2 * 128 * TW * (TH + 2 if ntaps == 9 else TH)
    npad = (cout + 15) // 16 * 16
    nkb = cin_total // 64 * ntaps
    na, nb = rings(npad, a_box, taps, cap)
    n_tiles = n_img * math.ceil(W / TW) * math.ceil(H / TH)
    return dict(n_tiles=n_tiles, grid=min(n_tiles, sm), na=na, nb=nb, nkb=nkb, nbox=nkb // taps, npad=npad, TW=TW, TH=TH)


def assert_regime(geo, regime):
    if "multi" in regime:                                   # >= 3 tiles per CTA, tile count not a multiple of the grid
        assert geo["n_tiles"] >= 3 * geo["grid"] and geo["n_tiles"] % geo["grid"] != 0, geo
    if "wraps" in regime:                                   # both ring positions move between tiles
        assert geo["nkb"] % geo["nb"] != 0 and geo["nbox"] % geo["na"] != 0, geo
    if "one" in regime:                                     # a single A box: each box's last tap drains the MMAs
        assert geo["na"] == 1, geo
    if "short" in regime:                                   # a tile's K loop is shorter than either ring
        assert geo["nkb"] < geo["nb"] and geo["nbox"] < geo["na"], geo
    if "H<TH" in regime:
        assert geo["H"] < geo["TH"], geo
    if "W<8" in regime:
        assert geo["W"] < 8, geo


@pytest.fixture(scope="module")
def dev():
    import bench
    torch.set_num_threads(bench.usable_cores())
    return torch.device("cuda:0")


# id: (n_img, H, W, source channels, source images (None = n_img, identity map), ntaps, cout, regime, extras)
CASES = {
    "wraps_np64_cin192": (60, 32, 32, [192], None, 9, 64, "multi wraps", dict(act="relu")),
    "np128_3src_maps": (60, 32, 32, [64, 64, 64], [40, 40, 40], 9, 128, "multi", dict(act="relu")),
    "wraps_np128_1x1": (60, 32, 32, [64, 256], [40, 60], 1, 128, "multi wraps", dict(act="relu")),
    "wraps_np192_res_pre": (60, 32, 32, [192], None, 9, 192, "multi wraps", dict(act="relu", res="self", res_mode=1)),
    "one_a_box_np256": (60, 32, 32, [192], None, 9, 256, "multi one", dict(act="relu")),
    "wraps_np48_1x1": (60, 32, 32, [192], None, 1, 48, "multi", dict(out="f32")),
    "short_1x1": (60, 32, 32, [64], None, 1, 64, "multi short", dict(act="relu")),
    "ragged_H5_W6": (400, 5, 6, [64], None, 9, 64, "multi H<TH W<8", dict(act="relu")),
    "ragged_H7_W20": (200, 7, 20, [64, 64], [150, 200], 9, 128, "multi H<TH", dict(act="sigmoid")),
    "ragged_H3_W45": (200, 3, 45, [64], None, 9, 96, "multi H<TH", dict(act="relu")),
    # the benchmark's layers at feature resolution: cfg2 (32 x 32, 144 images), cfg3 (64 x 64), cfg4 (128 x 128, 84 images)
    "cfg2_192_192_res_pre": (144, 32, 32, [192], None, 9, 192, "multi", dict(act="relu", res="self", res_mode=1)),
    "cfg2_128_64": (144, 32, 32, [128], None, 9, 64, "multi", dict(act="relu")),
    "cfg2_64_216": (144, 32, 32, [64], None, 9, 216, "multi", dict(act="sigmoid", act_from=144, out="f32")),
    "cfg3_192_64": (72, 64, 64, [192], None, 9, 64, "multi", dict(act="relu", check=4)),
    "cfg4_192_192_res_pre": (84, 128, 128, [192], None, 9, 192, "multi", dict(act="relu", res="self", res_mode=1, check=3)),
    "cfg4_128_64": (84, 128, 128, [128], None, 9, 64, "multi", dict(act="relu", check=3)),
    "cfg4_64_216": (84, 128, 128, [64], None, 9, 216, "multi", dict(act="sigmoid", act_from=144, out="f32", check=3)),
}


@pytest.mark.parametrize("name", list(CASES))
def test_conv_tc_reuse_vs_fp64(dev, name):
    from esr_b200 import layers as L
    from tests.test_tc_fp64_gpu import _check_images, _epilogue, _rand, check, emulations, product_terms
    n_img, H, W, chans, src_n, ntaps, cout, regime, ex = CASES[name]
    act, act_from, res_mode = ex.get("act"), ex.get("act_from", 0), ex.get("res_mode", 0)
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    k = 3 if ntaps == 9 else 1
    cin = sum(chans)
    geo = conv_geometry(n_img, H, W, cin, ntaps, cout)
    assert_regime(dict(geo, H=H, W=W), regime)
    src_n = src_n or [n_img] * len(chans)
    srcs = [_rand(g, n, c, H, W) for n, c in zip(src_n, chans)]
    maps = [None if n == n_img else torch.randint(0, n, (n_img,), generator=g) for n in src_n]
    w = _rand(g, cout, cin, k, k, scale=1.0 / math.sqrt(cin * ntaps))
    b = _rand(g, cout, scale=0.1)
    s_dev = [L.Split.from_nchw(t.to(dev)) for t in srcs]
    res_dev = s_dev[0] if ex.get("res") == "self" else None
    out, o32 = None, None
    if ex.get("out", "split") == "split":
        out = L.Split(n_img, cout, H, W, dev)
    else:
        o32 = torch.full((n_img, H, W, cout), -777.0, device=dev)
    L.conv_tc(s_dev, L.pack_weight(w.to(dev)), L.pad_bias(b.to(dev), cout), cout, ntaps=ntaps, act=act, act_from=act_from,
              src_img=maps, n_img=n_img, res=res_dev, res_mode=res_mode, out=out, out_f32=o32)
    got = out.to_nchw().cpu() if out is not None else o32.permute(0, 3, 1, 2).cpu()

    sel = torch.tensor(_check_images(n_img, ex.get("check", 12)))
    xcat = torch.cat([s[sel if m is None else m[sel]] for s, m in zip(srcs, maps)], 1)
    res64 = srcs[0][sel].double() if res_dev is not None else None
    conv = lambda a, bb: F.conv2d(a, bb, padding=k // 2)                 # noqa: E731
    ref = _epilogue(conv(xcat.double(), w.double()), b, act, act_from, res64, res_mode)
    deg = _epilogue(emulations(product_terms(conv, xcat, w))["drop_cross"], b, act, act_from, res64, res_mode)
    print(f"[reuse] {name}: tiles {geo['n_tiles']}, grid {geo['grid']}, rings A {geo['na']} / B {geo['nb']}, "
          f"nkb {geo['nkb']}, npad {geo['npad']}, tile {geo['TW']}x{geo['TH']}")
    check(name, "conv_split" if out is not None else "conv_f32", got[sel], ref, deg)


@pytest.mark.parametrize("n_frame", [3, 5])
def test_dense_fusion0_stepped_source_vs_fp64(dev, n_frame):
    """dense_fusion.0 at num_frame N: a 64-channel source standing for N - 1 chunks (VB images apart, through a permuting
    map) plus the middle frame through a repeating map, one launch; the A ring wraps across tiles."""
    from esr_b200 import layers as L
    from tests.test_tc_fp64_gpu import _check_images, _epilogue, _rand, check, emulations, product_terms
    VB, H, W, cout = 90, 32, 32, 64
    geo = conv_geometry(VB, H, W, 64 * n_frame, 9, cout)
    assert_regime(geo, "multi")
    assert geo["nbox"] % geo["na"] != 0, geo
    g = torch.Generator().manual_seed(n_frame * 313)
    fused = _rand(g, (n_frame - 1) * VB, 64, H, W)
    mid = _rand(g, 2 * VB, 64, H, W)
    perm = torch.randperm(VB, generator=g)
    mid_map = torch.randint(0, 2 * VB, (VB,), generator=g)
    w = _rand(g, cout, 64 * n_frame, 3, 3, scale=1.0 / math.sqrt(64 * n_frame * 9))
    b = _rand(g, cout, scale=0.1)
    out = L.Split(VB, cout, H, W, dev)
    L.conv_tc([L.Split.from_nchw(fused.to(dev)), L.Split.from_nchw(mid.to(dev))], L.pack_weight(w.to(dev)),
              L.pad_bias(b.to(dev), cout), cout, act="relu", src_img=[perm, mid_map], n_img=VB, out=out,
              src_chunks=[n_frame - 1, 0], chunk_img_step=[VB, 0])
    got = out.to_nchw().cpu()
    sel = torch.tensor(_check_images(VB, 12))
    xcat = torch.cat([fused[perm[sel] + j * VB] for j in range(n_frame - 1)] + [mid[mid_map[sel]]], 1)
    conv = lambda a, bb: F.conv2d(a, bb, padding=1)                      # noqa: E731
    ref = _epilogue(conv(xcat.double(), w.double()), b, "relu", 0, None, 0)
    deg = _epilogue(emulations(product_terms(conv, xcat, w))["drop_cross"], b, "relu", 0, None, 0)
    check(f"dense_fusion0_N{n_frame}", "conv_split", got[sel], ref, deg)


class _View:
    """A split tensor seen from image k0 on, with the plane distance of the whole tensor (net.cu's view of one GRU step)."""

    def __init__(self, s, k0):
        self.buf, self.n_img = s.buf[:, k0:], s.n_img


@pytest.mark.parametrize("n,H,W", [(16, 32, 32), (60, 32, 32), (4, 128, 128)])
def test_gru_epilogues_vs_fp64(dev, n, H, W):
    """EPI_GRU_ZR (N = 128) then EPI_GRU_OUT (N = 64): cfg2's single-wave step, a step of >= 3 tiles per CTA, and cfg4's
    step; h_prev is a view at an image offset of a larger state buffer."""
    from esr_b200 import layers as L
    from tests.test_tc_fp64_gpu import _rand, check, emulations, product_terms
    geo_zr, geo_o = conv_geometry(n, H, W, 128, 9, 128), conv_geometry(n, H, W, 128, 9, 64)
    if n == 60:
        assert_regime(geo_zr, "multi")
        assert_regime(geo_o, "multi")
    g = torch.Generator().manual_seed(n * 7919 + H)
    x, h_all = _rand(g, n, 64, H, W), _rand(g, 3 * n, 64, H, W, scale=0.5)
    k0 = n
    h = h_all[k0:k0 + n]
    wu, wr, wo = (_rand(g, 64, 128, 3, 3, scale=1 / 34) for _ in range(3))
    bu, br, bo = (_rand(g, 64, scale=0.1) for _ in range(3))
    xs, hs = L.Split.from_nchw(x.to(dev)), L.Split.from_nchw(h_all.to(dev))
    hv = _View(hs, k0)
    rh, hn = L.Split(n, 64, H, W, dev), L.Split(n, 64, H, W, dev)
    zb = torch.zeros(n, H, W, 64, device=dev)
    L.conv_tc([xs, hs], L.pack_weight(wu.to(dev), wr.to(dev)), torch.cat([bu, br]).to(dev), 128,
              src_img=[None, torch.arange(n) + k0], n_img=n, epi_mode=1, h_prev=hv, z_buf=zb, out=rh)
    L.conv_tc([xs, rh], L.pack_weight(wo.to(dev)), L.pad_bias(bo.to(dev), 64), 64, n_img=n, epi_mode=2, h_prev=hv, z_buf=zb,
              out=hn)
    z_got, rh_got, hn_got = zb.permute(0, 3, 1, 2).cpu(), rh.to_nchw().cpu(), hn.to_nchw().cpu()

    conv = lambda a, bb: F.conv2d(a, bb, padding=1)                      # noqa: E731
    xh = torch.cat([x, h], 1)
    wzr, bzr = torch.cat([wu, wr]), torch.cat([bu, br]).double().view(1, -1, 1, 1)
    acc = conv(xh.double(), wzr.double()) + bzr
    acc_deg = emulations(product_terms(conv, xh, wzr))["drop_cross"] + bzr
    h64 = h.double()
    check(f"gru_zr_z_{n}x{H}", "gru", z_got, torch.sigmoid(acc[:, :64]), torch.sigmoid(acc_deg[:, :64]))
    check(f"gru_zr_rh_{n}x{H}", "gru", rh_got, h64 * torch.sigmoid(acc[:, 64:]), h64 * torch.sigmoid(acc_deg[:, 64:]))
    xr = torch.cat([x, rh_got], 1)
    z = z_got.double()
    o = torch.tanh(conv(xr.double(), wo.double()) + bo.double().view(1, -1, 1, 1))
    o_deg = torch.tanh(emulations(product_terms(conv, xr, wo))["drop_cross"] + bo.double().view(1, -1, 1, 1))
    check(f"gru_out_{n}x{H}", "gru", hn_got, h64 * (1 - z) + o * z, h64 * (1 - z) + o_deg * z)
