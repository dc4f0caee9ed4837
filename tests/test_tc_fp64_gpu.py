"""The tensor-core kernels against float64, at the tile counts the benchmark runs.

k_conv_tc (through esr_b200.layers.conv_tc), the training operators esr_conv2d_forward / backward (k_conv_tc for y and dx,
k_wgrad_tc for dw; through esr_b200.train.conv2d) and the DCNv2 operator (esr_b200.dcn_v2_ext) are compared with float64
references computed on the CPU, at shapes where every CTA of the persistent kernels walks several tiles.

Norm (the project's): err = max |got - ref64| / max |ref64|.  Every case also evaluates, in float64, what a kernel computes
from the exact operands it sees (activations / packed weights / g = act'(y) dy split into bf16 hi + lo, DESIGN.md 3):
  split       A_hi B_hi + A_hi B_lo + A_lo B_hi           (what a correct kernel does, up to fp32 accumulation)
  degraded a  A_hi B_hi + A_hi B_lo                       (one cross term lost)
  degraded b  A_hi B_hi + A_lo B_hi                       (bf16-only B operand)
and asserts err <= TOL and TOL <= err(degraded a) / 4: the tolerance of the case is tight enough to catch a kernel that
dropped a product term at that shape.  The DCN weight gradient is an fp32 GEMM without split products; its degraded
kernel reads the features without their lo plane.  Bias gradients are plain fp32 sums and only get err <= TOL.
TOL is about 4x the error measured on an H100.
"""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

# ------------------------------------------------------------------------------------------------------------------
# emulation of the split-bf16 product (CPU)
# ------------------------------------------------------------------------------------------------------------------


def bf16_rne(x):
    """fp32 -> the nearest bf16 value (round to nearest, ties to even), returned as fp32.  Bit-level, independent of
    torch's own conversion; what __float2bfloat16_rn / cvt.rn.bf16x2.f32 do for finite inputs."""
    a = x.detach().float().contiguous().cpu().numpy().view(np.uint32).astype(np.uint64)
    r = ((a + 0x7FFF + ((a >> 16) & 1)) & 0xFFFF0000).astype(np.uint32)
    return torch.from_numpy(r.view(np.float32)).reshape(x.shape)


def split(x):
    """fp32 tensor -> (hi, lo) fp32 tensors holding bf16 values: hi = bf16(x), lo = bf16(x - hi) (split_bf16 in common.cuh)."""
    x = x.detach().float().cpu()
    hi = bf16_rne(x)
    return hi, bf16_rne(x - hi)


def product_terms(op, a, b):
    """op: a bilinear function of two float64 tensors.  -> (hh, hl, lh) = op(A_hi, B_hi), op(A_hi, B_lo), op(A_lo, B_hi)."""
    ah, al = (t.double() for t in split(a))
    bh, bl = (t.double() for t in split(b))
    return op(ah, bh), op(ah, bl), op(al, bh)


def emulations(terms):
    """-> dict of the three emulated products (float64)."""
    hh, hl, lh = terms
    return {"split": hh + hl + lh, "drop_cross": hh + hl, "bf16_b": hh + lh}


def rel(got, ref):
    got, ref = got.detach().double().cpu(), ref.detach().double().cpu()
    return ((got - ref).abs().max() / ref.abs().max().clamp_min(1e-30)).item()


# ------------------------------------------------------------------------------------------------------------------
# CPU tests of the helpers
# ------------------------------------------------------------------------------------------------------------------


def _from_bits(bits):
    return torch.from_numpy(np.array(bits, dtype=np.uint32).view(np.float32))


def _bits(x):
    return x.numpy().view(np.uint32).tolist()


def test_split_reconstructs_fp32_to_2_pow_minus_17():
    g = torch.Generator().manual_seed(1)
    x = torch.randn(1 << 16, generator=g) * torch.exp2(torch.randint(-40, 40, (1 << 16,), generator=g).float())
    hi, lo = split(x)
    assert torch.equal(bf16_rne(hi), hi) and torch.equal(bf16_rne(lo), lo)       # both planes are bf16 values
    r = ((hi.double() + lo.double() - x.double()).abs() / x.double().abs()).max().item()
    assert r <= 2.0 ** -17, r
    assert r > 2.0 ** -24                                                         # hi + lo is not exact: 16 of 24 bits


def test_bf16_rounding_is_nearest_even_with_ties():
    # (input bits, expected bf16 bits << 16): exact ties go to the even neighbour, also across a binade and for negatives
    cases = [(0x3F808000, 0x3F800000), (0x3F818000, 0x3F820000), (0x3F808001, 0x3F810000), (0x3F807FFF, 0x3F800000),
             (0xBF808000, 0xBF800000), (0xBF818000, 0xBF820000), (0x3FFF8000, 0x40000000), (0x3F7F8000, 0x3F800000),
             (0x00008000, 0x00000000), (0x00018000, 0x00020000), (0x3F800000, 0x3F800000)]
    got = _bits(bf16_rne(_from_bits([c[0] for c in cases])))
    assert got == [c[1] for c in cases]
    # and torch's own fp32 -> bf16 conversion agrees on random finite bit patterns
    g = torch.Generator().manual_seed(2)
    x = torch.randn(1 << 16, generator=g) * torch.exp2(torch.randint(-100, 100, (1 << 16,), generator=g).float())
    assert torch.equal(bf16_rne(x), x.to(torch.bfloat16).float())


def test_degraded_emulations_are_measurably_worse():
    g = torch.Generator().manual_seed(3)
    x = torch.randn(2, 64, 12, 12, generator=g)
    w = torch.randn(32, 64, 3, 3, generator=g) / 24
    ref = F.conv2d(x.double(), w.double(), padding=1)
    emu = emulations(product_terms(lambda a, b: F.conv2d(a, b, padding=1), x, w))
    e = {k: rel(v, ref) for k, v in emu.items()}
    assert e["split"] < 2e-5, e
    assert e["drop_cross"] > 30 * e["split"] and e["bf16_b"] > 30 * e["split"], e


# ------------------------------------------------------------------------------------------------------------------
# GPU cases
# ------------------------------------------------------------------------------------------------------------------
# TOL per kind of output: measured max err on one H100 80GB HBM3 x ~4 (DESIGN.md 3 lists the measurements)
TOL = {
    "conv_split": 4e-5,     # k_conv_tc, split-bf16 output (the hi + lo storage itself carries ~2^-17 relative)
    "conv_f32": 2.5e-5,     # k_conv_tc, fp32 output
    "gru": 3.5e-5,          # k_conv_tc GRU epilogues (fast sigmoid / tanh)
    "train_y": 1e-4,        # esr_conv2d_forward
    "train_dx": 4e-5,       # esr_conv2d_backward dx (k_conv_tc over g)
    "train_dw": 2e-4,       # k_wgrad_tc
    "train_db": 4e-6,       # bias gradient (fp32 sum, no product term)
    "dcn_out": 4e-5,
    "dcn_grad_input": 2e-5,
    "dcn_grad_offset": 2.5e-5,
    "dcn_grad_mask": 2.5e-5,
    "dcn_grad_weight": 1.5e-5,
    "dcn_grad_bias": 3e-6,
}


def check(name, kind, got, ref, degraded, degraded_is="A_lo B_hi dropped", tol=None):
    """err <= TOL[kind] and TOL[kind] <= err(degraded) / 4 (degraded None: no product term to lose).  tol: the
    tolerance of a kind another test module defines."""
    err = rel(got, ref)
    deg = rel(degraded, ref) if degraded is not None else None
    tol = TOL[kind] if tol is None else tol
    print(f"[tc64] {name} [{kind}]: err {err:.2e}, TOL {tol:.1e}, degraded {'n/a' if deg is None else format(deg, '.2e')}"
          f"{'' if deg is None else ' (' + degraded_is + ')'}")
    assert err <= tol, (name, kind, err, tol)
    if deg is not None:
        assert tol <= deg / 4, (name, kind, tol, deg)


pytestgpu = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    import bench
    torch.set_num_threads(bench.usable_cores())
    return torch.device("cuda:0")


def _props():
    p = torch.cuda.get_device_properties(0)
    return (p.multi_processor_count, getattr(p, "shared_memory_per_block_optin", 232448),
            getattr(p, "shared_memory_per_multiprocessor", 233472))


def tc_smem_bytes(npad, stages):
    return 1024 + stages * (2 * 16384 + 2 * npad * 128) + 2 * ((63 * 68 + 64) * 4) + 16 * stages


def conv_geometry(n_img, H, W, cin_total, ntaps, cout):
    """Launch geometry of k_conv_tc, by the rule of conv_tc_prepare / launch_np (tc_conv.cu)."""
    sm, cap, per_sm_smem = _props()
    TW = 32 if W >= 24 else (16 if W >= 12 else 8)
    TH = 128 // TW
    npad = (cout + 15) // 16 * 16
    nkb = cin_total // 64 * ntaps
    n_tiles = n_img * math.ceil(W / TW) * math.ceil(H / TH)
    stages = 6
    while stages > 2 and tc_smem_bytes(npad, stages) > cap:
        stages -= 1
    if n_tiles > sm and npad <= 64:
        s2 = stages
        while s2 > 2 and 2 * (tc_smem_bytes(npad, s2) + 1024) > cap:
            s2 -= 1
        if 2 * (tc_smem_bytes(npad, s2) + 1024) <= cap:
            stages = s2
    if stages > nkb:
        stages = max(nkb, 2)
    per_sm = max(1, min(2 if npad <= 64 else 1, per_sm_smem // (tc_smem_bytes(npad, stages) + 1024)))
    grid = max(1, min(n_tiles, per_sm * sm))
    return dict(n_tiles=n_tiles, grid=grid, per_sm=per_sm, stages=stages, nkb=nkb, npad=npad, TW=TW, TH=TH)


def wgrad_geometry(B, Cin, Cout, k, H, W):
    """Launch geometry of k_wgrad_tc, by the rule of wgrad_tc (wgrad_tc.cu)."""
    sm = _props()[0]
    cpad = (Cout + 63) // 64 * 64
    a_is_x = Cout == 64 and Cin >= 128
    m_ch, n_ch = (Cin, cpad) if a_is_x else (cpad, Cin)
    TW = 32 if W >= 24 else (16 if W >= 12 else 8)
    TH = 128 // TW
    n_tiles = B * math.ceil(W / TW) * math.ceil(H / TH)
    base = math.ceil(m_ch / 128) * (n_ch // 64) * (3 if k == 3 else 1)
    slices = max(1, min(math.ceil(sm / base), n_tiles))
    return dict(n_tiles=n_tiles, slices=slices, tiles_per_cta=n_tiles // slices, a_is_x=a_is_x, m_ch=m_ch,
                m_dup=(m_ch % 128) == 64, cpad=cpad, W=W, TW=TW)


def assert_multi_tile(geo, per_sm=None):
    assert geo["n_tiles"] >= 3 * geo["grid"] and geo["n_tiles"] % geo["grid"] != 0, geo
    if per_sm is not None:
        assert geo["per_sm"] == per_sm, geo


# ---------------------------------------------------------------------------------------------- k_conv_tc
ACT64 = {None: lambda v: v, "relu": torch.relu, "sigmoid": torch.sigmoid, "tanh": torch.tanh}


def _rand(g, *shape, scale=1.0):
    return torch.randn(*shape, generator=g) * scale


def _epilogue(acc, b, act, act_from, res, res_mode):
    v = acc + b.double().view(1, -1, 1, 1)
    if res_mode == 1:
        v = v + res
    if act is not None:
        v = torch.cat([v[:, :act_from], ACT64[act](v[:, act_from:])], 1)
    if res_mode == 2:
        v = v + res
    return v


# id: (n_img, H, W, source channels, source images (None = n_img, identity map), ntaps, cout, extras)
#   extras: act, act_from, ring ("wraps": nkb not a multiple of the stage count | "short": nkb < stages), res ("self" | n_res: separate residual of n_res images with a permuting res_img), res_mode,
#           out ("split" | "f32"), out_C, out_coff, regime ("multi" | "multi2" (two CTAs per SM) | None), check (# images)
CONV_CASES = {
    # persistence: >= 3 tiles per CTA, tile count not a multiple of the grid
    "persist_np16_2cta": (100, 32, 32, [64], None, 9, 16, dict(act="relu", out="f32", regime="multi2")),
    "persist_np64": (60, 32, 32, [64], None, 9, 64, dict(act="relu", regime="multi")),
    "persist_np128": (60, 32, 32, [64], None, 9, 128, dict(act="relu", regime="multi", ring="wraps")),
    # ring depth vs K
    "nkb1_1x1": (60, 32, 32, [64], None, 1, 64, dict(act="relu", regime="multi", ring="short")),
    "nkb2_1x1_2src": (60, 32, 32, [64, 64], None, 1, 64, dict(regime="multi")),
    "nkb3_1x1": (50, 32, 32, [192], None, 1, 96, dict(regime="multi")),
    "nkb4_1x1": (60, 32, 32, [256], None, 1, 64, dict(regime="multi", ring="wraps")),
    "nkb27_3src_dense_fusion0": (60, 32, 32, [64, 64, 64], [40, 40, 40], 9, 64, dict(act="relu", regime="multi")),
    "nkb27_3src_np128": (60, 32, 32, [64, 64, 64], [40, 40, 40], 9, 128, dict(act="relu", regime="multi", ring="wraps")),
    # epilogues
    "res_pre_permuted_coff64": (60, 32, 32, [192], None, 9, 192,
                                dict(act="relu", res=70, res_mode=1, out_C=256, out_coff=64, regime="multi")),
    "res_post_permuted_ragged": (70, 24, 40, [64], None, 9, 64, dict(act="relu", res=80, res_mode=2, regime="multi")),
    "act_from144_f32": (60, 32, 32, [64], None, 9, 216, dict(act="sigmoid", act_from=144, out="f32", regime="multi")),
    "act_from128_f32": (60, 32, 32, [64], None, 9, 216, dict(act="sigmoid", act_from=128, out="f32", regime="multi")),
    "f32_C18": (60, 32, 32, [64], None, 9, 18, dict(out="f32", regime="multi")),
    "f32_C20_cout18": (60, 32, 32, [64], None, 9, 18, dict(out="f32", out_C=20, regime="multi")),
    # geometry: the three tile-width classes, ragged H and W, W < 8, H < TH
    "geo_W6_ragged": (300, 40, 6, [64], None, 9, 64, dict(act="relu", regime="multi")),
    "geo_W19_H29": (60, 29, 19, [64], None, 9, 64, dict(act="relu", regime="multi")),
    "geo_W45_H27": (40, 27, 45, [64], None, 9, 128, dict(act="relu", regime="multi")),
    "geo_H3_W40": (200, 3, 40, [64], None, 9, 64, dict(act="relu", regime="multi")),
    # the benchmark's layers at feature resolution: cfg2 (32x32, 144 images) and cfg4 (128x128, 84 images)
    "cfg2_192_192_res_pre": (144, 32, 32, [192], None, 9, 192, dict(act="relu", res="self", res_mode=1, regime="multi")),
    "cfg2_128_64": (144, 32, 32, [128], None, 9, 64, dict(act="relu", regime="multi")),
    "cfg2_64_216": (144, 32, 32, [64], None, 9, 216, dict(act="sigmoid", act_from=144, out="f32", regime="multi")),
    "cfg4_192_192_res_pre": (84, 128, 128, [192], None, 9, 192,
                             dict(act="relu", res="self", res_mode=1, regime="multi", check=3)),
    "cfg4_128_64": (84, 128, 128, [128], None, 9, 64, dict(act="relu", regime="multi", check=3)),
    "cfg4_64_216": (84, 128, 128, [64], None, 9, 216, dict(act="sigmoid", act_from=144, out="f32", regime="multi", check=3)),
}
# every padded width esr_conv_tc accepts, at multi-tile size (split output where cout % 32 == 0)
for _c in range(16, 257, 16):
    CONV_CASES[f"width_{_c}"] = (100 if _c == 16 else 50, 32, 32, [64], None, 9, _c,
                                 dict(act="relu", out="split" if _c % 32 == 0 else "f32",
                                      regime="multi2" if _c == 16 else "multi"))


def _check_images(n_img, k):
    """The output images the CPU reference covers: first, last and spread between (all if few)."""
    if n_img <= k:
        return list(range(n_img))
    return sorted(set(np.linspace(0, n_img - 1, k).round().astype(int).tolist()))


@pytestgpu
@pytest.mark.parametrize("name", list(CONV_CASES))
def test_conv_tc_vs_fp64(dev, name):
    from esr_b200 import layers as L
    n_img, H, W, chans, src_n, ntaps, cout, ex = CONV_CASES[name]
    act, act_from, res_mode = ex.get("act"), ex.get("act_from", 0), ex.get("res_mode", 0)
    out_kind = ex.get("out", "split")
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    k = 3 if ntaps == 9 else 1
    cin = sum(chans)
    geo = conv_geometry(n_img, H, W, cin, ntaps, cout)
    if ex["regime"] == "multi2":
        assert_multi_tile(geo, per_sm=2)
    else:
        assert_multi_tile(geo)
    if ex.get("ring") == "wraps":
        assert geo["nkb"] % geo["stages"] != 0, geo                    # the ring position moves between tiles
    if ex.get("ring") == "short":
        assert geo["nkb"] < geo["stages"], geo
    src_n = src_n or [n_img] * len(chans)
    srcs = [_rand(g, n, c, H, W) for n, c in zip(src_n, chans)]
    maps = [None if n == n_img else torch.randint(0, n, (n_img,), generator=g) for n in src_n]   # repeat and permute
    w = _rand(g, cout, cin, k, k, scale=1.0 / math.sqrt(cin * ntaps))
    b = _rand(g, cout, scale=0.1)
    res_t, res_img = None, None
    if ex.get("res") == "self":
        res_t = srcs[0]
    elif ex.get("res") is not None:
        res_t = _rand(g, ex["res"], cout, H, W)
        res_img = torch.randperm(ex["res"], generator=g)[:n_img]

    s_dev = [L.Split.from_nchw(t.to(dev)) for t in srcs]
    res_dev = None if res_t is None else (s_dev[0] if ex.get("res") == "self" else L.Split.from_nchw(res_t.to(dev)))
    wp, bp = L.pack_weight(w.to(dev)), L.pad_bias(b.to(dev), cout)
    out, o32 = None, None
    if out_kind == "split":
        out = L.Split(n_img, ex.get("out_C", cout), H, W, dev)
    else:
        o32 = torch.full((n_img, H, W, ex.get("out_C", cout)), -777.0, device=dev)
    L.conv_tc(s_dev, wp, bp, cout, ntaps=ntaps, act=act, act_from=act_from, src_img=maps, n_img=n_img, res=res_dev,
              res_mode=res_mode, res_img=res_img, out=out, out_coff=ex.get("out_coff", 0), out_f32=o32)
    if out is not None:
        full = out.to_nchw().cpu()
        coff = ex.get("out_coff", 0)
        got = full[:, coff:coff + cout]
        if coff:
            assert full[:, :coff].abs().max().item() == 0.0                # channels below out_coff untouched
    else:
        full = o32.permute(0, 3, 1, 2).cpu()
        got = full[:, :cout]
        assert bool((full[:, cout:] == -777.0).all())                     # channels >= cout untouched

    imgs = _check_images(n_img, ex.get("check", 12))
    sel = torch.tensor(imgs)
    xcat = torch.cat([s[sel if m is None else m[sel]] for s, m in zip(srcs, maps)], 1)
    res64 = None
    if res_t is not None:
        res64 = res_t[sel if res_img is None else res_img[sel]].double()
    conv = lambda a, bb: F.conv2d(a, bb, padding=k // 2)                 # noqa: E731
    ref = _epilogue(conv(xcat.double(), w.double()), b, act, act_from, res64, res_mode)
    emu = emulations(product_terms(conv, xcat, w))
    deg = _epilogue(emu["drop_cross"], b, act, act_from, res64, res_mode)
    kind = "conv_split" if out is not None else "conv_f32"
    print(f"[tc64] {name}: tiles {geo['n_tiles']}, grid {geo['grid']} ({geo['per_sm']}/SM), stages {geo['stages']}, "
          f"nkb {geo['nkb']}, npad {geo['npad']}, images checked {len(imgs)}/{n_img}")
    check(name, kind, got[sel], ref, deg)


@pytestgpu
def test_split_from_nchw_matches_emulation(dev):
    """esr_split_from_nchw writes exactly the hi / lo planes of the emulation (bit for bit)."""
    from esr_b200 import layers as L
    g = torch.Generator().manual_seed(4)
    x = torch.randn(3, 128, 9, 13, generator=g) * torch.exp2(torch.randint(-20, 20, (3, 128, 9, 13), generator=g).float())
    s = L.Split.from_nchw(x.to(dev))
    hi, lo = split(x)
    got = s.buf.float().cpu()                                        # bf16 -> fp32 is exact
    assert torch.equal(got[0], hi.permute(0, 2, 3, 1)) and torch.equal(got[1], lo.permute(0, 2, 3, 1))



class _View:
    """A split tensor seen from image `k0` on: the hi / lo plane distance stays that of the whole tensor (how net.cu
    hands the ConvGRU the state of one step inside the state buffer)."""

    def __init__(self, s, k0):
        self.buf, self.n_img = s.buf[:, k0:], s.n_img


@pytestgpu
@pytest.mark.parametrize("cfg,n,H,W", [("cfg2", 16, 32, 32), ("cfg4", 4, 128, 128)])
def test_conv_tc_gru_epilogues_vs_fp64(dev, cfg, n, H, W):
    """EPI_GRU_ZR then EPI_GRU_OUT at the step size of the benchmark (2B images: both directions), with h_prev a view at a
    non-zero image offset of a larger state buffer.  Each launch is checked against float64 on the operands it read."""
    from esr_b200 import layers as L
    g = torch.Generator().manual_seed(n * 1000 + H)
    x, h_all = _rand(g, n, 64, H, W), _rand(g, 3 * n, 64, H, W, scale=0.5)
    k0 = n
    h = h_all[k0:k0 + n]
    wu, wr, wo = (_rand(g, 64, 128, 3, 3, scale=1 / 34) for _ in range(3))
    bu, br, bo = (_rand(g, 64, scale=0.1) for _ in range(3))
    geo_zr, geo_o = conv_geometry(n, H, W, 128, 9, 128), conv_geometry(n, H, W, 128, 9, 64)
    if cfg == "cfg4":
        assert_multi_tile(geo_zr)
        assert_multi_tile(geo_o)
    else:
        assert geo_zr["n_tiles"] <= geo_zr["grid"]                     # cfg2's step is a single wave

    xs, hs = L.Split.from_nchw(x.to(dev)), L.Split.from_nchw(h_all.to(dev))
    hv = _View(hs, k0)
    rh, hn = L.Split(n, 64, H, W, dev), L.Split(n, 64, H, W, dev)
    zb = torch.zeros(n, H, W, 64, device=dev)
    himg = torch.arange(n) + k0
    L.conv_tc([xs, hs], L.pack_weight(wu.to(dev), wr.to(dev)), torch.cat([bu, br]).to(dev), 128, src_img=[None, himg],
              n_img=n, epi_mode=1, h_prev=hv, z_buf=zb, out=rh)
    L.conv_tc([xs, rh], L.pack_weight(wo.to(dev)), L.pad_bias(bo.to(dev), 64), 64, n_img=n, epi_mode=2, h_prev=hv, z_buf=zb,
              out=hn)
    z_got, rh_got, hn_got = zb.permute(0, 3, 1, 2).cpu(), rh.to_nchw().cpu(), hn.to_nchw().cpu()

    conv = lambda a, bb: F.conv2d(a, bb, padding=1)                      # noqa: E731
    xh = torch.cat([x, h], 1)
    wzr, bzr = torch.cat([wu, wr]), torch.cat([bu, br]).double().view(1, -1, 1, 1)
    acc = conv(xh.double(), wzr.double()) + bzr
    acc_deg = emulations(product_terms(conv, xh, wzr))["drop_cross"] + bzr
    h64 = h.double()
    check(f"gru_zr_z_{cfg}", "gru", z_got, torch.sigmoid(acc[:, :64]), torch.sigmoid(acc_deg[:, :64]))
    check(f"gru_zr_rh_{cfg}", "gru", rh_got, h64 * torch.sigmoid(acc[:, 64:]), h64 * torch.sigmoid(acc_deg[:, 64:]))
    # the candidate launch on what it read: x, rh and z as the first launch left them
    xr = torch.cat([x, rh_got], 1)
    z = z_got.double()
    o = torch.tanh(conv(xr.double(), wo.double()) + bo.double().view(1, -1, 1, 1))
    o_deg = torch.tanh(emulations(product_terms(conv, xr, wo))["drop_cross"] + bo.double().view(1, -1, 1, 1))
    check(f"gru_out_{cfg}", "gru", hn_got, h64 * (1 - z) + o * z, h64 * (1 - z) + o_deg * z)


# ---------------------------------------------------------------------------------------------- training operators
def _act_grad(y, act):
    """act'(.) expressed through the output y, as the backward kernels do (fp32 in, same dtype out)."""
    if act == "relu":
        return (y > 0).to(y.dtype)
    if act == "sigmoid":
        return y * (1 - y)
    if act == "tanh":
        return 1 - y * y
    return torch.ones_like(y)


def _wgrad64(x, g, k, chunk=16):
    """dw[co, ci, ky, kx] = sum over images and pixels of g * shifted x, in float64 (im2col, chunked over images)."""
    co, ci = g.shape[1], x.shape[1]
    dw = torch.zeros(co, ci * k * k, dtype=torch.float64)
    for i in range(0, x.shape[0], chunk):
        cols = F.unfold(x[i:i + chunk], k, padding=k // 2)                # [n, ci*k*k, HW]
        gg = g[i:i + chunk].flatten(2)                                    # [n, co, HW]
        dw += torch.einsum("npl,nql->pq", gg, cols)
    return dw.view(co, ci, k, k)


# id: (B, Cin, Cout, k, act, H, W, deferred steps (0: plain autograd))
TRAIN_CASES = {
    "gru_zr_deferred_cfg2": (288, 128, 128, 3, "sigmoid", 32, 32, 18),     # update|reset gates: 18 steps x 16 images
    "gru_out_deferred_cfg2": (288, 128, 64, 3, "tanh", 32, 32, 18),       # candidate (a_is_x)
    "a_is_x_192_64": (24, 192, 64, 3, "relu", 32, 32, 0),
    "m_dup_64_64": (24, 64, 64, 3, "relu", 32, 32, 0),
    "m192_192_192": (16, 192, 192, 3, None, 32, 32, 0),                      # second M block half used
    "coutpad_64_32": (24, 64, 32, 3, "relu", 32, 32, 0),
    "coutpad_64_216": (16, 64, 216, 3, None, 32, 32, 0),
    "1x1_128_64": (60, 128, 64, 1, "relu", 32, 32, 0),
    "edge_W7_H21": (100, 64, 64, 3, "relu", 21, 7, 0),                        # tiles straddle the image edge, TW = 8
    "edge_W19_H23": (24, 128, 128, 3, "sigmoid", 23, 19, 0),                 # TW = 16
    "edge_W37_H30": (16, 64, 128, 3, "relu", 30, 37, 0),                      # TW = 32
}


@pytestgpu
@pytest.mark.parametrize("name", list(TRAIN_CASES))
def test_train_conv2d_vs_fp64(dev, name):
    from esr_b200 import train
    B, Cin, Cout, k, act, H, W, steps = TRAIN_CASES[name]
    geo = wgrad_geometry(B, Cin, Cout, k, H, W)
    assert geo["tiles_per_cta"] >= 2, geo                                  # every wgrad CTA accumulates several tiles
    if name.startswith("gru"):
        assert geo["tiles_per_cta"] >= 16, geo                              # each wgrad CTA walks many tiles
    if name.startswith("a_is_x") or name == "gru_out_deferred_cfg2":
        assert geo["a_is_x"], geo
    if name.startswith("m_dup"):
        assert geo["m_dup"] and geo["m_ch"] == 64, geo
    if name.startswith("m192"):
        assert geo["m_ch"] == 192 and geo["m_dup"], geo
    if name.startswith("coutpad"):
        assert geo["cpad"] > Cout, geo
    if name.startswith("edge"):
        assert W % geo["TW"] != 0, geo
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    x = _rand(g, B, Cin, H, W)
    w = _rand(g, Cout, Cin, k, k, scale=1.0 / math.sqrt(Cin * k * k))
    b = _rand(g, Cout, scale=0.1)
    dy = _rand(g, B, Cout, H, W)

    xg, wg, bg = (t.to(dev).requires_grad_() for t in (x, w, b))
    if steps:
        sunk = {}
        n = B // steps
        with train._defer_weight_grads() as d:
            ys = [train.conv2d(xg[i * n:(i + 1) * n], wg, bg, 1, act, defer=("k", lambda dw_, db_: sunk.update(dw=dw_, db=db_)))
                  for i in range(steps)]
            y = torch.cat(ys, 0)
            y.backward(dy.to(dev))
            assert wg.grad is None                                          # the weight gradient waits for flush()
            d.flush()
        dw_got, db_got = sunk["dw"].cpu(), sunk["db"].cpu()
    else:
        y = train.conv2d(xg, wg, bg, 1, act)
        y.backward(dy.to(dev))
        dw_got, db_got = wg.grad.cpu(), bg.grad.cpu()
    y_got, dx_got = y.detach().cpu(), xg.grad.cpu()

    pad = k // 2
    conv = lambda a, bb: F.conv2d(a, bb, padding=pad)                                     # noqa: E731
    b64 = b.double().view(1, -1, 1, 1)
    y64 = ACT64[act](conv(x.double(), w.double()) + b64)
    # the backward operator's reference on the y it is handed (the forward's output): act'(y) of relu is a step, and
    # fp32 and fp64 forwards disagree on the sign of near-zero outputs
    g64 = dy.double() * _act_grad(y_got.double(), act)
    dx64 = torch.nn.grad.conv2d_input(x.shape, w.double(), g64, padding=pad)
    dw64 = _wgrad64(x.double(), g64, k)
    # the operands the backward kernels see: g = dy * act'(y) in fp32 from the forward's own output
    g32 = dy * _act_grad(y_got, act)
    y_deg = ACT64[act](emulations(product_terms(conv, x, w))["drop_cross"] + b64)
    dx_deg = emulations(product_terms(lambda a, bb: torch.nn.grad.conv2d_input(x.shape, bb, a, padding=pad), g32, w))
    if geo["a_is_x"]:                                                    # M side = x: A = x, B = g
        dw_deg = emulations(product_terms(lambda a, bb: _wgrad64(a, bb, k), x, g32))
    else:                                                                # M side = g: A = g, B = x
        dw_deg = emulations(product_terms(lambda a, bb: _wgrad64(bb, a, k), g32, x))
    print(f"[tc64] {name}: wgrad tiles {geo['n_tiles']}, slices {geo['slices']}, >= {geo['tiles_per_cta']} tiles per CTA, "
          f"M side {'x' if geo['a_is_x'] else 'g'} ({geo['m_ch']} ch{', m_dup' if geo['m_dup'] else ''})")
    check(f"{name}.y", "train_y", y_got, y64, y_deg)
    check(f"{name}.dx", "train_dx", dx_got, dx64, dx_deg["drop_cross"])
    check(f"{name}.dw", "train_dw", dw_got, dw64, dw_deg["drop_cross"])
    check(f"{name}.db", "train_db", db_got, g64.sum((0, 2, 3)), None)


# ---------------------------------------------------------------------------------------------- DCNv2
def dcn_columns64(x, off, m, dg):
    """Sampled and modulated columns [B, C, 9, H, W] in float64 (the oracle's DCNv2 sampling, oracle/model_ref.py), with
    the sample position (y - 1 + i) + off formed in fp32 first, as the kernels and the reference's CUDA code do."""
    B, C, H, W = x.shape
    cpg = C // dg
    ys = torch.arange(H, dtype=torch.float32, device=x.device).view(1, 1, H, 1)
    xs = torch.arange(W, dtype=torch.float32, device=x.device).view(1, 1, 1, W)
    flat = x.reshape(B, C, H * W)
    r = lambda t: t.repeat_interleave(cpg, dim=1)                                         # noqa: E731
    cols = []
    for kk in range(9):
        i, j = kk // 3, kk % 3
        off_h = off[:, [gg * 18 + 2 * kk for gg in range(dg)]]
        off_w = off[:, [gg * 18 + 2 * kk + 1 for gg in range(dg)]]
        mk = m[:, [gg * 9 + kk for gg in range(dg)]]
        h_im = ((ys - 1 + i) + off_h.float()).double()
        w_im = ((xs - 1 + j) + off_w.float()).double()
        valid = (h_im > -1) & (w_im > -1) & (h_im < H) & (w_im < W)
        h_low, w_low = torch.floor(h_im), torch.floor(w_im)
        lh, lw = h_im - h_low, w_im - w_low
        hh, hw = 1 - lh, 1 - lw
        h_low, w_low = h_low.long(), w_low.long()
        h_high, w_high = h_low + 1, w_low + 1

        def corner(hi, wi, ok):
            ok = ok & valid
            idx = r(hi.clamp(0, H - 1) * W + wi.clamp(0, W - 1)).reshape(B, C, H * W)
            return torch.gather(flat, 2, idx).reshape(B, C, H, W) * r(ok)

        val = (r(hh * hw) * corner(h_low, w_low, (h_low >= 0) & (w_low >= 0))
               + r(hh * lw) * corner(h_low, w_high, (h_low >= 0) & (w_high <= W - 1))
               + r(lh * hw) * corner(h_high, w_low, (h_high <= H - 1) & (w_low >= 0))
               + r(lh * lw) * corner(h_high, w_high, (h_high <= H - 1) & (w_high <= W - 1)))
        cols.append(val * r(mk))
    return torch.stack(cols, 2)


def _lattice_offsets(g, B, dg, H, W, k=3, s=1, p=1, d=1):
    """Offsets (multiples of 1/8, exact in fp32) whose sample positions land on -1, 0, H-1, H (W-1, W), on integers and
    just inside / outside the border.  Any square geometry: tap (i, j) of output pixel (y, x) samples around
    (y*s - p + i*d, x*s - p + j*d); the output is [B, dg*2*k*k, Ho, Wo]."""
    def targets(n, size):
        special = torch.tensor([-1.125, -1.0, -0.875, -0.5, 0.0, 0.125, size - 1.5, size - 1.0, size - 0.875, size - 0.125,
                                float(size), size + 0.125])
        pick = torch.randint(0, 2, (n,), generator=g).bool()
        ints = torch.randint(-1, size + 1, (n,), generator=g).float()
        return torch.where(pick, special[torch.randint(0, len(special), (n,), generator=g)], ints)

    Ho, Wo = (H + 2 * p - d * (k - 1) - 1) // s + 1, (W + 2 * p - d * (k - 1) - 1) // s + 1
    off = torch.empty(B, dg, k * k, 2, Ho, Wo)
    yy = torch.arange(Ho).view(Ho, 1).float() * s - p
    xx = torch.arange(Wo).view(1, Wo).float() * s - p
    for kk in range(k * k):
        i, j = kk // k, kk % k
        n = B * dg * Ho * Wo
        off[:, :, kk, 0] = targets(n, H).view(B, dg, Ho, Wo) - (yy + i * d)
        off[:, :, kk, 1] = targets(n, W).view(B, dg, Ho, Wo) - (xx + j * d)
    return off.reshape(B, dg * 2 * k * k, Ho, Wo)


# id: (B, H, W, offsets)
DCN_CASES = {
    "production_96x32x32": (96, 32, 32, "random"),
    "lattice_borders": (4, 13, 21, "lattice"),
    # images smaller than one 16 x 8 / 8 x 16 tile: TMA's out-of-bounds fill supplies most of each box
    "subtile_1x1": (1, 1, 1, "lattice"),
    "subtile_2x300": (1, 2, 300, "lattice"),
    "subtile_300x2": (2, 300, 2, "lattice"),
    "subtile_7x9": (3, 7, 9, "lattice"),
}


@pytestgpu
@pytest.mark.parametrize("case", list(DCN_CASES))
def test_dcn_v2_vs_fp64(dev, case):
    """Forward and the five gradients of `_ext.dcn_v2_forward / backward` (64 -> 64, 8 groups) against float64."""
    from esr_b200 import dcn_v2_ext as ext
    g = torch.Generator().manual_seed(len(case))
    C, G = 64, 8
    B, H, W, offsets = DCN_CASES[case]
    if offsets == "random":
        off = _rand(g, B, G * 18, H, W, scale=2.0)
    else:
        off = _lattice_offsets(g, B, G, H, W)
    x = _rand(g, B, C, H, W)
    w = _rand(g, C, C, 3, 3, scale=1 / 24)
    b = _rand(g, C, scale=0.1)
    m = torch.rand(B, G * 9, H, W, generator=g)
    go = _rand(g, B, C, H, W)
    args = [t.to(dev) for t in (x, w, b, off, m)]
    out_got = ext.dcn_v2_forward(*args, 3, 3, 1, 1, 1, 1, 1, 1, G).cpu()
    grads_got = [t.cpu() for t in ext.dcn_v2_backward(*args, go.to(dev), 3, 3, 1, 1, 1, 1, 1, 1, G)]

    w2 = w.reshape(C, C * 9)
    contract = lambda wm, cols: torch.einsum("ok,bkhw->bohw", wm, cols.flatten(1, 2))      # noqa: E731
    back = lambda gom, wm: torch.einsum("ok,bohw->bkhw", wm, gom)                           # noqa: E731  (W^T gO)
    names = ["grad_input", "grad_offset", "grad_mask"]
    ref = {k: [] for k in ["out", "out_deg"] + names + [n + "_deg" for n in names]}
    gw, gw_deg = torch.zeros(C, C * 9, dtype=torch.float64), torch.zeros(C, C * 9, dtype=torch.float64)
    for i in range(0, B, 8):                                             # bounded memory: chunks of images
        sl = slice(i, i + 8)
        leaves = [t[sl].double().requires_grad_() for t in (x, off, m)]
        cols = dcn_columns64(leaves[0], leaves[1], leaves[2], G)
        ref["out"].append(contract(w2.double(), cols.detach()) + b.double().view(1, -1, 1, 1))
        cols32 = cols.detach().float().flatten(1, 2)                      # the sampled columns the contraction sees
        ref["out_deg"].append(emulations(product_terms(lambda a, bb: torch.einsum("bkhw,ok->bohw", a, bb), cols32, w2))
                              ["drop_cross"] + b.double().view(1, -1, 1, 1))
        gcols = back(go[sl].double(), w2.double()).view_as(cols)
        gcols_deg = emulations(product_terms(lambda a, bb: torch.einsum("bohw,ok->bkhw", a, bb), go[sl], w2))["drop_cross"]
        exact = torch.autograd.grad(cols, leaves, gcols, retain_graph=True)
        degr = torch.autograd.grad(cols, leaves, gcols_deg.view_as(cols))
        for n_, e_, d_ in zip(names, exact, degr):
            ref[n_].append(e_)
            ref[n_ + "_deg"].append(d_)
        gw += torch.einsum("bohw,bkhw->ok", go[sl].double(), cols.detach().flatten(1, 2))
        with torch.no_grad():                                            # features read without their lo plane
            cols_hi = dcn_columns64(bf16_rne(x[sl]).double(), off[sl].double(), m[sl].double(), G)
        gw_deg += torch.einsum("bohw,bkhw->ok", go[sl].double(), cols_hi.flatten(1, 2))
    cat = {k: torch.cat(v, 0) for k, v in ref.items()}
    check(f"dcn_{case}.out", "dcn_out", out_got, cat["out"], cat["out_deg"])
    for n_, got in zip(names, grads_got[:3]):
        check(f"dcn_{case}.{n_}", f"dcn_{n_}", got, cat[n_], cat[n_ + "_deg"])
    # grad_weight is an fp32 CUDA-core GEMM over columns re-sampled from the split features (dcn_bwd.cu): it has no
    # split product, so its degraded kernel is one that reads the features without their lo plane
    check(f"dcn_{case}.grad_weight", "dcn_grad_weight", grads_got[3], gw.view(C, C, 3, 3), gw_deg.view(C, C, 3, 3),
          degraded_is="features without lo plane")
    check(f"dcn_{case}.grad_bias", "dcn_grad_bias", grads_got[4], go.double().sum((0, 2, 3)), None)
