"""The element-wise glue of the inference plan (elementwise.cu) against exact fp32 emulations and float64, launcher by launcher.

esr_glue (through esr_b200.layers.glue) runs one of the launchers esr_net_forward calls: ltc_cat, chan_max, attn_mlp,
attn_apply, scale_aggregate, upsample2x, copy_split.  Inputs are split tensors built here plane by plane (hi, lo), so the
test knows the exact values a kernel reads: hi + lo in fp32.

Bit-exact where the arithmetic allows it.  k_ltc_cat, k_attn_apply and k_chan_max compile to fp32 adds of hi + lo, plain FMULs
(no FFMA) and the output split, so an fp32 CPU emulation -- the float64 restatement below run in fp32, with the products in the
kernel's order, then split() through bf16_rne -- reproduces both output planes bit for bit, and the channel maxima exactly.
copy_split is a byte-for-byte copy.  Should the compiler ever contract a product into the split's subtraction, only hi stays
bit-exact: then require equality on hi and hold hi + lo to the split's 2^-17.

Against float64 for the rest: k_scale_aggregate and k_upsample2x use FFMA, k_attn_mlp uses fmaf and expf.  Each case asserts
err <= TOL and TOL <= err(degraded) / 4 (tests.test_tc_fp64_gpu.check), where the degraded kernel reads its split inputs
without their lo plane (attn_mlp: the maxima rounded to bf16).  TOL is about 4x the error measured on an H100.

Outputs are pre-filled with a sentinel (NaN, or an int no maximum maps to): images >= n_img keep it, and every element below
n_img is written.  Every input holds more images than the launch reads, so a wrong plane stride shows.
"""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import model_ref
from tests.test_small_conv_fp64_gpu import up2_64
from tests.test_tc_fp64_gpu import _check_images, bf16_rne, check, rel, split

# ------------------------------------------------------------------------------------------------------------------
# float64 restatements of model_ref's expressions (NCHW); run in fp32 they are the kernels' own arithmetic where noted
# ------------------------------------------------------------------------------------------------------------------


def ltc64(f, maps, idx5):
    """cat(f[i0] * map[p0], f[i1], f[i2] * map[p1]) per row (i0, i1, i2, p0, p1) of idx5 (model_ref:178).  fp32: k_ltc_cat."""
    m0, m1 = maps[idx5[:, 3]].unsqueeze(1), maps[idx5[:, 4]].unsqueeze(1)
    return torch.cat([f[idx5[:, 0]] * m0, f[idx5[:, 1]], f[idx5[:, 2]] * m1], 1)


def chan_max64(t):
    """Global max pool per image and channel (model_ref:252).  Exact in any precision."""
    return t.flatten(2).amax(2)


def mlp64(mx, w0, b0, w1, b1):
    """Channel attention: sigmoid(w1 relu(w0 mx + b0) + b1) (model_ref:253-254)."""
    return torch.sigmoid(torch.relu(mx @ w0.T + b0) @ w1.T + b1)


def attn_apply64(al, mid, sk, ck):
    """cat((al sk0) ck[:C], (mid sk1) ck[C:]) (model_ref:255-256).  fp32: k_attn_apply, same product order."""
    C = al.shape[1]
    return torch.cat([al * sk[:, 0:1] * ck[:, :C, None, None], mid * sk[:, 1:2] * ck[:, C:, None, None]], 1)


def scale_aggregate64(x, feats, att, fidx, N):
    """x + mean over n < N of feats[f] att[f], f = fidx[img * N + n] (model_ref:264-266)."""
    fa = feats[fidx] * att[fidx].unsqueeze(1)
    return x + fa.view(x.shape[0], N, *fa.shape[1:]).sum(1) / N


# ------------------------------------------------------------------------------------------------------------------
# the plan's index tables (net.cu build()), restated
# ------------------------------------------------------------------------------------------------------------------


def plan_tables(B, L, N):
    """Tables and counts of the plan for (B, L, N): window slot vb = w * B + b reads bank frame b * L + w + i."""
    Wn = L - N + 1
    VB, mid = Wn * B, (N - 1) // 2

    def fr(vb, i):
        return (vb % B) * L + vb // B + i
    l5, mfr = [], []
    for vb in range(VB):
        for i in range(N):
            i0, i2 = (0 if i == 0 else i - 1), (N - 1 if i == N - 1 else i + 1)
            l5.append([fr(vb, i0), fr(vb, i), fr(vb, i2), vb * (N + 1) + i, vb * (N + 1) + i + 1])
            mfr.append(fr(vb, i))
    fm = [vb * N + mid for i in range(N) if i != mid for vb in range(VB)]
    return dict(VB=VB, VN=VB * N, nf=(N - 1) * VB, FR=B * L, NP=VB * (N + 1), l5=torch.tensor(l5), fr=torch.tensor(mfr),
                fm=torch.tensor(fm))


# ------------------------------------------------------------------------------------------------------------------
# CPU tests of the helpers
# ------------------------------------------------------------------------------------------------------------------


class _Spy:
    """model_ref's torch.nn.functional, recording the arguments and results of conv2d, linear and interpolate."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        fn = getattr(F, name)
        if name not in ("conv2d", "linear", "interpolate"):
            return fn

        def rec(*a, **k):
            r = fn(*a, **k)
            self.calls.append((name, a, r))
            return r
        return rec


@pytest.mark.parametrize("N", [3, 5])
def test_restatements_are_model_refs_expressions(N, monkeypatch):
    """One float64 forward of model_ref with its conv2d / linear / interpolate recorded: each restatement, applied to the
    recorded operands, reproduces the tensor model_ref computed."""
    sd = {k: v.double() for k, v in model_ref.seeded_state_dict(7, num_frame=N).items()}
    B, H, W = 2, 32, 40
    inp = torch.poisson(torch.full((B, N, 2, H, W), 0.5), generator=torch.Generator().manual_seed(N)).double()
    spy = _Spy()
    monkeypatch.setattr(model_ref, "F", spy)
    model_ref.forward(sd, inp)
    p = "spacetime_fuse."

    def conv_io(wname, k=0):
        """(input, output before the activation) of the k-th call of a layer"""
        hits = [(a[0], r) for n, a, r in spy.calls if n == "conv2d" and a[1] is sd[wname + ".weight"]]
        return hits[k]
    # local_time_corre: frames (i-1, i, i+1) edge-replicated, maps of pairs (i-1, i), (i, i+1)
    f = torch.relu(conv_io("feat_extract.convblock.2.conv2d")[1]).view(B, N, 64, H // 8, W // 8)
    tabs = plan_tables(1, N, N)
    for i in range(N):
        cat_in = conv_io("time_propagate.local_fusion.0.conv1", i)[0]
        m0 = torch.sigmoid(conv_io("time_propagate.pred_map.1.conv2d", 2 * i)[1][:, 0])
        m1 = torch.sigmoid(conv_io("time_propagate.pred_map.1.conv2d", 2 * i + 1)[1][:, 0])
        idx = tabs["l5"][i].clone()
        idx[3:] = torch.tensor([0, 1])
        got = torch.cat([ltc64(f[b], torch.stack([m0[b], m1[b]]), idx.view(1, 5)) for b in range(B)])
        assert (got - cat_in).abs().max().item() == 0.0, i
    # channel attention and its application, per non-middle frame
    lin = [(a, r) for n, a, r in spy.calls if n == "linear"]
    for k in range(N - 1):
        ft, sk = conv_io(p + "kernel.conv2d", k)
        sk = torch.sigmoid(sk)
        mx = chan_max64(ft)
        assert torch.equal(mx, lin[2 * k][0][0])
        ck = mlp64(mx, sd[p + "fc.0.layers.0.weight"], sd[p + "fc.0.layers.0.bias"], sd[p + "fc.0.layers.1.weight"],
                   sd[p + "fc.0.layers.1.bias"])
        assert (ck - torch.sigmoid(lin[2 * k + 1][1])).abs().max().item() < 1e-15
        al_f1 = conv_io(p + "convblock.0.conv2d", k)[0]
        y = attn_apply64(al_f1[:, :64], al_f1[:, 64:], sk, ck)
        assert (y - conv_io(p + "dcn_fusion.0.conv2d", k)[0]).abs().max().item() == 0.0
    # scale aggregation and the bilinear x2, at the three decoder scales
    ups = [(a[0], r) for n, a, r in spy.calls if n == "interpolate"]
    x = conv_io(p + "dense_fusion.1.conv2d")[1]
    for s in range(3):
        ft, at = conv_io(p + f"attens.{s}.conv2d")
        got = scale_aggregate64(x, ft, torch.sigmoid(at[:, 0]), torch.arange(B * N), N)
        assert (got - ups[s][0]).abs().max().item() < 1e-14 * ups[s][0].abs().max().item()
        assert (up2_64(ups[s][0]) - ups[s][1]).abs().max().item() < 1e-12
        x = torch.relu(conv_io(p + f"recons.{s}.conv2d")[1])


def test_plan_tables_are_the_windows_frames():
    """The restated tables against the windows model_ref.forward forms: slot i of window w, sample b, reads frames
    (i-1, i, i+1) edge-replicated, maps of pairs (i0, i) and (i, i2); the middle frame repeats for every neighbour."""
    for B, L, N in [(8, 8, 3), (2, 16, 3), (2, 7, 5), (1, 9, 7)]:
        t = plan_tables(B, L, N)
        for vb in range(t["VB"]):
            w, b = vb // B, vb % B
            for i in range(N):
                idx = [0, 0, 1] if i == 0 else ([N - 2, N - 1, N - 1] if i == N - 1 else [i - 1, i, i + 1])
                assert t["l5"][vb * N + i][:3].tolist() == [b * L + w + j for j in idx]
                assert t["fr"][vb * N + i].item() == b * L + w + i
        assert int(t["l5"][:, 3:].max()) == t["NP"] - 1 and int(t["l5"][:, :3].max()) == t["FR"] - 1
        assert sorted(set(t["fm"].tolist())) == [vb * N + (N - 1) // 2 for vb in range(t["VB"])]


# ------------------------------------------------------------------------------------------------------------------
# cases
# ------------------------------------------------------------------------------------------------------------------
CFG2, CFG4 = (8, 8, 3), (2, 16, 3)
# id: (op, H, W, C, extras)
#   plan (B, L, N): the launch's image counts and index tables are the plan's; otherwise n (images), N, in_n (input images)
#   idx: "plan" (the plan's table), "null" (identity), "rand" (a random table with repeats)
#   fill (chan_max): "neg" all negative, "zeros" +-0.0 and negatives, "lo" maxima decided by the lo plane
#   check: images compared on the host
GLUE_CASES = {
    "ltc_cat_cfg2": ("ltc_cat", 32, 32, 64, dict(plan=CFG2, idx="plan", check=8)),
    "ltc_cat_cfg4": ("ltc_cat", 128, 128, 64, dict(plan=CFG4, idx="plan", check=4)),
    "ltc_cat_n5_7x9": ("ltc_cat", 7, 9, 64, dict(plan=(2, 7, 5), idx="plan")),
    "chan_max_cfg2": ("chan_max", 32, 32, 64, dict(plan=CFG2, check=16)),
    "chan_max_cfg4": ("chan_max", 128, 128, 64, dict(plan=CFG4, check=8)),
    "chan_max_130x135": ("chan_max", 130, 135, 64, dict(n=3, in_n=5)),
    "chan_max_1x1": ("chan_max", 1, 1, 64, dict(n=7, in_n=9)),
    "chan_max_3x5": ("chan_max", 3, 5, 64, dict(n=5, in_n=6)),
    "chan_max_neg_37x29": ("chan_max", 37, 29, 64, dict(n=4, in_n=6, fill="neg")),
    "chan_max_zeros_19x21": ("chan_max", 19, 21, 64, dict(n=4, in_n=5, fill="zeros")),
    "chan_max_lo_33x17": ("chan_max", 33, 17, 64, dict(n=4, in_n=5, fill="lo")),
    "attn_mlp_cfg2": ("attn_mlp", 1, 1, 64, dict(plan=CFG2)),
    "attn_mlp_cfg4": ("attn_mlp", 1, 1, 64, dict(plan=CFG4)),
    "attn_apply_cfg2": ("attn_apply", 32, 32, 64, dict(plan=CFG2, idx="plan", check=8)),
    "attn_apply_cfg4": ("attn_apply", 128, 128, 64, dict(plan=CFG4, idx="plan", check=4)),
    "attn_apply_null_11x13": ("attn_apply", 11, 13, 64, dict(n=5, in_n=7, idx="null")),
    "scale_aggregate_c64_cfg2": ("scale_aggregate", 32, 32, 64, dict(plan=CFG2, idx="plan", check=6)),
    "scale_aggregate_c32_cfg2": ("scale_aggregate", 64, 64, 32, dict(plan=CFG2, idx="plan", check=6)),
    "scale_aggregate_c16_cfg2": ("scale_aggregate", 128, 128, 16, dict(plan=CFG2, idx="plan", check=4)),
    "scale_aggregate_c64_cfg4": ("scale_aggregate", 128, 128, 64, dict(plan=CFG4, idx="plan", check=3)),
    "scale_aggregate_n5_c32": ("scale_aggregate", 18, 22, 32, dict(plan=(2, 7, 5), idx="plan")),
    "scale_aggregate_n7_c16": ("scale_aggregate", 36, 44, 16, dict(plan=(1, 9, 7), idx="plan")),
    "scale_aggregate_null_n3_c8": ("scale_aggregate", 13, 7, 8, dict(n=4, N=3, in_n=6, idx="null")),
    "upsample2x_cfg2": ("upsample2x", 32, 32, 64, dict(plan=CFG2, check=6)),
    "upsample2x_cfg4": ("upsample2x", 128, 128, 64, dict(plan=CFG4, check=3)),
    "upsample2x_1x1": ("upsample2x", 1, 1, 64, dict(n=3, in_n=4)),
    "upsample2x_1x9": ("upsample2x", 1, 9, 32, dict(n=2, in_n=3)),
    "upsample2x_7x1": ("upsample2x", 7, 1, 16, dict(n=2, in_n=4)),
    "upsample2x_odd_13x7": ("upsample2x", 13, 7, 64, dict(n=3, in_n=5)),
    "upsample2x_wide_5x300": ("upsample2x", 5, 300, 8, dict(n=2, in_n=3)),
    "copy_split_cfg2": ("copy_split", 32, 32, 64, dict(n=16, in_n=16 * 25, idx="rand")),
    "copy_split_null_9x11": ("copy_split", 9, 11, 24, dict(n=3, in_n=5, idx="null")),
}
# TOL per op (float64 comparisons): measured max err on one H100 80GB HBM3 x ~4 (DESIGN.md 3 lists the measurements)
TOL = {
    "scale_aggregate": 2.5e-5,    # split output: the hi + lo storage itself carries ~2^-17 relative (measured 6.3e-6)
    "upsample2x": 2e-5,           # (4.7e-6)
    "attn_mlp": 1.2e-6,           # fp32 output, fmaf + expf (3.1e-7)
}
BIT_EXACT = {"ltc_cat", "chan_max", "attn_apply", "copy_split"}
NAN_ORD = 0x7FC00000              # the int sentinel of chan_max: above every ordered finite float


def _counts(op, ex):
    """(n_img, input images, second input images, N, index table or None) of a case."""
    if "plan" in ex:
        B, L, N = ex["plan"]
        t = plan_tables(B, L, N)
        return {"ltc_cat": (t["VN"], t["FR"] + 3, t["NP"] + 3, N, t["l5"]),
                "chan_max": (t["nf"], t["nf"] + 3, 0, N, None),
                "attn_mlp": (t["nf"], 0, 0, N, None),
                "attn_apply": (t["nf"], t["nf"] + 3, t["VN"] + 3, N, t["fm"]),
                "scale_aggregate": (t["VB"], t["VB"] + 3, t["FR"] + 3, N, t["fr"]),
                "upsample2x": (t["VB"], t["VB"] + 3, 0, N, None)}[op]
    n, N = ex["n"], ex.get("N", 0)
    return n, ex["in_n"], (n * N + 2 if op == "scale_aggregate" else ex["in_n"] + 2), N, None


def test_case_table_covers_every_edge():
    ids = lambda op: [k for k, v in GLUE_CASES.items() if v[0] == op]                       # noqa: E731
    assert {v[0] for v in GLUE_CASES.values()} == set(TOL) | BIT_EXACT
    # chan_max: the clamped grid (more than 64 x 256 pixels per image), images of fewer than 32 pixels, the fills
    cm = [GLUE_CASES[k] for k in ids("chan_max")]
    assert any(H * W > 64 * 256 for _, H, W, _, _ in cm) and any(H * W == 64 * 256 for _, H, W, _, _ in cm)
    assert any(H * W == 1 for _, H, W, _, _ in cm) and any(1 < H * W < 32 for _, H, W, _, _ in cm)
    assert {ex.get("fill") for *_, ex in cm} >= {"neg", "zeros", "lo"}
    # scale_aggregate: every C and N the plan runs; upsample2x: H = 1, W = 1, odd sizes, a row wider than one block
    sa = [(C, _counts("scale_aggregate", ex)[3]) for _, _, _, C, ex in (GLUE_CASES[k] for k in ids("scale_aggregate"))]
    assert {c for c, _ in sa} >= {64, 32, 16} and {n for _, n in sa} >= {3, 5, 7}
    up = [GLUE_CASES[k] for k in ids("upsample2x")]
    assert any(H == 1 for _, H, *_ in up) and any(W == 1 for _, _, W, *_ in up)
    assert any(H % 2 and W % 2 and H > 1 and W > 1 for _, H, W, *_ in up)
    assert any(2 * W * C // 8 > 256 and H * W < 4096 for _, H, W, C, _ in up)
    # index tables: the null and the table form where the launcher takes either; repeats, with the LTC boundary patterns
    for op in ("attn_apply", "scale_aggregate", "copy_split"):
        assert {GLUE_CASES[k][4]["idx"] for k in ids(op)} >= {"null", "plan" if op != "copy_split" else "rand"}, op
    for k in ids("ltc_cat"):
        l5 = _counts("ltc_cat", GLUE_CASES[k][4])[4]
        assert any(r[0] == r[1] for r in l5.tolist()) and any(r[1] == r[2] for r in l5.tolist())
    # every tensor holds more images than the launch processes; the plan's shapes at cfg2 and cfg4
    for k, (op, H, W, C, ex) in GLUE_CASES.items():
        n, in_n, in2_n, N, idx = _counts(op, ex)
        if op == "ltc_cat":
            assert in_n > int(idx[:, :3].max()) + 1 and in2_n > int(idx[:, 3:].max()) + 1, k
        elif op != "attn_mlp":
            assert in_n > n and (in2_n == 0 or in2_n > (n * N if idx is None else int(idx.max()) + 1)), k
    for op in TOL.keys() | BIT_EXACT - {"copy_split"}:
        assert {GLUE_CASES[k][4].get("plan") for k in ids(op)} >= {CFG2, CFG4}, op


# ------------------------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------------------------


@pytest.fixture(scope="module")
def dev():
    import bench
    torch.set_num_threads(bench.usable_cores())
    return torch.device("cuda:0")


def _split_tensor(dev, hi, lo):
    """A Split on `dev` with the given planes (fp32 NHWC tensors of bf16 values)."""
    from esr_b200 import layers as Lyr
    n, H, W, C = hi.shape
    s = Lyr.Split(n, C, H, W, dev)
    s.buf.copy_(torch.stack([hi, lo]).to(torch.bfloat16))
    return s


def _rand_planes(g, n, H, W, C, fill=None):
    """(hi, lo) of random fp32 values, or of a chan_max edge fill."""
    x = torch.randn(n, H, W, C, generator=g)
    if fill == "neg":
        return split(-x.abs() - 0.01)
    hi, lo = split(x)
    if fill == "zeros":                      # channels 0-7: only +-0.0; 8-15: -0.0 (both planes) and negatives
        z = torch.where(torch.rand(n, H, W, 8, generator=g) < 0.5, -0.0, 0.0)
        hi[..., :8], lo[..., :8] = z, z
        neg_hi, neg_lo = split(-x[..., 8:16].abs() - 0.01)
        zero = torch.rand(n, H, W, 8, generator=g) < 0.2
        hi[..., 8:16] = torch.where(zero, -0.0, neg_hi)
        lo[..., 8:16] = torch.where(zero, -0.0, neg_lo)
    if fill == "lo":                         # one hi per (image, channel); the maximum is decided by lo alone
        h = bf16_rne(torch.randn(n, 1, 1, C, generator=g)).expand(n, H, W, C).contiguous()
        return h, bf16_rne(h * torch.rand(n, H, W, C, generator=g) * 2.0 ** -10)
    return hi, lo


def _val(hi, lo):
    return hi + lo                           # fp32: what load8 reads


def _nchw(t):
    return t.permute(0, 3, 1, 2)


def _planes_of(s, sel):
    b = s.buf[:, sel].float().cpu()
    return b[0], b[1]


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(GLUE_CASES))
def test_glue_vs_fp64(dev, case):
    from esr_b200 import layers as Lyr
    op, H, W, C, ex = GLUE_CASES[case]
    n, in_n, in2_n, N, idx = _counts(op, ex)
    g = torch.Generator().manual_seed(sum(map(ord, case)))
    if ex.get("idx") == "rand":
        idx = torch.randint(0, in_n, (n,), generator=g)
    if ex.get("idx") == "null":
        idx = None
    sel = torch.tensor(_check_images(n, ex.get("check", 12)))
    nan = float("nan")
    Ho, Wo, Co = (2 * H, 2 * W, C) if op == "upsample2x" else (H, W, {"ltc_cat": 192, "attn_apply": 128}.get(op, C))
    print(f"[glue64] {case}: {op} n_img {n}, {H}x{W}x{C}, N {N}, inputs {in_n}/{in2_n} images, "
          f"table {'none' if idx is None else len(idx)}, images checked {len(sel)}/{n}")

    if op in ("chan_max", "attn_mlp"):
        if op == "chan_max":
            hi, lo = _rand_planes(g, in_n, H, W, C, ex.get("fill"))
            mx = torch.full((n + 2, 64), NAN_ORD, dtype=torch.int32, device=dev)
            Lyr.glue(op, n, H, W, C, x=_split_tensor(dev, hi, lo), mx=mx)
            got = mx.cpu()
            assert bool((got[n:] == NAN_ORD).all()) and not bool((got[:n] == NAN_ORD).any())
            got = got[:n]
            # ordered int -> float: i >= 0 ? i : i ^ 0x7fffffff
            gf = torch.from_numpy(np.where(got.numpy() >= 0, got.numpy(), got.numpy() ^ 0x7FFFFFFF).astype(np.int32).view(np.float32))
            want = chan_max64(_nchw(_val(hi, lo))[:n])
            assert torch.equal(gf, want), (gf - want).abs().max()
            bits = lambda t: t.numpy().view(np.int32)                                         # noqa: E731
            nz = want != 0
            assert (bits(gf)[nz.numpy()] == bits(want)[nz.numpy()]).all()
            if ex.get("fill") == "zeros":
                assert (bits(gf[:, 8:16]) == np.int32(-2 ** 31)).all()                          # -0.0, above every negative
            if ex.get("fill") == "lo":
                assert not torch.equal(want, chan_max64(_nchw(hi)[:n]))                         # the lo plane decides
            print(f"[glue64] {case}: channel maxima bit-exact")
            return
        mxf = torch.randn(n + 3, 64, generator=g) * 2
        ordi = mxf.numpy().view(np.int32)
        mx = torch.from_numpy(np.where(ordi >= 0, ordi, ordi ^ 0x7FFFFFFF).astype(np.int32)).to(dev)
        w0, b0 = torch.randn(32, 64, generator=g) / 8, torch.randn(32, generator=g) * 0.1
        w1, b1 = torch.randn(128, 32, generator=g) / math.sqrt(32), torch.randn(128, generator=g) * 0.1
        ck = torch.full((n + 2, 128), nan, device=dev)
        Lyr.glue(op, n, 1, 1, 64, mlp=[t.to(dev) for t in (w0, b0, w1, b1)], mx=mx, ck=ck)
        got = ck.cpu()
        assert bool(got[n:].isnan().all()) and not bool(got[:n].isnan().any())
        W64 = [t.double() for t in (w0, b0, w1, b1)]
        ref = mlp64(mxf[:n].double(), *W64)
        deg = mlp64(bf16_rne(mxf[:n]).double(), *W64)
        check(case, op, got[:n], ref, deg, "maxima rounded to bf16", tol=TOL[op])
        return

    # ---- split in, split out
    hi, lo = _rand_planes(g, in_n, H, W, C)
    x = _split_tensor(dev, hi, lo)
    kw = dict(x=x, idx=idx, N=N)
    if op == "ltc_cat":
        maps = torch.rand(in2_n, H, W, generator=g)
        kw["maps"] = maps.to(dev)
    if op == "attn_apply":
        hi2, lo2 = _rand_planes(g, in2_n, H, W, C)
        sk, ckv = torch.rand(n, H, W, 2, generator=g), torch.rand(n + 1, 128, generator=g)
        kw.update(x2=_split_tensor(dev, hi2, lo2), sk=sk.to(dev), ck_in=ckv.to(dev))
    if op == "scale_aggregate":
        hi2, lo2 = _rand_planes(g, in2_n, H, W, C)
        att = torch.rand(in2_n, H, W, generator=g)
        kw.update(x2=_split_tensor(dev, hi2, lo2), att=att.to(dev))
    out = Lyr.Split(n + 2, Co, Ho, Wo, dev)
    out.buf.fill_(nan)
    Lyr.glue(op, n, H, W, C, out=out, **kw)
    assert bool(out.buf[:, n:].isnan().all()), "images >= n_img written"
    assert not bool(out.buf[:, :n].isnan().any()), "output not fully written"
    gh, gl = _planes_of(out, sel)

    if op == "copy_split":
        src = torch.arange(n) if idx is None else idx
        assert torch.equal(out.buf[:, :n].view(torch.int16), x.buf[:, src.to(dev)].view(torch.int16))
        print(f"[glue64] {case}: byte-for-byte copy")
        return
    if op in ("ltc_cat", "attn_apply"):
        v = _nchw(_val(hi, lo))
        if op == "ltc_cat":
            y = ltc64(v, maps, idx[sel])
        else:
            mid = _nchw(_val(hi2, lo2))[sel if idx is None else idx[sel]]
            y = attn_apply64(v[sel], mid, sk[sel].permute(0, 3, 1, 2), ckv[sel])
        wh, wl = split(y.permute(0, 2, 3, 1))
        assert torch.equal(gh, wh) and torch.equal(gl, wl), (rel(gh + gl, wh + wl), (gh != wh).sum(), (gl != wl).sum())
        print(f"[glue64] {case}: both planes bit-exact")
        return

    got = _nchw(gh.double() + gl.double())
    v64, vhi = _nchw(hi.double() + lo.double()), _nchw(hi.double())
    if op == "scale_aggregate":
        fidx = (torch.arange(n * N) if idx is None else idx).view(n, N)[sel].flatten()
        f64, fhi = _nchw(hi2.double() + lo2.double()), _nchw(hi2.double())
        ref = scale_aggregate64(v64[sel], f64, att.double(), fidx, N)
        deg = scale_aggregate64(vhi[sel], fhi, att.double(), fidx, N)
    else:
        ref, deg = up2_64(v64[sel]), up2_64(vhi[sel])
    check(case, op, got, ref, deg, "input without lo plane", tol=TOL[op])


def _rejects(fn, what):
    from esr_b200 import _lib
    with pytest.raises(_lib.ESRError) as e:
        fn()
    assert "code -1" in str(e.value) and what in str(e.value), str(e.value)


@pytest.mark.gpu
def test_glue_rejects_bad_arguments(dev):
    """ESR_EINVAL, with a message, before any launch: missing pointers, a C the kernel has no code for, too few output or
    input images, grid limits.  A sentinel-filled output stays untouched by every refused call."""
    from esr_b200 import layers as Lyr
    g = torch.Generator().manual_seed(5)
    x = _split_tensor(dev, *_rand_planes(g, 4, 3, 5, 64))
    x8 = _split_tensor(dev, *_rand_planes(g, 4, 3, 5, 8))
    out = Lyr.Split(4, 64, 3, 5, dev)
    out.buf.fill_(float("nan"))
    mx = torch.zeros(4, 64, dtype=torch.int32, device=dev)
    att = torch.rand(12, 3, 5, device=dev)
    # missing pointers
    _rejects(lambda: Lyr.glue("copy_split", 4, 3, 5, 64, out=out), "missing input")
    _rejects(lambda: Lyr.glue("copy_split", 4, 3, 5, 64, x=x), "missing output")
    _rejects(lambda: Lyr.glue("ltc_cat", 2, 3, 5, 64, x=x, out=Lyr.Split(2, 192, 3, 5, dev)), "idx and maps")
    _rejects(lambda: Lyr.glue("chan_max", 4, 3, 5, 64, x=x), "missing mx")
    _rejects(lambda: Lyr.glue("attn_mlp", 4, 1, 1, 64, mx=mx, ck=torch.zeros(4, 128, device=dev)), "attn_mlp")
    _rejects(lambda: Lyr.glue("attn_apply", 4, 3, 5, 64, x=x, x2=x, out=Lyr.Split(4, 128, 3, 5, dev)), "sk or ck_in")
    _rejects(lambda: Lyr.glue("scale_aggregate", 4, 3, 5, 64, x=x, x2=x, N=1, out=out), "missing att")
    _rejects(lambda: Lyr.glue("scale_aggregate", 1, 3, 5, 64, x=x, out=out, att=att, N=3), "missing second input")
    # C the kernels are not written for
    _rejects(lambda: Lyr.glue("chan_max", 4, 3, 5, 32, x=x, mx=mx), "C=32")
    _rejects(lambda: Lyr.glue("copy_split", 4, 3, 5, 12, x=x8, out=out), "C=12")
    # too few images: outputs, and inputs read without a table
    _rejects(lambda: Lyr.glue("copy_split", 5, 3, 5, 64, x=_split_tensor(dev, *_rand_planes(g, 6, 3, 5, 64)), out=out), "output images")
    _rejects(lambda: Lyr.glue("chan_max", 5, 3, 5, 64, x=_split_tensor(dev, *_rand_planes(g, 6, 3, 5, 64)), mx=mx), "output images")
    _rejects(lambda: Lyr.glue("upsample2x", 4, 3, 5, 64, x=x, out=Lyr.Split(3, 64, 6, 10, dev)), "output images")
    _rejects(lambda: Lyr.glue("copy_split", 4, 3, 5, 64, x=_split_tensor(dev, *_rand_planes(g, 3, 3, 5, 64)), out=out), "input holds")
    _rejects(lambda: Lyr.glue("scale_aggregate", 4, 3, 5, 64, x=x, x2=x, att=att, N=3, out=out), "frames for")
    # grid limits
    big = torch.zeros(65536, 64, dtype=torch.int32, device=dev)
    _rejects(lambda: Lyr.glue("chan_max", 65536, 1, 1, 64, x=Lyr.Split(65536, 64, 1, 1, dev), mx=big), "65535")
    _rejects(lambda: Lyr.glue("upsample2x", 1, 32768, 1, 8, x=Lyr.Split(1, 8, 32768, 1, dev), out=Lyr.Split(1, 8, 65536, 2, dev)),
             "65535")
    _rejects(lambda: Lyr.glue("upsample2x", 65536, 1, 1, 8, x=Lyr.Split(65536, 8, 1, 1, dev), out=Lyr.Split(65536, 8, 2, 2, dev)),
             "65535")
    assert bool(out.buf.isnan().all())
