"""The generic DCNv2 operators (csrc/dcn_generic.cu) against float64, at every geometry they serve.

`_ext.dcn_v2_forward` / `dcn_v2_backward` (esr_b200.dcn_v2_ext) run every configuration other than the network's own
(64 -> 64, 3x3, stride 1, pad 1, dilation 1, 8 groups) on fp32 CUDA-core kernels: k_dcng_columns (sampling),
k_dcng_gemm in three transposes (out, grad_columns, grad_weight), k_dcng_bias_grad and k_dcng_bwd_sample (grad_input /
grad_offset / grad_mask).  Each case here runs the forward and the backward through `_ext` and compares the six outputs
with `dcn64`, a float64 restatement of modulated deformable convolution for any square geometry.  The table also holds
the network's own configuration (the other side of the dispatch, under test_tc_fp64_gpu.py's tolerances); further cases
put every sample outside the image and drive the grid-stride loops into their second pass.  The last tests check that
both operators reject malformed arguments before anything is launched.

`dcn64` is anchored on the CPU: it equals torchvision.ops.deform_conv2d in float64 to 1e-12, forward and all five
gradients, over the whole case table at reduced sizes.

Norm: err = max |got - ref64| / max |ref64| (test_tc_fp64_gpu.py).  The kernels are fp32 FFMA with no split product, so
their degraded kernel (marked * in DESIGN.md 3) is the same float64 computation on operands rounded to bf16: the features
for out, grad_offset, grad_mask and grad_weight, grad_output for grad_input.  Every case asserts err <= TOL and
TOL <= err(degraded) / 4; grad_bias is a plain sum and only gets err <= TOL.  TOL is about 4x the largest error measured
on an H100.
"""
import math
import os
import re

import pytest
import torch

from tests.test_tc_fp64_gpu import TOL as TUNED_TOL
from tests.test_tc_fp64_gpu import _lattice_offsets, bf16_rne, rel

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "esr_b200", "csrc")

# ------------------------------------------------------------------------------------------------------------------
# float64 restatement (CPU)
# ------------------------------------------------------------------------------------------------------------------


def out_size(H, W, k, s, p, d):
    return (H + 2 * p - d * (k - 1) - 1) // s + 1, (W + 2 * p - d * (k - 1) - 1) // s + 1


def _position(base, off):
    """base (fp32, integer-valued) + off, formed in fp32 as the kernels do and only then widened.  The value is the fp32
    sum; the derivative with respect to off is exactly 1 (no fp32 rounding on the way back)."""
    v = (base + off.detach().float()).double()
    return v + (off - off.detach())


def dcn64(x, off, m, w, b, k, s, p, d, G, y0=0, x_row0=0, H=None):
    """Modulated deformable convolution in float64, differentiable in all five operands by autograd.

    x [B, C, Hx, W], off [B, G*2*k*k, Ho, Wo] (per group and tap: dy, dx), m [B, G*k*k, Ho, Wo], w [Co, C, k, k], b [Co].
    Tap (i, j) of output pixel (y, x) samples channel c of group c // (C/G) at (y*s - p + i*d + dy, x*s - p + j*d + dx),
    bilinearly; a sample counts only inside (-1, H) x (-1, W), and corners outside the image read as zero.
    A band of a tall image: off / m hold output rows y0.., x holds input rows x_row0.. of an image H rows high; every
    corner the band reads must lie in x."""
    B, C, Hx, W = x.shape
    H = Hx if H is None else H
    Co, K = w.shape[0], k * k
    Ho, Wo = off.shape[2:]
    cpg, P = C // G, Ho * Wo
    ys = (torch.arange(Ho, dtype=torch.float32).view(Ho, 1) + y0) * s - p
    xs = torch.arange(Wo, dtype=torch.float32).view(1, Wo) * s - p
    flat = x.reshape(B, G, cpg, Hx * W)
    offv, mv = off.reshape(B, G, K, 2, Ho, Wo), m.reshape(B, G, K, Ho, Wo)
    cols = []
    for kk in range(K):
        i, j = kk // k, kk % k
        h, wp = _position(ys + i * d, offv[:, :, kk, 0]), _position(xs + j * d, offv[:, :, kk, 1])
        valid = (h > -1) & (wp > -1) & (h < H) & (wp < W)
        h_low, w_low = torch.floor(h.detach()), torch.floor(wp.detach())
        lh, lw = h - h_low, wp - w_low
        hh, hw = 1 - lh, 1 - lw
        h_low, w_low = h_low.long(), w_low.long()

        def corner(hi, wi):
            ok = valid & (hi >= 0) & (hi <= H - 1) & (wi >= 0) & (wi <= W - 1)
            r = hi - x_row0
            assert bool(((r >= 0) & (r < Hx))[ok].all()), "the band reads rows outside x"
            idx = (r.clamp(0, Hx - 1) * W + wi.clamp(0, W - 1)).reshape(B, G, 1, P).expand(B, G, cpg, P)
            return torch.gather(flat, 3, idx).reshape(B, G, cpg, Ho, Wo) * ok.unsqueeze(2).to(x.dtype)

        val = ((hh * hw).unsqueeze(2) * corner(h_low, w_low) + (hh * lw).unsqueeze(2) * corner(h_low, w_low + 1)
               + (lh * hw).unsqueeze(2) * corner(h_low + 1, w_low) + (lh * lw).unsqueeze(2) * corner(h_low + 1, w_low + 1))
        cols.append(val * mv[:, :, kk].unsqueeze(2))
    cols = torch.stack(cols, 3).reshape(B, C * K, P)                  # row c*K + tap, as the kernels' columns
    out = torch.einsum("or,brp->bop", w.reshape(Co, C * K), cols)
    return out.reshape(B, Co, Ho, Wo) + b.view(1, Co, 1, 1)


def dcn64_grads(x, off, m, w, b, go, geo, chunk=2, **band):
    """-> [out, grad_input, grad_offset, grad_mask, grad_weight, grad_bias] in float64 (chunks of `chunk` images)."""
    k, s, p, d, G = geo
    w64, b64 = w.double().requires_grad_(), b.double().requires_grad_()
    outs, gx, goff, gm = [], [], [], []
    gw, gb = torch.zeros_like(w64), torch.zeros_like(b64)
    for i in range(0, x.shape[0], chunk):
        sl = slice(i, i + chunk)
        leaves = [t[sl].double().requires_grad_() for t in (x, off, m)]
        out = dcn64(*leaves, w64, b64, k, s, p, d, G, **band)
        grads = torch.autograd.grad(out, leaves + [w64, b64], go[sl].double())
        outs.append(out.detach())
        for acc, gr in zip((gx, goff, gm), grads[:3]):
            acc.append(gr)
        gw += grads[3]
        gb += grads[4]
    return [torch.cat(outs), torch.cat(gx), torch.cat(goff), torch.cat(gm), gw, gb]


# ------------------------------------------------------------------------------------------------------------------
# the case table
# ------------------------------------------------------------------------------------------------------------------
# id: (B, C, Co, H, W, k, s, p, d, G, scale of the random offsets)
CASES = {
    "ref_tiny": (2, 2, 2, 4, 4, 3, 1, 1, 1, 1, 1.0),              # the reference's own tests (testcuda.py:14-17)
    "k1_p0": (3, 5, 7, 11, 13, 1, 1, 0, 1, 1, 0.5),
    "k5_g3": (2, 12, 40, 17, 23, 5, 1, 2, 1, 3, 2.0),              # two M tiles with a remainder, 4 channels per group
    "s2_g2": (2, 16, 24, 19, 21, 3, 2, 1, 1, 2, 1.5),              # 10 x 11 output
    "s3_p0": (1, 8, 8, 20, 17, 3, 3, 0, 1, 1, 3.0),                # 6 x 5 output, floor in Ho
    "d2_g4": (2, 32, 33, 15, 26, 3, 1, 2, 2, 4, 2.0),              # dilated taps
    "s2_p3_d3_depthwise": (2, 6, 6, 23, 18, 3, 2, 3, 3, 6, 4.0),   # one channel per group, pad > k / 2
    "out_1x1": (2, 4, 5, 3, 3, 3, 1, 0, 1, 2, 1.0),                # a single output pixel
    "row_1x9": (2, 4, 5, 1, 9, 3, 1, 1, 1, 2, 1.0),                # a one-row input
    # one parameter away from the network's configuration: each takes the generic path
    "tuned_nb_s2": (2, 64, 64, 24, 20, 3, 2, 1, 1, 8, 2.0),
    "tuned_nb_p0": (2, 64, 64, 24, 20, 3, 1, 0, 1, 8, 2.0),
    "tuned_nb_d2_p2": (2, 64, 64, 24, 20, 3, 1, 2, 2, 8, 2.0),
    "tuned_nb_k1_p0": (2, 64, 64, 24, 20, 1, 1, 0, 1, 8, 2.0),
    "tuned_nb_g4": (2, 64, 64, 24, 20, 3, 1, 1, 1, 4, 2.0),
    "tuned_nb_co32": (2, 64, 32, 24, 20, 3, 1, 1, 1, 8, 2.0),
    "tuned_nb_c128": (2, 128, 64, 24, 20, 3, 1, 1, 1, 8, 2.0),
    # the network's own configuration (wgmma path, test_tc_fp64_gpu.py's tolerances): the other side of the dispatch
    "tuned": (2, 64, 64, 24, 20, 3, 1, 1, 1, 8, 2.0),
    # grad_weight summed over 8 x 64 x 64 = 32 768 pixels: a 4096-long fp32 reduction per image, images added by atomics
    "long_reduction": (8, 64, 64, 128, 128, 3, 2, 1, 1, 8, 2.0),
}

# measured max err on one H100 80GB HBM3 (700 W power limit) x ~4, worst case named (DESIGN.md 3)
TOL = {
    "out": 5e-6,            # 1.2e-6, tuned_nb_c128 (K = 1152)
    "grad_input": 5e-6,     # 1.1e-6, long_reduction (fp32 atomics)
    "grad_offset": 1.2e-6,  # 2.9e-7
    "grad_mask": 1.2e-6,    # 2.8e-7
    "grad_weight": 6e-6,    # 1.4e-6, long_reduction (4096-pixel fp32 sums, images added by atomics)
    "grad_bias": 1.2e-6,    # 2.9e-7, long_reduction
}
OUTPUTS = ["out", "grad_input", "grad_offset", "grad_mask", "grad_weight", "grad_bias"]
TUNED_KIND = {"out": "dcn_out", "grad_input": "dcn_grad_input", "grad_offset": "dcn_grad_offset", "grad_mask": "dcn_grad_mask",
              "grad_weight": "dcn_grad_weight", "grad_bias": "dcn_grad_bias"}


def _source(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def tuned_config():
    """(C, Co, kernel, stride, pad, dil, G) of dcn_is_tuned (net.cuh): the one configuration on the wgmma path."""
    m = re.search(r"dcn_is_tuned\([^)]*\)\s*\{\s*return C == (\d+) && Co == (\d+) && kernel == (\d+) && stride == (\d+) && "
                  r"pad == (\d+) && dil == (\d+) && G == (\d+);", _source("net.cuh"))
    assert m, "dcn_is_tuned changed: restate it here"
    return tuple(int(v) for v in m.groups())


def is_tuned(case):
    B, C, Co, H, W, k, s, p, d, G, _ = case
    return (C, Co, k, s, p, d, G) == tuned_config()


def grid_cap():
    """Threads of the largest grid1d launch (dcn_generic.cu): past it the grid-stride loops take a second pass."""
    m = re.search(r"grid1d\(size_t total\)\s*\{\s*return \(unsigned\)\(total / 256 \+ 1 > (\d+)u \* (\d+)u", _source("dcn_generic.cu"))
    assert m, "grid1d changed: restate it here"
    return int(m.group(1)) * int(m.group(2)) * 256


def gemm_dims(case):
    """(M, N, K) of the three k_dcng_gemm launches: out = W . columns, grad_columns = W^T . grad_out,
    grad_weight = grad_out . columns^T."""
    B, C, Co, H, W, k, s, p, d, G, _ = case
    Ho, Wo = out_size(H, W, k, s, p, d)
    P, R = Ho * Wo, C * k * k
    return {"out": (Co, P, R), "grad_columns": (R, P, Co), "grad_weight": (Co, R, P)}


def test_case_table_covers_the_generic_operator():
    """Every value of every geometric parameter the cases promise, both sides of the dispatch, and in each of the three
    GEMM launches an M, an N and a K remainder after at least one full 32-wide tile."""
    rows = list(CASES.values())
    col = lambda i: {r[i] for r in rows}                                  # noqa: E731
    assert {1, 3, 5} <= col(5) and {1, 2, 3} <= col(6) and {0, 1, 2, 3} <= col(7) and {1, 2, 3} <= col(8)
    assert {1, 2, 3, 4, 6, 8} <= col(9)
    assert any(r[1] == r[9] for r in rows)                                # one channel per group
    assert any(r[7] > r[5] // 2 for r in rows)                            # padding beyond the kernel's half width
    sizes = [(r[3], r[4], out_size(r[3], r[4], *r[5:9])) for r in rows]
    assert any(o == (1, 1) for _, _, o in sizes) and any(h == 1 for h, _, _ in sizes)
    assert any((r[3] + 2 * r[7] - r[8] * (r[5] - 1) - 1) % r[6] for r in rows if r[6] > 1)   # Ho rounds down
    assert all(min(*o) >= 1 for _, _, o in sizes)
    # dispatch: exactly "tuned" is the network's configuration; each neighbour differs from it and runs generic
    assert [n for n, r in CASES.items() if is_tuned(r)] == ["tuned"]
    neighbours = [n for n in CASES if n.startswith("tuned_nb_")]
    assert len(neighbours) == 7
    for n in neighbours:
        assert CASES[n][1:3] + CASES[n][5:10] != CASES["tuned"][1:3] + CASES["tuned"][5:10]
    for gemm in ("out", "grad_columns", "grad_weight"):
        for axis, name in enumerate("MNK"):
            assert any(gemm_dims(r)[gemm][axis] > 32 and gemm_dims(r)[gemm][axis] % 32 for r in rows if not is_tuned(r)), \
                (gemm, name)
    # the grid-stride case: B C Ho Wo (columns) and B G K Ho Wo (sampling backward) threads, 4096 past the cap
    B, C, G, H, W = GRID_STRIDE
    assert B * C * H * W == B * G * H * W == grid_cap() + 4096 == 1 << 28
    assert 4096 == 4 * W                                                  # the last four rows of channel / group C-1 of image B-1


def _reduced(case):
    B, C, Co, H, W, k, s, p, d, G, scale = case
    return (1, C, Co, min(H, 13), min(W, 13), k, s, p, d, G, scale)


def _dyadic_offsets(g, B, G, H, W, k, s, p, d):
    """Multiples of 2^-8 with |off| < 8, exact in fp32, moved by 2^-8 where a position would land exactly on -1 or H
    (-1 or W).  There torchvision's offset gradient differs from the reference operator's: the reference
    (dcn_v2_im2col_cuda.cu) zeroes the coordinate gradient of a sample outside (-1, H) x (-1, W), torchvision takes it
    from the one corner inside.  The GPU cases pin the reference's rule at those positions with lattice offsets."""
    Ho, Wo = out_size(H, W, k, s, p, d)
    off = (torch.randint(-2046, 2047, (B, G, k * k, 2, Ho, Wo), generator=g).double() / 256)
    taps = torch.arange(k * k)
    base_h = (torch.arange(Ho) * s - p).view(Ho, 1) + (taps // k * d).view(-1, 1, 1)
    base_w = (torch.arange(Wo) * s - p).view(1, Wo) + (taps % k * d).view(-1, 1, 1)
    for a, base, size in ((0, base_h, H), (1, base_w, W)):
        pos = off[:, :, :, a] + base
        off[:, :, :, a] += ((pos == -1) | (pos == size)).double() / 256
    return off.reshape(B, G * 2 * k * k, Ho, Wo)


@pytest.mark.parametrize("name", list(CASES))
def test_dcn64_matches_torchvision(name):
    """dcn64 == torchvision.ops.deform_conv2d in float64 to 1e-12, forward and the five gradients, on dyadic offsets so
    that both references see the same sample positions."""
    tv = pytest.importorskip("torchvision.ops")
    B, C, Co, H, W, k, s, p, d, G, _ = _reduced(CASES[name])
    Ho, Wo = out_size(H, W, k, s, p, d)
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    x = torch.randn(B, C, H, W, generator=g, dtype=torch.float64)
    off = _dyadic_offsets(g, B, G, H, W, k, s, p, d)
    m = torch.rand(B, G * k * k, Ho, Wo, generator=g, dtype=torch.float64) * 2 - 0.5
    w = torch.randn(Co, C, k, k, generator=g, dtype=torch.float64)
    b = torch.randn(Co, generator=g, dtype=torch.float64)
    go = torch.randn(B, Co, Ho, Wo, generator=g, dtype=torch.float64)
    got = dcn64_grads(x, off, m, w, b, go, (k, s, p, d, G))
    leaves = [t.clone().requires_grad_() for t in (x, off, m, w, b)]
    out = tv.deform_conv2d(leaves[0], leaves[1], leaves[3], leaves[4], stride=s, padding=p, dilation=d, mask=leaves[2])
    want = [out.detach()] + list(torch.autograd.grad(out, leaves, go))
    for n_, a, bb in zip(OUTPUTS, got, want):
        assert a.shape == bb.shape, (n_, a.shape, bb.shape)
        assert rel(a, bb) <= 1e-12, (name, n_, rel(a, bb))


def test_dcn64_is_the_3x3_columns_of_test_tc_fp64():
    """At 3x3 / s1 / p1 / d1 dcn64 contracts the columns of test_tc_fp64_gpu.dcn_columns64 (the tuned path's reference)."""
    from tests.test_tc_fp64_gpu import dcn_columns64
    g = torch.Generator().manual_seed(5)
    B, C, Co, H, W, G = 2, 16, 8, 9, 11, 4
    x, w = torch.randn(B, C, H, W, generator=g), torch.randn(Co, C, 3, 3, generator=g)
    off = torch.randn(B, G * 18, H, W, generator=g) * 2
    m, b = torch.rand(B, G * 9, H, W, generator=g), torch.randn(Co, generator=g)
    cols = dcn_columns64(x.double(), off.double(), m.double(), G)
    want = torch.einsum("ok,bkhw->bohw", w.reshape(Co, C * 9).double(), cols.flatten(1, 2)) + b.double().view(1, -1, 1, 1)
    assert rel(dcn64(x.double(), off.double(), m.double(), w.double(), b.double(), 3, 1, 1, 1, G), want) <= 1e-14


# ------------------------------------------------------------------------------------------------------------------
# GPU cases
# ------------------------------------------------------------------------------------------------------------------
pytestgpu = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    import bench
    torch.set_num_threads(bench.usable_cores())
    return torch.device("cuda:0")


def check(name, kind, got, ref, degraded, tol, degraded_is):
    """err <= tol and tol <= err(degraded) / 4 (degraded None: no product term to lose)."""
    err = rel(got, ref)
    deg = rel(degraded, ref) if degraded is not None else None
    print(f"[dcn64] {name}.{kind}: err {err:.2e}, tol {tol:.1e}, degraded "
          f"{'n/a' if deg is None else format(deg, '.2e') + ' (' + degraded_is + ')'}")
    assert err <= tol, (name, kind, err, tol)
    if deg is not None:
        assert tol <= deg / 4, (name, kind, tol, deg)


def _generic_ws_bytes(B, C, k, Ho, Wo):
    return (B * C * k * k * Ho * Wo * 4 + 255) // 256 * 256


def _run_ext(dev, x, w, b, off, m, go, k, s, p, d, G):
    from esr_b200 import dcn_v2_ext as ext
    args = [t.to(dev) for t in (x, w, b, off, m)]
    cfg = (k, k, s, s, p, p, d, d, G)
    out = ext.dcn_v2_forward(*args, *cfg)
    grads = ext.dcn_v2_backward(*args, go.to(dev), *cfg)
    return [out.cpu()] + [t.cpu() for t in grads]


def _compare(name, got, ref, deg_x, deg_go, tuned):
    degraded = {"out": deg_x[0], "grad_input": deg_go[1], "grad_offset": deg_x[2], "grad_mask": deg_x[3],
                "grad_weight": deg_x[4], "grad_bias": None}
    for i, kind in enumerate(OUTPUTS):
        tol = TUNED_TOL[TUNED_KIND[kind]] if tuned else TOL[kind]
        check(name, kind, got[i], ref[i], degraded[kind], tol,
              "grad_output rounded to bf16" if kind == "grad_input" else "features rounded to bf16")


@pytestgpu
@pytest.mark.parametrize("offsets", ["random", "lattice"])
@pytest.mark.parametrize("name", list(CASES))
def test_dcn_generic_vs_fp64(dev, name, offsets):
    """Forward and the five gradients of `_ext` at one geometry of the table, against dcn64."""
    from esr_b200 import _lib
    B, C, Co, H, W, k, s, p, d, G, scale = CASES[name]
    Ho, Wo = out_size(H, W, k, s, p, d)
    tuned = is_tuned(CASES[name])
    # the launch takes the path the case claims: the two paths size their workspaces differently
    L = _lib.lib()
    ws = L.esr_dcn_v2_workspace_bytes_ex(B, C, H, W, Co, k, s, p, d, G, 0)
    assert ws == (L.esr_dcn_v2_workspace_bytes(B, H, W) if tuned else _generic_ws_bytes(B, C, k, Ho, Wo)), (name, ws)
    g = torch.Generator().manual_seed(sum(map(ord, name + offsets)))
    x = torch.randn(B, C, H, W, generator=g)
    if offsets == "random":
        off = torch.randn(B, G * 2 * k * k, Ho, Wo, generator=g) * scale
    else:
        off = _lattice_offsets(g, B, G, H, W, k, s, p, d)
    m = torch.rand(B, G * k * k, Ho, Wo, generator=g) * 2 - 0.5          # negative and > 1 masks too
    w = torch.randn(Co, C, k, k, generator=g) / math.sqrt(C * k * k)
    b = torch.randn(Co, generator=g) * 0.1
    go = torch.randn(B, Co, Ho, Wo, generator=g)
    got = _run_ext(dev, x, w, b, off, m, go, k, s, p, d, G)
    geo = (k, s, p, d, G)
    ref = dcn64_grads(x, off, m, w, b, go, geo)
    deg_x = dcn64_grads(bf16_rne(x), off, m, w, b, go, geo)
    deg_go = dcn64_grads(x, off, m, w, b, bf16_rne(go), geo)
    _compare(f"{name}_{offsets}", got, ref, deg_x, deg_go, tuned)


@pytestgpu
def test_dcn_generic_every_sample_outside(dev):
    """Every sample outside (-1, H) x (-1, W), on one axis or both, including exactly -1 and H: the forward is the bias,
    bit for bit, and grad_input, grad_offset, grad_mask and grad_weight are exactly zero."""
    B, C, Co, H, W, k, s, p, d, G = 2, 8, 6, 9, 11, 3, 2, 1, 1, 2
    Ho, Wo = out_size(H, W, k, s, p, d)
    g = torch.Generator().manual_seed(11)
    n = B * G * k * k * Ho * Wo

    def outside(size):
        far = torch.tensor([-1.0, -1.125, -3.5, -40.0, float(size), size + 0.125, size + 2.5, size + 40.0])
        return far[torch.randint(0, len(far), (n,), generator=g)]

    def inside(size):
        return torch.randint(-7, 8 * size - 7, (n,), generator=g).float() / 8           # in (-1, size)

    axis = torch.randint(0, 3, (n,), generator=g)                         # 0: h outside, 1: w outside, 2: both
    th = torch.where(axis == 1, inside(H), outside(H)).view(B, G, k * k, Ho, Wo)
    tw = torch.where(axis == 0, inside(W), outside(W)).view(B, G, k * k, Ho, Wo)
    taps = torch.arange(k * k)
    base_h = (torch.arange(Ho).float() * s - p).view(1, 1, 1, Ho, 1) + (taps // k * d).float().view(1, 1, -1, 1, 1)
    base_w = (torch.arange(Wo).float() * s - p).view(1, 1, 1, 1, Wo) + (taps % k * d).float().view(1, 1, -1, 1, 1)
    off = torch.stack([th - base_h, tw - base_w], 3).reshape(B, G * 2 * k * k, Ho, Wo)
    x = torch.randn(B, C, H, W, generator=g)
    m = torch.rand(B, G * k * k, Ho, Wo, generator=g) * 2 - 0.5
    w, b = torch.randn(Co, C, k, k, generator=g), torch.randn(Co, generator=g)
    go = torch.randn(B, Co, Ho, Wo, generator=g)
    out, gi, goff, gm, gw, gb = _run_ext(dev, x, w, b, off, m, go, k, s, p, d, G)
    assert torch.equal(out, b.view(1, Co, 1, 1).expand_as(out))
    for name_, t in (("grad_input", gi), ("grad_offset", goff), ("grad_mask", gm), ("grad_weight", gw)):
        assert t.abs().max().item() == 0.0, name_
    check("all_outside", "grad_bias", gb, go.double().sum((0, 2, 3)), None, TOL["grad_bias"], None)


# B, C (= G), G, H, W with a 1x1 kernel, pad 0, Co 8
GRID_STRIDE = (2, 128, 128, 1024, 1024)


@pytestgpu
def test_dcn_generic_grid_stride_second_pass(dev):
    """B 2, C = G = 128 -> Co 8 at 1024 x 1024, 1x1 kernel, pad 0: B C Ho Wo and B G K Ho Wo are 2^28 threads, 4096 more
    than the largest grid1d launch covers, so the last four rows of channel / group 127 of image 1 are handled by the
    second pass of the grid-stride loops of k_dcng_columns and k_dcng_bwd_sample.

    The float64 reference covers a band: output rows 1016-1023 of image 1, all channels, for out, grad_offset and
    grad_mask, and input rows 1017-1023 for grad_input (with |off| < 1 they receive nothing from outside the band).
    grad_weight and grad_bias have no grid-stride loop and are left to the other cases.  Inputs are generated on the
    device; peak device memory is 10.1 GiB (inputs 4 GiB, gradients 4 GiB, the backward's two column buffers 2 GiB),
    and everything is freed before the float64 reference runs."""
    B, C, G, H, W = GRID_STRIDE
    Co, y0 = 8, H - 8
    gen = torch.Generator(device=dev).manual_seed(3)
    x = torch.randn(B, C, H, W, device=dev, generator=gen)
    off = torch.rand(B, 2 * G, H, W, device=dev, generator=gen).mul_(2).sub_(1)          # (-1, 1)
    m = torch.rand(B, G, H, W, device=dev, generator=gen).mul_(2).sub_(0.5)
    w = torch.randn(Co, C, 1, 1, device=dev, generator=gen) / math.sqrt(C)
    b = torch.randn(Co, device=dev, generator=gen) * 0.1
    go = torch.randn(B, Co, H, W, device=dev, generator=gen)
    torch.cuda.reset_peak_memory_stats(dev)
    from esr_b200 import dcn_v2_ext as ext
    cfg = (1, 1, 1, 1, 0, 0, 1, 1, G)
    out = ext.dcn_v2_forward(x, w, b, off, m, *cfg)
    out_band = out[1:, :, y0:].cpu()
    del out
    gi, goff, gm, gw, gb = ext.dcn_v2_backward(x, w, b, off, m, go, *cfg)
    got = [out_band, gi[1:, :, y0 + 1:].cpu(), goff[1:, :, y0:].cpu(), gm[1:, :, y0:].cpu()]
    band = [t[1:, :, y0 - 1:].cpu() for t in (x,)] + [t[1:, :, y0:].cpu() for t in (off, m, go)]
    wb = [w.cpu(), b.cpu()]
    peak = torch.cuda.max_memory_allocated(dev) / 2 ** 30
    del x, off, m, go, gi, goff, gm, gw, gb
    torch.cuda.empty_cache()
    print(f"[dcn64] grid_stride: peak device memory {peak:.1f} GiB")
    assert float(band[1].abs().max()) <= 1
    xb, ob, mb, gob = band
    geo = (1, 1, 0, 1, G)
    kw = dict(y0=y0, x_row0=y0 - 1, H=H)
    ref = dcn64_grads(xb, ob, mb, *wb, gob, geo, **kw)
    deg_x = dcn64_grads(bf16_rne(xb), ob, mb, *wb, gob, geo, **kw)
    deg_go = dcn64_grads(xb, ob, mb, *wb, bf16_rne(gob), geo, **kw)
    # grad_input of the band's x: rows y0-1 .. H-1; rows y0+1 .. H-1 are complete
    for i, kind in enumerate(OUTPUTS[:4]):
        r, dx, dg = ref[i], deg_x[i], deg_go[i]
        if kind == "grad_input":
            r, dx, dg = r[:, :, 2:], dx[:, :, 2:], dg[:, :, 2:]
        degraded = dg if kind == "grad_input" else dx
        check("grid_stride", kind, got[i], r, degraded, TOL[kind],
              "grad_output rounded to bf16" if kind == "grad_input" else "features rounded to bf16")


# ------------------------------------------------------------------------------------------------------------------
# argument validation: both operators raise before any launch
# ------------------------------------------------------------------------------------------------------------------
def _valid_args(dev):
    """B 2, C 4 -> Co 6, 7 x 9, 3x3, stride 2, pad 1, 2 groups: Ho x Wo = 4 x 5."""
    g = torch.Generator().manual_seed(0)
    B, C, Co, H, W, G, Ho, Wo = 2, 4, 6, 7, 9, 2, 4, 5
    t = dict(input=torch.randn(B, C, H, W, generator=g), weight=torch.randn(Co, C, 3, 3, generator=g),
             bias=torch.randn(Co, generator=g), offset=torch.randn(B, G * 18, Ho, Wo, generator=g),
             mask=torch.rand(B, G * 9, Ho, Wo, generator=g), grad_output=torch.randn(B, Co, Ho, Wo, generator=g))
    return {k: v.to(dev) for k, v in t.items()}, [3, 3, 2, 2, 1, 1, 1, 1, G]


def _call(op, t, cfg):
    from esr_b200 import dcn_v2_ext as ext
    if op == "forward":
        return ext.dcn_v2_forward(t["input"], t["weight"], t["bias"], t["offset"], t["mask"], *cfg)
    return ext.dcn_v2_backward(t["input"], t["weight"], t["bias"], t["offset"], t["mask"], t["grad_output"], *cfg)


def _shape(name, *shape):
    return lambda t, cfg: t.__setitem__(name, torch.zeros(shape, device=t["input"].device))


def _arg(i, v):
    return lambda t, cfg: cfg.__setitem__(i, v)


# id: (change to the valid call, message (regex), forward too)
REJECTIONS = {
    "kernel_h_ne_w": (_arg(1, 5), r"only square kernels / strides", True),
    "stride_h_ne_w": (_arg(3, 1), r"only square kernels / strides", True),
    "pad_h_ne_w": (_arg(5, 0), r"only square kernels / strides", True),
    "dilation_h_ne_w": (_arg(7, 2), r"only square kernels / strides", True),
    "weight_kernel_shape": (_shape("weight", 6, 4, 5, 5), r"Input shape and kernel shape wont match: \(3 x 3 vs 5 x 5\)", True),
    "weight_more_channels": (_shape("weight", 6, 8, 3, 3), r"Input shape and kernel channels wont match: \(4 vs 8\)", True),
    "weight_fewer_channels": (_shape("weight", 6, 2, 3, 3), r"Input shape and kernel channels wont match: \(4 vs 2\)", True),
    "offset_channels": (_shape("offset", 2, 18, 4, 5), r"offset has shape \[2, 18, 4, 5\], expected \[2, 36, 4, 5\]", True),
    "offset_spatial": (_shape("offset", 2, 36, 7, 9), r"offset has shape \[2, 36, 7, 9\], expected \[2, 36, 4, 5\]", True),
    "offset_batch": (_shape("offset", 1, 36, 4, 5), r"offset has shape", True),
    "mask_channels": (_shape("mask", 2, 9, 4, 5), r"mask has shape \[2, 9, 4, 5\], expected \[2, 18, 4, 5\]", True),
    "mask_spatial": (_shape("mask", 2, 18, 4, 6), r"mask has shape", True),
    "bias_length": (_shape("bias", 7), r"bias has shape \[7\], expected \[6\]", True),
    "grad_output_spatial": (_shape("grad_output", 2, 6, 7, 9),
                            r"grad_output has shape \[2, 6, 7, 9\], expected \[2, 6, 4, 5\]", False),
    "grad_output_channels": (_shape("grad_output", 2, 4, 4, 5), r"grad_output has shape", False),
    "cpu_tensor_first": (lambda t, cfg: (t.__setitem__("input", t["input"].cpu()), cfg.__setitem__(1, 5)),
                         r"^Not compiled with CPU support$", True),
    "weight_on_cpu": (lambda t, cfg: t.__setitem__("weight", t["weight"].cpu()), r"expected all tensors on cuda", True),
}


@pytestgpu
def test_valid_call_runs(dev):
    t, cfg = _valid_args(dev)
    assert _call("forward", t, cfg).shape == (2, 6, 4, 5)
    assert [tuple(r.shape) for r in _call("backward", t, cfg)] == [(2, 4, 7, 9), (2, 36, 4, 5), (2, 18, 4, 5), (6, 4, 3, 3), (6,)]


@pytestgpu
@pytest.mark.parametrize("name", list(REJECTIONS))
def test_invalid_arguments_raise(dev, name):
    """Each operator raises RuntimeError with the same message (but for the operator's name) where the other does;
    dcn_v2_backward checks grad_output as well."""
    change, msg, fwd = REJECTIONS[name]
    messages = {}
    for op in (["forward"] if fwd else []) + ["backward"]:
        t, cfg = _valid_args(dev)
        change(t, cfg)
        with pytest.raises(RuntimeError, match=msg) as e:
            _call(op, t, cfg)
        messages[op] = str(e.value).replace(f"dcn_v2_{op}", "dcn_v2_<op>")
    assert len(set(messages.values())) == 1, messages
    torch.cuda.synchronize()
