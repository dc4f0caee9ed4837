"""The drop-in boundary: after esr_b200.dropin.install() the module names the reference binds its native pieces under --
`_ext` (models/DCNv2/dcn_v2.py:13), `dataloader.cython_cnt2event.cnt2event` (cnt2event_api.py:1),
`dataloader.cython_event_redistribute.event_redistribute` (encodings.py:5) and `models.model` -- resolve to this package's
implementations.  Runs in a subprocess (it rewires sys.modules).  The GPU half drives the same call pattern as the reference's autograd Function (dcn_v2.py:17-68) and nn.Module (DCN_sep,
:197-227; example_dconv of testcuda.py:169-180 with deformable_groups=2) through `_ext` and checks it against the oracle."""
import os
import subprocess
import sys
import textwrap

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run(code):
    r = subprocess.run([sys.executable, "-c", textwrap.dedent(code)], capture_output=True, text=True, timeout=600, cwd=ROOT,
                       env=dict(os.environ, PYTHONPATH=ROOT))
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    return r.stdout


def test_install_without_reference_checkout_provides_stub_packages():
    out = _run("""
        import sys
        import esr_b200.dropin
        esr_b200.dropin.install()
        import _ext
        from dataloader.cython_cnt2event import cnt2event
        from dataloader.cython_event_redistribute import event_redistribute
        from models.model import DeepRecurrNet
        import esr_b200.cnt2event, esr_b200.event_redistribute, esr_b200.dcn_v2_ext, esr_b200.model
        assert _ext is esr_b200.dcn_v2_ext and cnt2event is esr_b200.cnt2event
        assert event_redistribute is esr_b200.event_redistribute and DeepRecurrNet is esr_b200.model.DeepRecurrNet
        # `from models.model import *` (train_ours_cnt_seq.py:20) yields the network with the reference's 68 state_dict entries
        ns = {}
        exec("from models.model import *", ns)
        assert ns["DeepRecurrNet"] is esr_b200.model.DeepRecurrNet
        assert len(ns["DeepRecurrNet"](inch=2, basech=8, num_frame=3).state_dict()) == 68
        # the CPU entry points fail loudly (no fallback), with the reference operator's message for a CPU tensor (dcn_v2.h:26)
        import torch
        w = torch.zeros(64, 64, 3, 3)
        try:
            _ext.dcn_v2_forward(torch.zeros(1, 64, 4, 4), w, torch.zeros(64), torch.zeros(1, 144, 4, 4), torch.zeros(1, 72, 4, 4),
                                3, 3, 1, 1, 1, 1, 1, 1, 8)
            raise SystemExit("expected RuntimeError")
        except RuntimeError as e:
            assert "CPU" in str(e)
        print("stub-ok")
    """)
    assert "stub-ok" in out


class _RefStyleDCN(torch.autograd.Function):
    """The call pattern of the reference's _DCNv2 Function (models/DCNv2/dcn_v2.py:17-68): forward through
    `_ext.dcn_v2_forward` (14 arguments), backward through `_ext.dcn_v2_backward` (15 arguments, five gradients)."""

    @staticmethod
    def forward(ctx, input, offset, mask, weight, bias, stride, padding, dilation, deformable_groups):
        import _ext as _backend
        ctx.cfg = (weight.shape[2], weight.shape[3], stride, stride, padding, padding, dilation, dilation, deformable_groups)
        out = _backend.dcn_v2_forward(input, weight, bias, offset, mask, *ctx.cfg)
        ctx.save_for_backward(input, offset, mask, weight, bias)
        return out

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_output):
        import _ext as _backend
        input, offset, mask, weight, bias = ctx.saved_tensors
        gi, go, gm, gw, gb = _backend.dcn_v2_backward(input, weight, bias, offset, mask, grad_output, *ctx.cfg)
        return gi, go, gm, gw, gb, None, None, None, None


@pytest.mark.gpu
@pytest.mark.parametrize("B,C,Co,H,W,G", [(2, 64, 64, 32, 32, 8), (2, 64, 64, 24, 40, 2), (1, 64, 64, 16, 16, 1), (2, 64, 64, 20, 12, 4),
                                         (2, 2, 2, 4, 4, 1), (1, 16, 24, 9, 7, 2), (1, 128, 64, 10, 10, 8)])
def test_ext_operator_through_reference_call_pattern(B, C, Co, H, W, G):
    """incl. example_dconv's DCN(64, 64, deformable_groups=2) (testcuda.py:169-180) and the reference tests' own tiny
    configuration N=2, inC=outC=2, 4x4, one group (testcuda.py:14-17); forward and all five gradients vs autograd through
    the oracle's modulated deformable convolution."""
    import esr_b200.dropin
    from oracle import model_ref
    esr_b200.dropin.install(patch_models=False)
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(B * 100 + C + G)
    x = torch.randn(B, C, H, W, generator=g)
    off = torch.randn(B, 2 * G * 9, H, W, generator=g) * 1.5
    msk = torch.sigmoid(torch.randn(B, G * 9, H, W, generator=g))
    wgt = torch.randn(Co, C, 3, 3, generator=g) * (1.0 / (C * 9)) ** 0.5
    bia = torch.randn(Co, generator=g) * 0.1
    gout = torch.randn(B, Co, H, W, generator=g)
    ref_in = [t.clone().requires_grad_() for t in (x, off, msk, wgt, bia)]
    want = model_ref.dcn_v2_forward(ref_in[0], ref_in[3], ref_in[4], ref_in[1], ref_in[2], G)
    want.backward(gout)
    got_in = [t.clone().to(dev).requires_grad_() for t in (x, off, msk, wgt, bia)]
    got = _RefStyleDCN.apply(got_in[0], got_in[1], got_in[2], got_in[3], got_in[4], 1, 1, 1, G)
    got.backward(gout.to(dev))
    rel = lambda a, b: ((a.cpu() - b).abs().max() / b.abs().max().clamp_min(1e-20)).item()
    assert rel(got.detach(), want.detach()) < 1e-4
    for name, a, b in zip(("input", "offset", "mask", "weight", "bias"), got_in, ref_in):
        assert rel(a.grad, b.grad) < 5e-4, (name, rel(a.grad, b.grad))


@pytest.mark.gpu
def test_zero_offset_identity_known_answer():
    """models/DCNv2/testcuda.py:32-67 (check_zero_offset) at the reference's own sizes: identity kernel, zero offsets, mask 0.5
    => 2 * out == in."""
    import esr_b200.dropin
    esr_b200.dropin.install(patch_models=False)
    import _ext
    dev = torch.device("cuda:0")
    N, inC, H, W = 2, 2, 4, 4
    x = torch.randn(N, inC, H, W, device=dev)
    w = torch.zeros(inC, inC, 3, 3, device=dev)
    for p in range(inC):
        w[p, p, 1, 1] = 1.0
    out = _ext.dcn_v2_forward(x, w, torch.zeros(inC, device=dev), torch.zeros(N, 18, H, W, device=dev),
                              torch.full((N, 9, H, W), 0.5, device=dev), 3, 3, 1, 1, 1, 1, 1, 1, 1)
    assert (x - 2 * out).abs().max().item() < 1e-6
