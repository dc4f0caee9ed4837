"""Generate tests/golden/model_nf_golden.npz: the REFERENCE's own models/model.py at num_frame = 5, 7 and 9
(build container only; same stubs and seeded weights as make_golden_model.py).

`DeepRecurrNet(inch=2, basech=8, num_frame=N)` loads `oracle.model_ref.seeded_state_dict(seed, num_frame=N)`.
Each case runs `nwin` sliding windows of N frames with the ConvGRU state carried, keeps every window's output and a
slice of the carried forward state.  Seeds and Poisson rates are chosen so that every case's output peaks at 1e-2 or
more (at seed 0 / lam 0.3 the N = 5 output peaks at 2.6e-3, which would make a relative bar weak); the tests assert
that floor.
"""
import os
import sys
import types

import numpy as np
import torch
import torchvision

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(1, "/root/reference")

sys.modules["myutils.vis_events.matplotlib_plot_events"] = types.ModuleType("stub")
ext = types.ModuleType("_ext")
ext.dcn_v2_forward = lambda inp, w, b, off, m, kh, kw, sh, sw, ph, pw, dh, dw, dg: \
    torchvision.ops.deform_conv2d(inp, off, w, b, stride=(sh, sw), padding=(ph, pw), dilation=(dh, dw), mask=m)
sys.modules["_ext"] = ext

from models.model import DeepRecurrNet  # noqa: E402  (the reference)
from oracle import model_ref  # noqa: E402

OUT_FLOOR = 1e-2

CASES = [
    # name, N, seed, B, H, W, lam, n_windows, zero_offset_init
    ("n5a", 5, 16, 2, 32, 32, 0.4, 3, False),
    ("n5b", 5, 18, 2, 36, 44, 1.0, 2, False),    # padded to 40x48 and cropped back
    ("n7", 7, 14, 1, 24, 40, 1.0, 2, False),
    ("n9", 9, 11, 1, 32, 32, 1.0, 1, False),
    ("n5z", 5, 16, 1, 32, 40, 0.4, 2, True),     # conv_offset_mask zero-initialised like the shipped model
]


def make_input(seed, B, N, H, W, lam, n_windows):
    g = torch.Generator().manual_seed(2000 + seed)
    return torch.poisson(torch.full((B, n_windows + N - 1, 2, H, W), lam), generator=g)


def case_state_dict(seed, N, zero_off):
    sd = model_ref.seeded_state_dict(seed, num_frame=N)
    if zero_off:
        sd = {k: (torch.zeros_like(v) if "conv_offset_mask" in k else v) for k, v in sd.items()}
    return sd


def main():
    torch.manual_seed(0)
    torch.set_num_threads(8)
    out = {"cases": np.array([c[0] for c in CASES])}
    for name, N, seed, B, H, W, lam, nwin, zero_off in CASES:
        sd = case_state_dict(seed, N, zero_off)
        net = DeepRecurrNet(inch=2, basech=8, num_frame=N)
        assert list(net.state_dict().keys()) == list(sd.keys()), "state_dict key order differs from the reference"
        net.load_state_dict(sd)
        net.eval()
        frames = make_input(seed, B, N, H, W, lam, nwin)
        outs = []
        with torch.no_grad():
            net.reset_states()
            for wdx in range(nwin):
                outs.append(net(frames[:, wdx:wdx + N].contiguous()).clone())
            state_fwd = net.time_propagate.states[0].clone()
        peak = max(o.abs().max().item() for o in outs)
        assert peak >= OUT_FLOOR, f"{name}: output peaks at {peak:.3g} < {OUT_FLOOR}; pick another seed / lam"
        out[f"{name}_meta"] = np.array([seed, B, H, W, nwin, int(zero_off), N])
        out[f"{name}_lam"] = np.array(lam)
        out[f"{name}_out"] = torch.stack(outs).numpy()
        out[f"{name}_state_fwd"] = state_fwd.numpy()[:, :4]   # a slice of the carried state
        o = model_ref.OracleNet(sd)                            # cross-check the restatement right here
        for wdx in range(nwin):
            err = (o(frames[:, wdx:wdx + N]) - outs[wdx]).abs().max().item()
            print(name, wdx, "oracle vs reference max abs err", err, "ref max", outs[wdx].abs().max().item())
    path = os.path.join(HERE, "model_nf_golden.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path))


if __name__ == "__main__":
    main()
