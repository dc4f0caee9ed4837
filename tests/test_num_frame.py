"""CPU: DeepRecurrNet at num_frame = 5, 7, 9 (the config's SEQN).

The fp32 oracle against tests/golden/model_nf_golden.npz (the reference's own models/model.py at those num_frame,
tests/golden/make_golden_model_nf.py), the module's parameter inventory against the reference's, the packed-parameter
sizes of the C ABI, and the configurations that keep raising."""
import os

import numpy as np
import pytest
import torch

from oracle import model_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ["n5a", "n5b", "n7", "n9", "n5z"]
OUT_FLOOR = 1e-2      # every fixture's output peaks above this, so that a relative bar means something


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(ROOT, "tests", "golden", "model_nf_golden.npz"))


def golden_case(g, name):
    """-> (state_dict, frames [B, nwin + N - 1, 2, H, W], nwin, N) of fixture case `name`."""
    seed, B, H, W, nwin, zero_off, N = (int(v) for v in g[f"{name}_meta"])
    lam = float(g[f"{name}_lam"])
    sd = model_ref.seeded_state_dict(seed, num_frame=N)
    if zero_off:
        sd = {k: (torch.zeros_like(v) if "conv_offset_mask" in k else v) for k, v in sd.items()}
    gen = torch.Generator().manual_seed(2000 + seed)
    frames = torch.poisson(torch.full((B, nwin + N - 1, 2, H, W), lam), generator=gen)
    return sd, frames, nwin, N


def test_fixture_cases_cover_the_issue(golden):
    assert [str(n) for n in golden["cases"]] == NAMES
    metas = {n: [int(v) for v in golden[f"{n}_meta"]] for n in NAMES}
    assert metas["n5a"][1:5] == [2, 32, 32, 3] and metas["n5a"][6] == 5     # B = 2, 32x32, three windows
    assert metas["n5b"][2:4] == [36, 44] and metas["n5b"][6] == 5           # padded / cropped
    assert metas["n7"][1:5] == [1, 24, 40, 2] and metas["n7"][6] == 7
    assert metas["n9"][4] == 1 and metas["n9"][6] == 9
    assert metas["n5z"][5] == 1 and metas["n5z"][6] == 5                    # zero conv_offset_mask
    for n in NAMES:
        assert np.abs(golden[f"{n}_out"]).max(axis=(1, 2, 3, 4)).min() >= OUT_FLOOR, n


@pytest.mark.parametrize("name", NAMES)
def test_oracle_matches_reference_fixtures(golden, name):
    torch.set_num_threads(8)
    sd, frames, nwin, N = golden_case(golden, name)
    net = model_ref.OracleNet(sd)
    want = golden[f"{name}_out"]
    assert np.abs(want).max() >= OUT_FLOOR
    for w in range(nwin):
        got = net(frames[:, w:w + N]).numpy()
        assert got.shape == want[w].shape
        np.testing.assert_allclose(got, want[w], rtol=0, atol=2e-6 + 1e-5 * np.abs(want[w]).max())
    np.testing.assert_allclose(net.states[0].numpy()[:, :4], golden[f"{name}_state_fwd"], rtol=0, atol=1e-5)


@pytest.mark.parametrize("N", [5, 7, 9])
def test_module_has_the_reference_inventory(N):
    from esr_b200.model import DeepRecurrNet
    net = DeepRecurrNet(inch=2, basech=8, num_frame=N)
    sd = net.state_dict()
    want = model_ref.param_shapes(num_frame=N)
    assert list(sd.keys()) == list(want.keys())
    assert {k: tuple(v.shape) for k, v in sd.items()} == want
    assert tuple(sd["spacetime_fuse.dense_fusion.0.conv2d.weight"].shape) == (64, 64 * N, 3, 3)
    ref_sd = model_ref.seeded_state_dict(3, num_frame=N)                      # a reference-format state_dict loads
    net.load_state_dict(ref_sd)
    assert all(torch.equal(net.state_dict()[k], v) for k, v in ref_sd.items())


def test_param_bytes_grow_by_the_dense_fusion_weight():
    from esr_b200 import _lib, build
    build.build()
    L = _lib.lib()
    base = L.esr_net_param_bytes()
    assert L.esr_net_param_bytes_n(3) == base
    dn0 = lambda n: L.esr_conv_weight_bytes(64, 64 * n, 3)                   # noqa: E731  (its 256-byte alignment holds)
    assert dn0(3) % 256 == 0
    for n in (5, 7):
        assert L.esr_net_param_bytes_n(n) - base == dn0(n) - dn0(3), n
    for n in (1, 2, 4, 6):
        assert L.esr_net_param_bytes_n(n) == 0, n


@pytest.mark.parametrize("kw", [dict(num_frame=4), dict(num_frame=1), dict(num_frame=2), dict(num_frame=3, basech=16),
                                dict(num_frame=5, basech=16), dict(num_frame=5, norm="BN"), dict(num_frame=5, has_ltc=False)])
def test_unsupported_configurations_raise(kw):
    from esr_b200 import _lib
    from esr_b200.model import DeepRecurrNet
    args = dict(inch=2, basech=8)
    args.update(kw)
    try:
        net = DeepRecurrNet(**args)
    except Exception:                   # noqa: BLE001 -- a module that cannot even be built does not run either
        return
    with pytest.raises(_lib.ESRError):
        net._check_supported()


@pytest.mark.parametrize("N", [3, 5, 7, 9])
def test_supported_num_frames_pass_the_check(N):
    from esr_b200.model import DeepRecurrNet
    DeepRecurrNet(inch=2, basech=8, num_frame=N)._check_supported()
