"""Time LPIPS (esr_b200.lpips) against torch / cuDNN, alone and inside the evaluation loop.

    python tools/bench_lpips.py [--reps 5] [--recordings 27] [--out result.json]

  * LPIPS pairs/s at 180 x 320 and 720 x 1280: evaluation-shaped batches (esr, bicubic and gt count planes of n windows x 2
    channels, each plane repeated to 3 channels; 2 pairs per gt plane, gt's features computed once).
  * evaluate_recordings windows/s at the tools/bench_eval.py workload (27 recordings, 180 x 320 / 120 x 160 HR, B = 4
    chunks): without LPIPS, with esr_b200.lpips, and with the torch baseline in its place.
The baseline is torchvision's AlexNet features with the same (seeded) weights and the LPIPS head arithmetic in torch, fp32,
run with cuDNN TF32 off (fp32) and on (torch's cuDNN default for convolutions, what the reference's GPU run does).
Achieved TFLOP/s use the algorithmic FLOPs of AlexNet's five convolutions (flops_per_image); the share of the 989 TFLOP/s
dense BF16 figure of the H100 SXM data sheet is given for this project's kernels, whose split-bf16 products issue three
MMAs per multiply-add (so 1/3 of that figure is their ceiling).  Host clocks around work ending in a device synchronise,
best of --reps after a warm-up.  The card's name and power limit are read in the same run.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from esr_b200 import evaluate, lpips  # noqa: E402
from bench_eval import CONFIG, gpu_info, timed, write_recordings  # noqa: E402

PEAK_BF16 = 989e12


def flops_per_image(H, W):
    h1, w1 = (H - 7) // 4 + 1, (W - 7) // 4 + 1
    h2, w2 = (h1 - 3) // 2 + 1, (w1 - 3) // 2 + 1
    h3, w3 = (h2 - 3) // 2 + 1, (w2 - 3) // 2 + 1
    return 2 * (h1 * w1 * 64 * 363 + h2 * w2 * 192 * 1600 + h3 * w3 * (384 * 1728 + 256 * 3456 + 256 * 2304))


def seeded_weights(seed=0):
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for name, shape in lpips.ALEXNET_KEYS:
        if name.endswith("weight"):
            sd[name] = torch.randn(shape, generator=g) * (2.0 / (shape[1] * shape[2] * shape[3])) ** 0.5
        else:
            sd[name] = torch.rand(shape, generator=g) * 0.1
    heads = {k: torch.rand(shape, generator=g) * 0.1 for k, shape in lpips.LIN_KEYS}
    return sd, heads


class TorchLPIPS:
    """The baseline: torchvision AlexNet features (cuDNN) + LPIPS v0.1 heads in torch, fp32."""

    def __init__(self, sd, heads, tf32):
        import torchvision
        net = torchvision.models.alexnet()
        net.load_state_dict(sd, strict=False)
        self.features = net.features[:12].cuda().eval()
        self.heads = [heads[k].cuda() for k, _ in lpips.LIN_KEYS]
        self.shift = torch.tensor([-.030, -.088, -.188], device="cuda")[None, :, None, None]
        self.scale = torch.tensor([.458, .448, .450], device="cuda")[None, :, None, None]
        self.tf32 = tf32

    def feats(self, x):
        x = ((2 * x - 1) - self.shift) / self.scale
        out = []
        for i, layer in enumerate(self.features):
            x = layer(x)
            if i in (1, 4, 7, 9, 11):
                out.append(x / (torch.sqrt(torch.sum(x ** 2, dim=1, keepdim=True)) + 1e-10))
        return out

    def distances(self, imgs, pa, pb):
        prev = torch.backends.cudnn.allow_tf32
        torch.backends.cudnn.allow_tf32 = self.tf32
        try:
            with torch.no_grad():
                f = self.feats(imgs)
                d = 0
                for l, w in enumerate(self.heads):
                    d = d + F.conv2d((f[l][pa] - f[l][pb]) ** 2, w).mean([2, 3])
                return d.view(-1)
        finally:
            torch.backends.cudnn.allow_tf32 = prev

    def window_pairs(self, esr, bicubic, gt):
        n, C, H, W = esr.shape
        imgs = torch.cat([esr, bicubic, gt]).reshape(3 * n * C, 1, H, W).expand(-1, 3, -1, -1)
        k = torch.arange(n * C, device=esr.device)
        d = self.distances(imgs, torch.cat([2 * n * C + k, 2 * n * C + k]), torch.cat([k, n * C + k]))
        return d.double().view(2, n, C).mean(dim=2)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--recordings", type=int, default=27)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_lpips: needs a CUDA device")
    torch.cuda.set_device(0)
    sd, heads = seeded_weights()
    ours = lpips.LPIPS(sd, heads)
    base = {"torch fp32": TorchLPIPS(sd, heads, False), "torch tf32": TorchLPIPS(sd, heads, True)}
    res = {"gpu": gpu_info(), "lpips": [], "evaluate": []}
    rng = np.random.default_rng(0)
    for H, W, n in ((180, 320, 16), (720, 1280, 4)):       # n windows: 6 n planes, 4 n pairs
        planes = torch.from_numpy(rng.poisson(2.0, (6 * n, H, W)).astype(np.float32)).cuda()
        src = np.repeat(np.arange(6 * n), 3).reshape(-1, 3)
        k = np.arange(2 * n)
        pa, pb = np.concatenate([4 * n + k, 4 * n + k]), np.concatenate([k, 2 * n + k])
        n_pairs, n_img = len(pa), 6 * n
        fl = flops_per_image(H, W) * n_img
        t = timed(lambda: ours.distances(planes, src, pa, pb), a.reps)
        row = {"H": H, "W": W, "pairs": n_pairs, "images": n_img,
               "esr_b200": {"s": t, "pairs_per_s": n_pairs / t, "tflops": fl / t / 1e12, "share_of_989": fl / t / PEAK_BF16}}
        imgs = planes[:, None].expand(-1, 3, -1, -1)
        tpa, tpb = torch.as_tensor(pa, device="cuda"), torch.as_tensor(pb, device="cuda")
        for name, b in base.items():
            tb = timed(lambda: b.distances(imgs, tpa, tpb), a.reps)
            row[name] = {"s": tb, "pairs_per_s": n_pairs / tb, "tflops": fl / tb / 1e12}
        d_ours = ours.distances(planes, src, pa, pb)
        d_base = base["torch fp32"].distances(imgs, tpa, tpb).double()
        row["max_rel_diff_vs_torch_fp32"] = float(((d_ours - d_base).abs() / d_base.abs()).max())
        res["lpips"].append(row)

    from bench_eval import DeepRecurrNet, model_ref  # the evaluation workload's network and weights
    import tempfile
    net = DeepRecurrNet(inch=2, basech=8, num_frame=3)
    net.load_state_dict(model_ref.seeded_state_dict(0))
    net = net.cuda().eval()
    with tempfile.TemporaryDirectory() as d:
        stores = write_recordings(d, a.recordings)
        n_win = sum(len(evaluate._Recording(s, CONFIG, 3).windows) for s in stores)
        for label, lp in (("no LPIPS", None), ("esr_b200 LPIPS", ours), ("torch fp32 LPIPS", base["torch fp32"]),
                          ("torch tf32 LPIPS", base["torch tf32"])):
            t = timed(lambda: evaluate.evaluate_recordings(net, stores, CONFIG, batch=4, lpips=lp), max(1, a.reps // 2))
            res["evaluate"].append({"config": label, "seconds": t, "windows_per_s": n_win / t})
        res["windows"] = n_win
    print(f"{res['gpu']}")
    for r in res["lpips"]:
        o = r["esr_b200"]
        print(f"  LPIPS {r['H']} x {r['W']}, {r['pairs']} pairs / {r['images']} images: esr_b200 {o['pairs_per_s']:.1f} pairs/s "
              f"({o['tflops']:.1f} TFLOP/s, {100 * o['share_of_989']:.1f} % of 989), torch fp32 {r['torch fp32']['pairs_per_s']:.1f}, "
              f"torch tf32 {r['torch tf32']['pairs_per_s']:.1f}; max rel diff vs torch fp32 {r['max_rel_diff_vs_torch_fp32']:.1e}")
    for r in res["evaluate"]:
        print(f"  evaluate B=4 {r['config']:18s} {r['seconds']:8.3f} s  {r['windows_per_s']:8.1f} windows/s")
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
