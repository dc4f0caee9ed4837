"""BASELINE.json configs[4]: event->count scatter and count->event redistribution sweep, 1e5..1e8 events per chunk,
achieved GB/s against the measured HBM peak.  Algorithmic bytes (SURVEY 8d): scatter 12*n + 8*H*W per frame;
cnt2event 8*H*W + 16*E per sample (sort traffic not counted).  Prints one JSON line per point."""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from esr_b200 import encodings as enc          # noqa: E402
from esr_b200.expand import expand              # noqa: E402

dev = torch.device("cuda:0")
peak = 3350.0                                   # H100 SXM data sheet HBM3 GB/s; MEASURED_PEAKS.json overrides
try:
    peak = json.load(open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")))["hbm_gbs"]
except Exception:
    pass
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)


def timed(fn, reps=5):
    fn()
    ts = []
    for _ in range(reps):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return sorted(ts)[len(ts) // 2]


g = torch.Generator(device=dev).manual_seed(1)
for H in (256, 1024):
    for n in (10**5, 3 * 10**5, 10**6, 3 * 10**6, 10**7, 3 * 10**7, 10**8):
        xs = torch.randint(0, H, (n,), generator=g, device=dev).float()
        ys = torch.randint(0, H, (n,), generator=g, device=dev).float()
        ps = (torch.randint(0, 2, (n,), generator=g, device=dev) * 2 - 1).float()
        off = torch.tensor([0, n], dtype=torch.int64, device=dev)
        ms = timed(lambda: enc.encode_frames(xs, ys, ps, off, hr_size=(H, H), n_max_frame=n))
        b = 12 * n + 8 * H * H
        print(json.dumps({"op": "scatter_cnt", "grid": H, "events": n, "ms": ms, "GBps": b / ms / 1e6, "frac_hbm": b / ms / 1e6 / peak,
                          "Mev_per_s": n / ms / 1e3}), flush=True)
        del xs, ys, ps
    for E in (10**5, 10**6, 10**7, 10**8):
        lam = E / (2.0 * H * H)
        cnt = torch.poisson(torch.full((1, 2, H, H), lam, device=dev), generator=g)
        Et = int(cnt.sum().item())
        ms = timed(lambda: expand(cnt, 0, 0), reps=3)
        b = 8 * H * H + 16 * Et
        print(json.dumps({"op": "cnt2event", "grid": H, "events": Et, "ms": ms, "GBps": b / ms / 1e6, "frac_hbm": b / ms / 1e6 / peak,
                          "Mev_per_s": Et / ms / 1e3}), flush=True)
        del cnt
