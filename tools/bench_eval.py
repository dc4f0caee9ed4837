"""Time the GPU evaluation loop (esr_b200.evaluate) and the count-image renderer (esr_b200.render).

    python tools/bench_eval.py [--recordings 27] [--batches 4,8,16] [--reps 3] [--out result.json]

Writes synthetic recordings to EventStore files in a temporary directory: ENFS-like down16 inputs at two sensor sizes
(720 x 1280 -> 45 x 80 LR / 180 x 320 HR, and 480 x 640 -> 30 x 40 / 120 x 160), 40-110 dataset frames each, evaluated
with the shipped inference settings (scale 4, seql 9, step_size 1, seqn 3) and seeded weights.  It times:
  * batch 1, one window per model call (the reference's loop structure, on this project's kernels);
  * batched evaluation (forward_sequence chunks, slots refilled across recordings) at each B of --batches;
  * the renderer on a batch of 180 x 320 count images against the numpy restatement (tests/render_ref.py) on the CPU.
Wall times are host clocks around calls that end in a device synchronise, best of --reps after one warm-up run; they
include gathering and encoding the events, the metrics and their copy to the host, not image writing.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from esr_b200 import evaluate, render  # noqa: E402
from esr_b200.eventstore import EventStore  # noqa: E402
from esr_b200.model import DeepRecurrNet  # noqa: E402
from oracle import model_ref  # noqa: E402
from tests import render_ref  # noqa: E402

WINDOW, SLIDING = 512, 256                     # 256 input events per dataset frame
CONFIG = dict(scale=4, ori_scale="down16", time_bins=1, need_gt_frame=False, need_gt_events=True, mode="events",
              window=WINDOW, sliding_window=SLIDING, data_augment=dict(enabled=False), hot_filter=dict(enabled=False),
              sequence=dict(sequence_length=9, seqn=3, step_size=1, pause=dict(enabled=False)))


def write_recordings(d, n, seed=0):
    rng = np.random.default_rng(seed)
    stores = []
    for i in range(n):
        sensor = (720, 1280) if i % 3 else (480, 640)
        length = int(rng.integers(40, 111))
        cols = {}
        for prex, div, per in (("down16", 16, SLIDING), ("down4", 4, SLIDING * 16)):
            m = length * per + WINDOW * 16
            H, W = sensor[0] // div, sensor[1] // div
            cols[prex] = {"xs": rng.integers(0, W, m), "ys": rng.integers(0, H, m), "ts": np.sort(rng.random(m)) * 10.0,
                          "ps": rng.choice([-1.0, 1.0], m)}
        path = os.path.join(d, f"rec{i:02d}.esr")
        EventStore.write(path, cols, sensor)
        stores.append(EventStore(path))
    return stores


def timed(fn, reps):
    fn()                                       # warm-up: plans, workspaces, module loads
    best = float("inf")
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        best = min(best, time.perf_counter() - t0)
    return best


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()[0]
    except Exception:
        q = torch.cuda.get_device_name()
    return q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--recordings", type=int, default=27)
    ap.add_argument("--batches", default="4,8,16")
    ap.add_argument("--chunk", type=int, default=8)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_eval: needs a CUDA device")
    torch.cuda.set_device(0)
    net = DeepRecurrNet(inch=2, basech=8, num_frame=3)
    net.load_state_dict(model_ref.seeded_state_dict(0))
    net = net.cuda().eval()
    res = {"gpu": gpu_info(), "recordings": a.recordings, "chunk": a.chunk}
    with tempfile.TemporaryDirectory() as d:
        stores = write_recordings(d, a.recordings)
        n_win = sum(len(evaluate._Recording(s, CONFIG, 3).windows) for s in stores)
        res["windows"] = n_win
        rows = []

        def run(batch, consecutive):
            return lambda: evaluate.evaluate_recordings(net, stores, CONFIG, batch=batch, chunk=a.chunk, consecutive=consecutive)

        for label, batch, consecutive in [("B=1, one window per call", 1, False), ("B=1, chunks", 1, None)] + \
                                          [(f"B={b}, chunks", b, None) for b in map(int, a.batches.split(","))]:
            t = timed(run(batch, consecutive), a.reps)
            dev_ms = run(batch, consecutive)()[1]["time"]
            rows.append({"config": label, "seconds": t, "windows_per_s": n_win / t, "device_ms_per_window": dev_ms})
        res["evaluate"] = rows
    # renderer: 64 HR count images of 180 x 320
    rng = np.random.default_rng(1)
    cnt = rng.poisson(0.5, (64, 2, 180, 320)).astype(np.float32)
    dcnt = torch.from_numpy(cnt).cuda()
    t_gpu = timed(lambda: render.render_event_cnt(dcnt), max(a.reps, 10))
    t0 = time.perf_counter()
    render_ref.render(cnt[:8])
    t_np = (time.perf_counter() - t0) / 8 * 64
    res["render"] = {"images": 64, "H": 180, "W": 320, "gpu_s": t_gpu, "numpy_s": t_np, "gpu_planes_per_s": 128 / t_gpu,
                     "numpy_planes_per_s": 128 / t_np}
    print(f"{res['gpu']}: {n_win} windows in {a.recordings} recordings")
    for r in res["evaluate"]:
        print(f"  {r['config']:28s} {r['seconds']:8.3f} s  {r['windows_per_s']:9.1f} windows/s  {r['device_ms_per_window']:.3f} device ms/window")
    rr = res["render"]
    print(f"  render 180x320: GPU {rr['gpu_planes_per_s']:.0f} planes/s, numpy {rr['numpy_planes_per_s']:.1f} planes/s")
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
