"""Time esr_b200.superresolve end to end and its esr_events_to_columns kernel on its own.

    python tools/bench_superresolve.py [--recordings 27] [--batches 4,8,16] [--reps 3] [--tail-bias 0.6] [--out result.json]

Synthetic recordings as tools/bench_eval.py builds them (ENFS-like down16 inputs at 720 x 1280 -> 45 x 80 LR / 180 x 320 HR and
480 x 640 -> 30 x 40 / 120 x 160, 40-110 dataset frames each, 256 input events per frame), without a ground-truth stream and
with sliding_window 0, because overlapping frames are refused.  Seeded weights; --tail-bias shifts the last layer's bias so
that the SR counts are not almost all zero (the events per window that result are reported).  It times:
  * super_resolve_recordings at each B of --batches: host clock around the whole call, which ends with every file written
    (gather, encode, network, cnt2event, columns, collection in host memory, EventStore.write); best of --reps after a warm-up;
  * esr_events_to_columns alone on the rows of one 64-sample call at 180 x 320 with Poisson(1) counts (about 7.4 M events:
    its 36 B per event exceed the 50 MB L2, so repeated launches read and write HBM): CUDA events around --launches
    launches; to device memory, the bytes it moves (16 B read + 20 B written per event) over that time; to pinned host
    memory, the 20 B per event that cross the host link over that time.
The HBM figure it is compared with is the data sheet's 3.35 TB/s for an H100 SXM allowed 700 W, not a measured peak.
There is no CPU path: without a CUDA device the script exits with an error.
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

from esr_b200 import superresolve as sr  # noqa: E402
from esr_b200.eventstore import EventStore  # noqa: E402
from esr_b200.expand import expand_begin, expand_finish  # noqa: E402
from esr_b200.model import DeepRecurrNet  # noqa: E402
from oracle import model_ref  # noqa: E402

WINDOW = 256
CONFIG = dict(scale=4, ori_scale="down16", time_bins=1, need_gt_frame=False, need_gt_events=False, mode="events",
              window=WINDOW, sliding_window=0, data_augment=dict(enabled=False), hot_filter=dict(enabled=False),
              sequence=dict(sequence_length=9, seqn=3, step_size=1, pause=dict(enabled=False)))
HBM_DATASHEET = 3.35e12                       # bytes / s, H100 SXM at 700 W


def write_recordings(d, n, seed=0):
    rng = np.random.default_rng(seed)
    stores = []
    for i in range(n):
        sensor = (720, 1280) if i % 3 else (480, 640)
        m = int(rng.integers(40, 111)) * WINDOW + 16
        cols = {"down16": {"xs": rng.integers(0, sensor[1] // 16, m), "ys": rng.integers(0, sensor[0] // 16, m),
                           "ts": np.sort(rng.random(m)) * 10.0, "ps": rng.choice([-1.0, 1.0], m)}}
        path = os.path.join(d, f"rec{i:02d}.esr")
        EventStore.write(path, cols, sensor)
        stores.append(EventStore(path))
    return stores


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                       timeout=30)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name() + ", power limit unknown"


def bench_kernel(launches):
    """one large call's worth of rows: 64 windows of 180 x 320 with Poisson(1) counts"""
    dev = torch.device("cuda", torch.cuda.current_device())
    g = torch.Generator(device=dev).manual_seed(0)
    cnt = torch.poisson(torch.full((64, 2, 180, 320), 1.0, device=dev), generator=g)
    ctx = expand_begin(cnt, 0, 0)
    rows = expand_finish(ctx, 0).contiguous()
    n = len(ctx.ev)
    desc, total = sr.plan_segment(ctx.ev, np.arange(n, dtype=np.float64), np.arange(n, dtype=np.float64) + 0.5)
    desc_d = torch.from_numpy(desc.view(np.uint8)).to(dev)
    res = {"samples": n, "maxlen": int(rows.shape[1]), "events": total, "bytes": 36 * total, "launches": launches}
    for where in ("device", "pinned"):
        buf = torch.empty((20 * total,), dtype=torch.uint8, device=dev) if where == "device" else torch.empty((20 * total,), dtype=torch.uint8).pin_memory()
        cols = sr._segment_views(buf, total)
        for _ in range(10):
            sr.events_to_columns(rows, desc_d, int(ctx.ev.max()), *cols)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(launches):
            sr.events_to_columns(rows, desc_d, int(ctx.ev.max()), *cols)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / launches
        moved = 36 * total if where == "device" else 20 * total       # pinned: what crosses the host link
        res[where] = {"ms": ms, "bytes_per_s": moved / (ms * 1e-3), "events_per_s": total / (ms * 1e-3)}
    res["device"]["share_of_hbm_datasheet"] = res["device"]["bytes_per_s"] / HBM_DATASHEET
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--recordings", type=int, default=27)
    ap.add_argument("--batches", default="4,8,16")
    ap.add_argument("--chunk", type=int, default=8)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--launches", type=int, default=100)
    ap.add_argument("--tail-bias", type=float, default=0.6)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_superresolve: needs a CUDA device")
    torch.cuda.set_device(0)
    sd = model_ref.seeded_state_dict(0)
    sd["tail.conv2d.bias"] = sd["tail.conv2d.bias"] + a.tail_bias
    net = DeepRecurrNet(inch=2, basech=8, num_frame=3)
    net.load_state_dict(sd)
    net = net.cuda().eval()
    res = {"gpu": gpu_info(), "recordings": a.recordings, "chunk": a.chunk, "tail_bias": a.tail_bias, "end_to_end": []}
    with tempfile.TemporaryDirectory() as d:
        stores = write_recordings(d, a.recordings)
        outs = [os.path.join(d, "sr_" + os.path.basename(s.path)) for s in stores]
        for b in map(int, a.batches.split(",")):
            report = sr.super_resolve_recordings(net, stores, CONFIG, outs, batch=b, chunk=a.chunk)      # warm-up
            best = float("inf")
            for _ in range(a.reps):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                sr.super_resolve_recordings(net, stores, CONFIG, outs, batch=b, chunk=a.chunk)
                torch.cuda.synchronize()
                best = min(best, time.perf_counter() - t0)
            nw, ne = sum(r["windows"] for r in report), sum(r["events"] for r in report)
            res["end_to_end"].append({"batch": b, "seconds": best, "windows": nw, "events": ne, "windows_per_s": nw / best,
                                      "events_per_s": ne / best})
    res["kernel"] = bench_kernel(a.launches)
    print(res["gpu"])
    for r in res["end_to_end"]:
        print(f"  B={r['batch']:3d}: {r['windows']} windows, {r['events']} events in {r['seconds']:.3f} s  "
              f"{r['windows_per_s']:.1f} windows/s  {r['events_per_s'] / 1e6:.2f} M events/s (files written)")
    k = res["kernel"]
    print(f"  esr_events_to_columns, {k['events']} events in {k['samples']} samples of {k['maxlen']} rows: "
          f"device {k['device']['ms']:.4f} ms = {k['device']['bytes_per_s'] / 1e9:.0f} GB/s "
          f"({100 * k['device']['share_of_hbm_datasheet']:.1f}% of the data sheet's 3.35 TB/s), "
          f"pinned host {k['pinned']['ms']:.4f} ms = {k['pinned']['bytes_per_s'] / 1e9:.1f} GB/s written over the host link")
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
