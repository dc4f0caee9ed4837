"""Replay synthetic recordings through esr_b200.stream.EventStream and time it against super_resolve_recordings.

    python tools/bench_stream.py [--recordings 4] [--frames 64] [--window 2048] [--chunk 8] [--tail-bias 0.6] [--out result.json]

Two shapes: the shipped one (720 x 1280 at down16: 45 x 80 LR -> 90 x 160 HR, scale 2) and a 4x one (45 x 80 -> 180 x 320).
Recordings of --frames frames of --window events each (plus 100), uniform coordinates, seeded; seeded weights with the tail's
bias raised by --tail-bias, as tools/bench_superresolve.py does, so that windows emit events.  Pushes of 256 events, W and 16 W,
with a pull after every push.  Per shape and push size, after one warm-up replay:
  * sustained input events/s: all recordings replayed back to back (each a stream of its own, closed at its end), host clock
    from the first push to the last close; the GPU never waits for input, so this is the stream's own ceiling;
  * per-window latency: host clock from the start of the push (or close) that makes window i's last frame final -- frame
    m + (N - 1) // 2 for its middle frame m -- to the end of the pull that first returns window i; median and 99th percentile;
  * the offline ceiling: super_resolve_recordings on the same recordings (batch 4, chunk --chunk), host clock around the call,
    input events / s.
The card's name and power limit are read in the same run.  There is no CPU path: without a CUDA device the script exits.
"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from esr_b200 import superresolve as sr  # noqa: E402
from esr_b200.eventstore import EventStore  # noqa: E402
from esr_b200.model import DeepRecurrNet  # noqa: E402
from esr_b200.stream import EventStream  # noqa: E402
from oracle import model_ref  # noqa: E402
from tools.bench_superresolve import gpu_info  # noqa: E402

SENSOR, LR = (720, 1280), (45, 80)


def config(window, scale):
    return dict(scale=scale, ori_scale="down16", time_bins=1, need_gt_frame=False, need_gt_events=False, mode="events",
                window=window, sliding_window=0, data_augment=dict(enabled=False), hot_filter=dict(enabled=False),
                sequence=dict(sequence_length=3, seqn=3, step_size=1, pause=dict(enabled=False)))


def write_recordings(d, n, frames, window, seed=0):
    rng = np.random.default_rng(seed)
    stores = []
    for i in range(n):
        m = frames * window + 100
        cols = {"down16": {"xs": rng.integers(0, LR[1], m), "ys": rng.integers(0, LR[0], m),
                           "ts": np.sort(rng.random(m)) * 10.0, "ps": rng.choice([-1.0, 1.0], m)}}
        path = os.path.join(d, f"rec{i:02d}.esr")
        EventStore.write(path, cols, SENSOR)
        stores.append(EventStore(path))
    return stores


def replay(net, recs, scale, window, chunk, push):
    """-> (seconds, input events, output events, per-window latencies in seconds)"""
    N = net._cfg["num_frame"]
    lat, n_in, n_out = [], 0, 0
    torch.cuda.synchronize()
    start = time.perf_counter()
    for xs, ys, ts, ps in recs:
        s = EventStream(net, LR, scale, window, chunk=chunk)
        ready, seen = [], 0                                     # host clock at which window i became ready; windows timed
        cuts = list(range(0, len(ts), push)) + [None]           # None: close()
        for a in cuts:
            t0 = time.perf_counter()
            if a is None:
                out = s.close()
            else:
                s.push(xs[a:a + push], ys[a:a + push], ts[a:a + push], ps[a:a + push])
                out = s.pull()
            ready += [t0] * (max(s.frames - N + 1, 0) - len(ready))
            t1 = time.perf_counter()
            lat += [t1 - ready[i] for i in range(seen, s.windows_returned)]
            seen = s.windows_returned
            n_out += len(out["ts"])
        n_in += len(ts)
    torch.cuda.synchronize()
    return time.perf_counter() - start, n_in, n_out, np.asarray(lat)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--recordings", type=int, default=4)
    ap.add_argument("--frames", type=int, default=64)
    ap.add_argument("--window", type=int, default=2048)
    ap.add_argument("--chunk", type=int, default=8)
    ap.add_argument("--tail-bias", type=float, default=0.6)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_stream: needs a CUDA device")
    torch.cuda.set_device(0)
    W = a.window
    res = {"gpu": gpu_info(), "recordings": a.recordings, "frames": a.frames, "window": W, "chunk": a.chunk,
           "tail_bias": a.tail_bias, "rows": []}
    with tempfile.TemporaryDirectory() as d:
        stores = write_recordings(d, a.recordings, a.frames, W)
        recs = [[np.asarray(s.columns["down16"][c]) for c in ("xs", "ys", "ts", "ps")] for s in stores]
        for scale in (2, 4):
            sd = model_ref.seeded_state_dict(0)
            sd["tail.conv2d.bias"] = sd["tail.conv2d.bias"] + a.tail_bias
            net = DeepRecurrNet(inch=2, basech=8, num_frame=3)
            net.load_state_dict(sd)
            net = net.cuda().eval()
            outs = [os.path.join(d, f"sr_{i:02d}.esr") for i in range(len(stores))]
            sr.super_resolve_recordings(net, stores, config(W, scale), outs, batch=4, chunk=a.chunk)      # warm-up
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            rep = sr.super_resolve_recordings(net, stores, config(W, scale), outs, batch=4, chunk=a.chunk)
            torch.cuda.synchronize()
            offline = time.perf_counter() - t0
            n_in = sum(len(r[2]) for r in recs)
            n_sr = sum(r["events"] for r in rep)
            for push in (256, W, 16 * W):
                replay(net, recs[:1], scale, W, a.chunk, push)                                            # warm-up
                sec, n, n_out, lat = replay(net, recs, scale, W, a.chunk, push)
                assert n == n_in and n_out == n_sr, (n, n_in, n_out, n_sr)
                res["rows"].append({"lr": list(LR), "hr": [LR[0] * scale, LR[1] * scale], "push": push, "seconds": sec,
                                    "events_per_s": n / sec, "sr_events": n_out, "windows": len(lat),
                                    "latency_ms_median": 1e3 * float(np.median(lat)),
                                    "latency_ms_p99": 1e3 * float(np.percentile(lat, 99)),
                                    "offline_seconds": offline, "offline_events_per_s": n_in / offline})
    print(res["gpu"])
    print("| LR -> HR | push | input events/s | latency median / p99 (ms) | offline super_resolve_recordings events/s |")
    print("|---|---|---|---|---|")
    for r in res["rows"]:
        print(f"| {r['lr'][0]}x{r['lr'][1]} -> {r['hr'][0]}x{r['hr'][1]} | {r['push']} | {r['events_per_s'] / 1e6:.2f} M | "
              f"{r['latency_ms_median']:.2f} / {r['latency_ms_p99']:.2f} | {r['offline_events_per_s'] / 1e6:.2f} M |")
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
