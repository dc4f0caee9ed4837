"""S live streams through one esr_b200.stream.EventStreamPool against S EventStreams on S model objects, in one process.

    python tools/bench_stream_pool.py [--streams 1,4,16,64] [--frames 32] [--window 2048] [--slots 16] [--chunk 8]
                                      [--tail-bias 0.6] [--reps 2] [--out result.json]

Recordings and weights as tools/bench_stream.py makes them (45 x 80 LR at down16 of 720 x 1280, uniform coordinates, seeded;
seeded weights with the tail's bias raised by --tail-bias), at 45 x 80 -> 90 x 160 and -> 180 x 320, W = --window.  Per round
every stream pushes W events, then the pool runs one round (run()) and every stream is pulled; the separate streams are pushed
and pulled round-robin (each push runs its own windows).  After a warm-up of every call shape, the two are timed alternately,
--reps times each, for every S (the separate streams for S <= 16 only).  Reported per run:
  * aggregate input events/s: host clock from the first push to the last close;
  * per-window latency as in bench_stream.py: host clock from the start of the push that makes window i's last frame final to
    the end of the pull that first returns window i; median and 99th percentile;
  * per model call: host milliseconds (the call's Python, launches and its host synchronisation), the device span from CUDA
    events around the call, and the network's device time (CUDA events around forward_sequence);
  * the pool's plans and their total workspace, and the bytes per stream (ring and state row).
Also the round upload at S = 64, W events each: esr_events_append_rings reading the pinned buffer directly against one
host-to-device copy followed by the kernel reading device memory.  The card's name and power limit are read in the same run.
There is no CPU path: without a CUDA device the script exits.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from esr_b200 import _lib  # noqa: E402
from esr_b200.model import DeepRecurrNet  # noqa: E402
from esr_b200.stream import RING_DESC, EventStream, EventStreamPool  # noqa: E402
from oracle import model_ref  # noqa: E402
from tools.bench_stream import LR  # noqa: E402
from tools.bench_superresolve import gpu_info  # noqa: E402


def recordings(n, frames, window, seed=0):
    """bench_stream.write_recordings' columns, in memory"""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        m = frames * window + 100
        out.append([rng.integers(0, LR[1], m).astype(np.int16), rng.integers(0, LR[0], m).astype(np.int16),
                    np.sort(rng.random(m)) * 10.0, rng.choice([-1.0, 1.0], m)])
    return out


def model(tail_bias):
    sd = model_ref.seeded_state_dict(0)
    sd["tail.conv2d.bias"] = sd["tail.conv2d.bias"] + tail_bias
    net = DeepRecurrNet(inch=2, basech=8, num_frame=3)
    net.load_state_dict(sd)
    return net.cuda().eval()


class CallTimer:
    """Host ms, device span and network device time of every model call of the given pools"""

    def __init__(self, pools):
        self.rows, self.models = [], [p.model for p in pools]
        for p in pools:
            call, fwd = p._call, p.model.forward_sequence

            def timed_fwd(x, fwd=fwd):
                e = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
                e[0].record()
                out = fwd(x)
                e[1].record()
                self._net = e
                return out

            def timed_call(*a, call=call):
                e = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
                t = time.perf_counter()
                e[0].record()
                call(*a)
                e[1].record()
                self.rows.append((time.perf_counter() - t, e, self._net))

            p._call = timed_call
            p.model.forward_sequence = timed_fwd

    def summary(self):
        for m in self.models:
            m.__dict__.pop("forward_sequence", None)            # the class's method again
        torch.cuda.synchronize()
        host = np.array([r[0] for r in self.rows]) * 1e3
        span = np.array([r[1][0].elapsed_time(r[1][1]) for r in self.rows])
        net = np.array([r[2][0].elapsed_time(r[2][1]) for r in self.rows])
        return {"calls": len(self.rows), "host_ms_per_call": float(host.mean()), "device_span_ms_per_call": float(span.mean()),
                "network_ms_per_call": float(net.mean())}


def replay(recs, window, N, push_all, run_round, pull, close, frames_of, returned):
    """-> (seconds, input events, output events, latencies in seconds); stream k is recs[k]"""
    S = len(recs)
    ready, seen = [[] for _ in range(S)], [0] * S
    lat, n_out = [], 0
    rounds = max(len(r[2]) for r in recs) // window + 1
    torch.cuda.synchronize()
    start = time.perf_counter()
    for i in range(rounds + 1):
        t_push = [time.perf_counter()] * S
        for k, (xs, ys, ts, ps) in enumerate(recs):
            a = i * window
            t_push[k] = time.perf_counter()
            if i < rounds:
                push_all(k, xs[a:a + window], ys[a:a + window], ts[a:a + window], ps[a:a + window])
        if i < rounds:
            run_round()
        for k in range(S):
            if i < rounds:
                ready[k] += [t_push[k]] * (max(frames_of(k) - N + 1, 0) - len(ready[k]))
                out = pull(k)
            else:
                out, nf = close(k)
                ready[k] += [t_push[k]] * (max(nf - N + 1, 0) - len(ready[k]))
            t1 = time.perf_counter()
            r = returned(k)
            lat += [t1 - ready[k][j] for j in range(seen[k], r)]
            seen[k] = r
            n_out += len(out["ts"])
    torch.cuda.synchronize()
    return time.perf_counter() - start, sum(len(r[2]) for r in recs), n_out, np.asarray(lat)


def run_pool(net, recs, scale, a):
    pool = EventStreamPool(net, LR, scale, a.window, slots=a.slots, chunk=a.chunk, capacity=len(recs))
    timer = CallTimer([pool])
    sids = [pool.open() for _ in recs]
    st = {}

    def close(k):
        out, s = pool._close(sids[k])
        st[k] = s
        return out, s.n // a.window

    res = replay(recs, a.window, net._cfg["num_frame"], lambda k, *c: pool.push(sids[k], *c), pool.run,
                 lambda k: pool.pull(sids[k]), close, lambda k: pool.frames(sids[k]),
                 lambda k: st[k].returned if k in st else pool.windows_returned(sids[k]))
    return res, timer.summary()


def run_separate(nets, recs, scale, a):
    streams = [EventStream(n, LR, scale, a.window, chunk=a.chunk) for n in nets[:len(recs)]]
    timer = CallTimer([s._pool for s in streams])

    def close(k):
        out = streams[k].close()
        return out, streams[k].frames

    res = replay(recs, a.window, nets[0]._cfg["num_frame"], lambda k, *c: streams[k].push(*c), lambda: None,
                 lambda k: streams[k].pull(), close, lambda k: streams[k].frames, lambda k: streams[k].windows_returned)
    return res, timer.summary()


def upload_choice(S, window, reps=50):
    """esr_events_append_rings from pinned memory vs one H2D copy + the kernel from device memory; ms per round"""
    dev = torch.device("cuda")
    cap = 11 * window
    rings = [torch.zeros((S, cap), dtype=dt, device=dev) for dt in (torch.int16, torch.int16, torch.float64)]
    total = S * window
    host = torch.empty((12 * total,), dtype=torch.uint8).pin_memory()
    devbuf = torch.empty((12 * total,), dtype=torch.uint8, device=dev)
    desc = np.zeros(S, RING_DESC)
    for r in range(S):
        desc[r] = (*[v[r].data_ptr() for v in rings], cap, 5 * window + 7, window, r * window)
    desc_d = torch.from_numpy(desc.view(np.uint8)).to(dev)

    def cols(buf):
        T = total
        return buf[:2 * T].view(torch.int16), buf[2 * T:4 * T].view(torch.int16), buf[4 * T:].view(torch.float64)

    def append(buf):
        _lib.check(_lib.lib().esr_events_append_rings(_lib.ptr(desc_d), S, window, *map(_lib.ptr, cols(buf)), _lib.stream_ptr()),
                   "esr_events_append_rings")

    def direct():
        append(host)

    def copied():
        devbuf.copy_(host, non_blocking=True)
        append(devbuf)

    out = {}
    for name, fn in (("pinned_direct", direct), ("h2d_copy_then_kernel", copied)) * 2:
        fn()
        e = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        e[0].record()
        for _ in range(reps):
            fn()
        e[1].record()
        torch.cuda.synchronize()
        out.setdefault(name, []).append(e[0].elapsed_time(e[1]) / reps)
    return {"streams": S, "events": total, "bytes": 12 * total, **out}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", default="1,4,16,64")
    ap.add_argument("--frames", type=int, default=32)
    ap.add_argument("--window", type=int, default=2048)
    ap.add_argument("--slots", type=int, default=16)
    ap.add_argument("--chunk", type=int, default=8)
    ap.add_argument("--tail-bias", type=float, default=0.6)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_stream_pool: needs a CUDA device")
    torch.cuda.set_device(0)
    S_list = [int(s) for s in a.streams.split(",")]
    res = {"gpu": gpu_info(), "frames": a.frames, "window": a.window, "slots": a.slots, "chunk": a.chunk,
           "tail_bias": a.tail_bias, "rows": [], "upload": upload_choice(max(S_list), a.window)}
    recs = recordings(max(S_list), a.frames, a.window)
    warm = recordings(a.slots, a.chunk + 4, a.window, seed=1)
    for scale in (2, 4):
        kH, kW = LR[0] * scale, LR[1] * scale
        net = model(a.tail_bias)
        nets = [model(a.tail_bias) for _ in range(min(max(S_list), 16))]
        # warm-up: every call shape of the pool (B 1 .. slots, s 1 .. chunk) and of the separate streams
        for S in sorted({1 << i for i in range(a.slots.bit_length())} | {a.slots}):
            p = EventStreamPool(net, LR, scale, a.window, slots=a.slots, chunk=a.chunk, capacity=S)
            ids = [p.open() for _ in range(S)]
            for part in (slice(0, (a.chunk + 2) * a.window + 1), slice((a.chunk + 2) * a.window + 1, (a.chunk + 3) * a.window + 1)):
                for k, sid in enumerate(ids):                       # calls of chunk windows, then of one window
                    p.push(sid, *(c[part] for c in warm[k]))
                p.run()
            for sid in ids:
                p.close(sid)
        for n in nets:
            run_separate([n], warm[:1], scale, a)
        N = net._cfg["num_frame"]
        Bs = sorted({1 << i for i in range(a.slots.bit_length()) if 1 << i <= a.slots} | {a.slots})
        ss = [1 << i for i in range(a.chunk.bit_length())]
        ws = [_lib.lib().esr_net_workspace_bytes(B, N, s + N - 1, kH, kW) for B in Bs for s in ss]
        res.setdefault("plans", {})[f"{kH}x{kW}"] = {"count": len(ws), "workspace_mib": sum(ws) / 2**20,
                                                     "ring_bytes_per_stream": 12 * (a.chunk + N) * a.window,
                                                     "state_row_bytes": _lib.lib().esr_net_state_bytes(kH, kW)}
        for S in S_list:
            for rep in range(a.reps):
                modes = [("pool", lambda: run_pool(net, recs[:S], scale, a))]
                if S <= len(nets):
                    modes.append(("separate", lambda: run_separate(nets, recs[:S], scale, a)))
                for name, fn in modes:
                    (sec, n_in, n_out, lat), calls = fn()
                    res["rows"].append({"hr": [kH, kW], "streams": S, "mode": name, "rep": rep, "seconds": sec,
                                        "events_per_s": n_in / sec, "sr_events": n_out, "windows": len(lat),
                                        "latency_ms_median": 1e3 * float(np.median(lat)),
                                        "latency_ms_p99": 1e3 * float(np.percentile(lat, 99)), **calls})
    print(res["gpu"])
    print(json.dumps(res["plans"]))
    print(json.dumps(res["upload"]))
    print("| LR -> HR | S | mode | input events/s | latency median / p99 (ms) | calls | host ms / call | device span ms / call "
          "| network ms / call |")
    print("|---|---|---|---|---|---|---|---|---|")
    for r in res["rows"]:
        print(f"| {LR[0]}x{LR[1]} -> {r['hr'][0]}x{r['hr'][1]} | {r['streams']} | {r['mode']} | {r['events_per_s'] / 1e6:.2f} M | "
              f"{r['latency_ms_median']:.2f} / {r['latency_ms_p99']:.2f} | {r['calls']} | {r['host_ms_per_call']:.2f} | "
              f"{r['device_span_ms_per_call']:.2f} | {r['network_ms_per_call']:.2f} |")
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
