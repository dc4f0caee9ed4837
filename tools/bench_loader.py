"""SequenceReader.load_batch with the training config's flips (and optionally pauses) against the same reader with
augmentation off, alternating in one run at the cfg2 input (B = 8 sequences x L = 8 frames, 128 x 128 LR, 2x SR, the
shipped config's window of 2048 events).  Synthetic columns in a temporary EventStore, resident in pinned memory or HBM.
Prints one JSON line with the card's name and power limit.
    python tools/bench_loader.py [--where pinned|device] [--rounds 20] [--batches 10] [--pause]"""
import argparse
import copy
import json
import os
import random
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    name, limit = torch.cuda.get_device_name(), None
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        limit = float(r.stdout.strip().splitlines()[0])
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        pass
    return name, limit


def synth_store(path, sensor, n_lr, rng):
    """down2 (LR) and ori (HR, 4x the events) columns: int16 x / y, sorted float64 t, +-1 p."""
    cols = {}
    for prex, div, n in (("down2", 2, n_lr), ("ori", 1, 4 * n_lr)):
        H, W = sensor[0] // div, sensor[1] // div
        cols[prex] = {"xs": rng.integers(0, W, n).astype(np.int16), "ys": rng.integers(0, H, n).astype(np.int16),
                      "ts": np.sort(rng.random(n)) * 20.0, "ps": rng.choice([-1.0, 1.0], n)}
    from esr_b200.eventstore import EventStore
    EventStore.write(path, cols, sensor)
    return EventStore(path)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--where", default="pinned", choices=["pinned", "device"])
    ap.add_argument("--rounds", type=int, default=20)
    ap.add_argument("--batches", type=int, default=10, help="load_batch calls per timed round")
    ap.add_argument("--pause", action="store_true", help="also enable sequence.pause in the augmented reader")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_loader measures the GPU reader: no CUDA device"
    from esr_b200 import eventstore as es
    B, L = 8, 8
    cfg = dict(scale=2, ori_scale="down2", time_bins=1, need_gt_events=True, need_gt_frame=False, mode="events", window=2048,
               sliding_window=1024,
               data_augment=dict(enabled=True, augment=["Horizontal", "Vertical", "Polarity"], augment_prob=[0.5, 0.5, 0.5]),
               sequence=dict(sequence_length=L, seqn=3, step_size=None,
                             pause=dict(enabled=args.pause, proba_pause_when_running=0.05, proba_pause_when_paused=0.9)))
    off = copy.deepcopy(cfg)
    off["data_augment"]["enabled"] = False
    off["sequence"]["pause"]["enabled"] = False
    rng = np.random.default_rng(0)
    with tempfile.TemporaryDirectory() as tmp:
        store = synth_store(os.path.join(tmp, "bench.esrc"), (256, 256), 1024 * 8 * 8 * 8 + 2048, rng)
        readers = {"augmented": es.SequenceReader(store, cfg, where=args.where), "plain": es.SequenceReader(store, off, where=args.where)}
        n_seq = len(readers["plain"])
        order = [rng.permutation(n_seq)[:B].tolist() for _ in range(args.batches)]
        random.seed(0)
        for rd in readers.values():                    # warm up both paths
            for seqs in order[:3]:
                rd.load_batch(seqs)
        torch.cuda.synchronize()
        times = {k: [] for k in readers}
        for r in range(args.rounds):
            for k in (("augmented", "plain") if r % 2 == 0 else ("plain", "augmented")):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for seqs in order:
                    readers[k].load_batch(seqs)
                torch.cuda.synchronize()
                times[k].append((time.perf_counter() - t0) / len(order) * 1e3)
    name, limit = card()
    res = {k: {"median_ms_per_batch": float(np.median(v)), "min_ms": float(np.min(v)), "max_ms": float(np.max(v))}
           for k, v in times.items()}
    print(json.dumps({"metric": "SequenceReader.load_batch ms per batch (inp_cnt + inp_scaled_cnt + gt_cnt banks)",
                      "batch": [B, L], "lr": [128, 128], "scale": 2, "window": 2048, "where": args.where, "pause": args.pause,
                      "rounds": args.rounds, "batches_per_round": args.batches, "results": res,
                      "augmented_over_plain": res["augmented"]["median_ms_per_batch"] / res["plain"]["median_ms_per_batch"],
                      "gpu": name, "power_limit_w": limit,
                      "note": "wall clock incl. host decisions, the one H2D copy of the frame tables, gathers and scatters; "
                              "alternating order per round"}))


if __name__ == "__main__":
    main()
