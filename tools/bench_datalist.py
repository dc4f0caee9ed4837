"""ms per batch of the datalist loader (HDF5DataLoaderSequence.load: one esr_encode_frames_multi launch per event stream for
a batch drawn across recordings) against the per-recording path (SequenceReader.load_batch once per recording in the batch,
banks joined with torch.cat), alternating in one process, with columns in pinned host memory and in HBM.

16 synthetic recordings of different lengths in temporary EventStore files, the training config's flips on, at two shapes:
  train: batch 2, SEQL 9, a 720 x 1280 sensor at down16 (45 x 80 LR), 2x SR (down8 ground truth), window 2048 / 1024;
  cfg2:  batch 8, L 8, 128 x 128 LR (256 x 256 sensor at down2), 2x SR, window 2048 / 1024.
Prints one JSON line with the card's name and power limit.
    python tools/bench_datalist.py [--rounds 20] [--batches 10]"""
import argparse
import json
import os
import random
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.bench_loader import card  # noqa: E402

SHAPES = {"train": dict(B=2, L=9, sensor=(720, 1280), lr="down16", gt="down8", div=16),
          "cfg2": dict(B=8, L=8, sensor=(256, 256), lr="down2", gt="ori", div=2)}
N_REC = 16


def write_recordings(tmp, shape, rng):
    from esr_b200.eventstore import EventStore
    paths = []
    for r in range(N_REC):
        n_lr = 1024 * shape["L"] * (4 + r % 4) + 2048
        cols = {}
        for prex, div, n in ((shape["lr"], shape["div"], n_lr), (shape["gt"], shape["div"] // 2, 4 * n_lr)):
            H, W = round(shape["sensor"][0] / div), round(shape["sensor"][1] / div)
            cols[prex] = {"xs": rng.integers(0, W, n).astype(np.int16), "ys": rng.integers(0, H, n).astype(np.int16),
                          "ts": np.sort(rng.random(n)) * 20.0, "ps": rng.choice([-1.0, 1.0], n)}
        paths.append(EventStore.write(os.path.join(tmp, f"rec{r}.esrc"), cols, shape["sensor"]))
    with open(os.path.join(tmp, "datalist.txt"), "w") as f:
        f.write("\n".join(paths) + "\n")
    return paths


def dataset_config(shape):
    return dict(scale=2, ori_scale=shape["lr"], time_bins=1, need_gt_events=True, need_gt_frame=False, mode="events", window=2048,
                sliding_window=1024,
                data_augment=dict(enabled=True, augment=["Horizontal", "Vertical", "Polarity"], augment_prob=[0.5, 0.5, 0.5]),
                sequence=dict(sequence_length=shape["L"], seqn=3, step_size=None,
                              pause=dict(enabled=False, proba_pause_when_running=0.05, proba_pause_when_paused=0.9)))


def bench_shape(name, shape, rounds, n_batches, rng):
    from esr_b200 import eventstore as es
    from esr_b200.loader import HDF5DataLoaderSequence
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        paths = write_recordings(tmp, shape, rng)
        ds = dataset_config(shape)
        for where in ("pinned", "device"):
            cfg = dict(use_ddp=False, path_to_datalist_txt=os.path.join(tmp, "datalist.txt"), batch_size=shape["B"], shuffle=True,
                       num_workers=0, pin_memory=where == "pinned", drop_last=True, dataset=ds)
            dl = HDF5DataLoaderSequence(cfg)
            readers = [es.SequenceReader(es.EventStore(p), ds, where) for p in paths]
            counts = [len(d) for d in dl.dataset.datasets]
            pairs = [(r, s) for r, c in enumerate(counts) for s in range(c)]
            order = [[pairs[i] for i in rng.permutation(len(pairs))[:shape["B"]]] for _ in range(n_batches)]

            def multi():
                for batch in order:
                    dl.load(batch, es.draw_decisions(ds, len(batch), shape["L"]))

            def per_recording():
                for batch in order:
                    by_rec = {}
                    for r, s in batch:
                        by_rec.setdefault(r, []).append(s)
                    parts = [readers[r].load_batch(seqs)[0]["bank"] for r, seqs in by_rec.items()]
                    bank = {k: torch.cat([p[k] for p in parts]) for k in parts[0]}
                    N = 3
                    _ = [dict({k: v[:, w:w + N] for k, v in bank.items()}, bank=bank) for w in range(shape["L"] - N + 1)]

            paths_fn = {"multi": multi, "per_recording": per_recording}
            random.seed(0)
            for fn in paths_fn.values():                 # warm up both paths
                fn()
            torch.cuda.synchronize()
            times = {k: [] for k in paths_fn}
            for r in range(rounds):
                for k in (("multi", "per_recording") if r % 2 == 0 else ("per_recording", "multi")):
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    paths_fn[k]()
                    torch.cuda.synchronize()
                    times[k].append((time.perf_counter() - t0) / n_batches * 1e3)
            res = {k: {"median_ms_per_batch": float(np.median(v)), "min_ms": float(np.min(v)), "max_ms": float(np.max(v))}
                   for k, v in times.items()}
            mem = dl.memory_bytes()
            res["per_recording_over_multi"] = res["per_recording"]["median_ms_per_batch"] / res["multi"]["median_ms_per_batch"]
            res["bytes_per_recording"] = {k: v / N_REC for k, v in mem.items()}
            res["lr"], res["hr"] = dl.inp_sensor_resolution, dl.gt_sensor_resolution
            out[where] = res
            del dl, readers
            torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=20)
    ap.add_argument("--batches", type=int, default=10, help="batches per timed round")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_datalist measures the GPU loader: no CUDA device"
    rng = np.random.default_rng(0)
    results = {name: dict(batch=[s["B"], s["L"]], **bench_shape(name, s, args.rounds, args.batches, rng)) for name, s in SHAPES.items()}
    name, limit = card()
    print(json.dumps({"metric": "ms per batch: HDF5DataLoaderSequence.load vs SequenceReader.load_batch per recording + torch.cat",
                      "recordings": N_REC, "flips": True, "rounds": args.rounds, "batches_per_round": args.batches,
                      "results": results, "gpu": name, "power_limit_w": limit,
                      "note": "wall clock incl. host decisions, descriptor copies and launches; alternating order per round"}))


if __name__ == "__main__":
    main()
