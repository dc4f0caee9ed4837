"""Time `python -m esr_b200.infer` against evaluate_recordings alone on the same recordings.

    python tools/bench_infer.py [--recordings 16] [--reps 2] [--out result.json]

Writes synthetic recordings with BGR image frames to EventStore files in a temporary directory, at the shape of
scripts/infer_ours.sh (720 x 1280 sensor, down16 input 45 x 80, scale 2 -> down8 ground truth 90 x 160, window 2048 /
sliding 1024, seql 9, step_size 1, seqn 3), 30-60 dataset frames each, with seeded weights.  It times, as host wall
clocks around calls that end in a device synchronise (best of --reps after a warm-up):
  * evaluate_recordings alone: without images, and with the event images and gt_img written;
  * the command in this process (checkpoint load, checks, evaluation, PNGs, YAML), with and without --need_gt_frame;
  * with two or more GPUs, the command under torchrun --nproc_per_node 2 (process start-up included).
LPIPS is off (--no_lpips) because its weights are not shipped.  The card's name and power limit are read in the same run.
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from esr_b200 import evaluate, infer  # noqa: E402
from esr_b200.eventstore import EventStore  # noqa: E402
from esr_b200.model import DeepRecurrNet  # noqa: E402
from oracle import model_ref  # noqa: E402

SENSOR = (720, 1280)
ARGS = ["--infer_mode", "1", "--scale", "2", "--seqn", "3", "--seql", "9", "--step_size", "1", "--time_bins", "1",
        "--ori_scale", "down16", "--mode", "events", "--window", "2048", "--sliding_window", "1024", "--need_gt_events",
        "--no_lpips"]


def write_recordings(d, n, seed=0):
    rng = np.random.default_rng(seed)
    paths = []
    for i in range(n):
        length = int(rng.integers(30, 61))
        cols = {}
        for prex, div, per in (("down16", 16, 1024), ("down8", 8, 4096)):
            m = (length + 1) * per + 4 * 2048
            H, W = SENSOR[0] // div, SENSOR[1] // div
            cols[prex] = {"xs": rng.integers(0, W, m), "ys": rng.integers(0, H, m), "ts": np.sort(rng.random(m)) * 10.0,
                          "ps": rng.choice([-1.0, 1.0], m)}
        n_img = length // 2 + 2
        imgs = rng.integers(0, 256, (n_img, *SENSOR, 3), dtype=np.uint8)
        path = os.path.join(d, f"rec{i:02d}.esr")
        EventStore.write(path, cols, SENSOR, np.linspace(0.0, 10.0, n_img), imgs)
        paths.append(path)
    with open(os.path.join(d, "data.txt"), "w") as f:
        f.write("".join(p + "\n" for p in paths))
    return paths


def timed(fn, reps):
    fn()
    best = float("inf")
    for _ in range(reps):
        torch.cuda.synchronize()
        t = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        best = min(best, time.perf_counter() - t)
    return best


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                       text=True)
    return q.stdout.strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--recordings", type=int, default=16)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    torch.cuda.set_device(0)
    res = {"card": card(), "recordings": a.recordings}
    with tempfile.TemporaryDirectory() as d:
        paths = write_recordings(d, a.recordings)
        net = DeepRecurrNet(inch=2, basech=8, num_frame=3)
        net.load_state_dict(model_ref.seeded_state_dict(0))
        ckpt = os.path.join(d, "model.pth")
        torch.save({"config": {"SEQN": 3, "model": {"name": "DeepRecurrNet", "args": {"inch": 2, "basech": 8, "num_frame": 3}}},
                    "model": {"name": "DeepRecurrNet", "states": net.state_dict()}}, ckpt)
        net = net.cuda().eval()
        flags = ARGS + ["--need_gt_frame"]
        cfg = infer.dataloader_config(infer.get_flags(flags + ["--output_path", "x"]))["dataset"]
        stores = [EventStore(p) for p in paths]
        res["windows"] = int(sum(infer.window_counts(stores, cfg)))
        k = [0]

        def fresh():
            k[0] += 1
            out = os.path.join(d, f"o{k[0]}")
            shutil.rmtree(os.path.join(d, f"o{k[0] - 1}"), ignore_errors=True)
            return out

        res["evaluate_s"] = timed(lambda: evaluate.evaluate_recordings(net, stores, cfg, batch=8, chunk=8), a.reps)
        res["evaluate_images_s"] = timed(lambda: evaluate.evaluate_recordings(net, stores, cfg, batch=8, chunk=8, image_dir=fresh(),
                                                                              gt_img=True), a.reps)
        common = ["--model_path", ckpt, "--data_list", os.path.join(d, "data.txt")]
        res["command_gt_img_s"] = timed(lambda: infer.main(common + flags + ["--output_path", fresh()]), a.reps)
        res["command_no_gt_img_s"] = timed(lambda: infer.main(common + ARGS + ["--output_path", fresh()]), a.reps)
        if torch.cuda.device_count() >= 2:
            env = dict(os.environ, PYTHONPATH=ROOT)
            cmd = [sys.executable, "-m", "torch.distributed.run", "--standalone", "--nproc_per_node", "2", "-m", "esr_b200.infer"]
            res["command_2ranks_s"] = timed(lambda: subprocess.run(cmd + common + flags + ["--output_path", fresh()], env=env,
                                                                   check=True, capture_output=True), a.reps)
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f)


if __name__ == "__main__":
    main()
