"""DeepRecurrNet.forward_sequence at num_frame N = 3, 5 and 7 on the cfg2 input (B = 8 sequences x L = 9 frames, 128 x 128 LR
lifted to 256 x 256 for 2x SR), the three models built in one process and timed alternately with CUDA events; then one
GraphedTrainStep iteration at N = 3 and N = 5, also alternating.  Prints one JSON line with the card's name and power limit.
    python tools/bench_num_frame.py [--steps 20] [--warmup 3] [--rounds 5]

LR frames/s counts the B * L input frames of a sequence batch (bench.py's metric); a forward_sequence produces
B * (L - N + 1) SR frames, one per window."""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def _time(fn, steps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20, help="timed calls per round and model")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5, help="alternating rounds; the median over rounds is reported")
    ap.add_argument("--train-steps", type=int, default=10)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_num_frame measures the GPU plan: no CUDA device"
    from esr_b200 import _lib, train
    from esr_b200.model import DeepRecurrNet
    from oracle import model_ref
    from tools.bench_loader import card
    dev = torch.device("cuda:0")
    B, L, lr, scale = 8, 9, (128, 128), 2
    H, W = lr[0] * scale, lr[1] * scale
    g = torch.Generator().manual_seed(0)
    frames = torch.poisson(torch.full((B, L, 2, H, W), 0.1), generator=g).to(dev)
    gt = torch.poisson(torch.full((B, L, 2, H, W), 0.1), generator=g).to(dev)
    Ns = (3, 5, 7)
    nets = {}
    for N in Ns:
        net = DeepRecurrNet(inch=2, basech=8, num_frame=N)
        net.load_state_dict(model_ref.seeded_state_dict(0, num_frame=N))
        nets[N] = net.to(dev).eval()
    with torch.no_grad():
        for N in Ns:
            for _ in range(args.warmup):
                nets[N].forward_sequence(frames)
        torch.cuda.synchronize()
        ms = {N: [] for N in Ns}
        for r in range(args.rounds):
            for N in (Ns if r % 2 == 0 else Ns[::-1]):
                ms[N].append(_time(lambda: nets[N].forward_sequence(frames), args.steps))
    infer = {}
    for N in Ns:
        m, Wn = float(np.median(ms[N])), L - N + 1
        infer[str(N)] = {"ms_per_forward_sequence": m, "min_ms": float(np.min(ms[N])), "max_ms": float(np.max(ms[N])),
                         "windows": Wn, "ms_per_window": m / Wn, "lr_frames_per_s": B * L / (m * 1e-3),
                         "sr_frames_per_s": B * Wn / (m * 1e-3),
                         "workspace_bytes": int(_lib.lib().esr_net_workspace_bytes(B, N, L, H, W)),
                         "param_bytes": int(_lib.lib().esr_net_param_bytes_n(N))}
    del nets
    torch.cuda.empty_cache()

    steps = {}
    for N in (3, 5):
        net = DeepRecurrNet(inch=2, basech=8, num_frame=N)
        net.load_state_dict(model_ref.seeded_state_dict(0, num_frame=N))
        net = net.to(dev)
        opt = train.Adam(net.parameters(), lr=1e-4, weight_decay=1e-4, amsgrad=True)
        steps[N] = train.GraphedTrainStep(net, opt, tuple(frames.shape), dev)
    torch.cuda.synchronize()
    tms = {N: [] for N in steps}
    for r in range(args.rounds):
        for N in ((3, 5) if r % 2 == 0 else (5, 3)):
            tms[N].append(_time(lambda: steps[N](frames, gt), args.train_steps))
    trn = {str(N): {"ms_per_iteration": float(np.median(v)), "min_ms": float(np.min(v)), "max_ms": float(np.max(v)),
                    "lr_frames_per_s": B * L / (float(np.median(v)) * 1e-3)} for N, v in tms.items()}
    name, limit = card()
    print(json.dumps({"metric": "forward_sequence / GraphedTrainStep ms by num_frame", "batch": [B, L], "lr": list(lr),
                      "scale": scale, "steps": args.steps, "rounds": args.rounds, "inference": infer, "train": trn,
                      "gpu": name, "power_limit_w": limit,
                      "note": "CUDA events around --steps back-to-back calls per round; models alternate per round; median of rounds"}))


if __name__ == "__main__":
    main()
