"""Times the training iteration (esr_b200.train.train_step: zero_grad, reset_states, L-2 windows forward with carried
state, summed MSE, one backward, Adam amsgrad) on one GPU and prints one JSON line.  Optional kernel table through
torch.profiler (CUPTI) with --kernels FILE.  --deterministic sets torch.backends.cudnn.deterministic, as the reference
trainer's init_seeds does, so the iteration runs the bitwise-reproducible kernels (esr_b200.train.deterministic()).

    python tools/bench_train.py --workload cfg2 --steps 5 --warmup 2 [--deterministic] [--kernels train_kernels.txt]
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402  (workload table + synthetic weights)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="cfg2", choices=sorted(bench.WORKLOADS))
    ap.add_argument("--batch", type=int, default=None)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--kernels", default=None)
    ap.add_argument("--deterministic", action="store_true")
    args = ap.parse_args()
    torch.backends.cudnn.deterministic = args.deterministic
    from esr_b200 import train
    from esr_b200.model import DeepRecurrNet

    wl = bench.WORKLOADS[args.workload]
    B, L, scale = args.batch or wl["B"], wl["L"], wl["scale"]
    H, W = wl["lr"][0] * scale, wl["lr"][1] * scale
    dev = torch.device("cuda", 0)
    net = DeepRecurrNet(inch=2, basech=8, num_frame=3)
    net.load_state_dict(bench.synth_weights(0))
    net = net.to(dev)
    opt = train.Adam(net.parameters(), lr=1e-3, weight_decay=1e-4, amsgrad=True)
    g = torch.Generator().manual_seed(0)
    frames = torch.poisson(torch.full((B, L, 2, H, W), 0.1), generator=g).to(dev)
    gt = torch.poisson(torch.full((B, L, 2, H, W), 0.1), generator=g).to(dev)

    def phases():
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        opt.zero_grad()
        net.reset_states()
        ev[0].record()
        pred = net(frames)                                      # all windows in one graph (window-major)
        loss = (L - 2) * train.mse_loss(pred, gt[:, 1:L - 1].transpose(0, 1).reshape(pred.shape))
        ev[1].record()
        loss.backward()
        ev[2].record()
        opt.step()
        ev[3].record()
        torch.cuda.synchronize()
        return [ev[i].elapsed_time(ev[i + 1]) for i in range(3)], loss.item()

    for _ in range(args.warmup):
        phases()
    acc, losses = [0.0, 0.0, 0.0], []
    for _ in range(args.steps):
        p, l = phases()
        acc = [a + b for a, b in zip(acc, p)]
        losses.append(l)
    fwd, bwd, step = (a / args.steps for a in acc)
    tot = fwd + bwd + step
    out = {"metric": "training LR event-frames/sec (fwd + bwd + Adam)", "value": B * L / (tot * 1e-3), "unit": "frames/s",
           "ms_per_step": tot, "forward_ms": fwd, "backward_ms": bwd, "optimizer_ms": step, "steps": args.steps,
           "config": {"workload": args.workload, "B": B, "L": L, "hr": [H, W],
                                                                   "deterministic": args.deterministic},
           "device": torch.cuda.get_device_name(dev), "loss_first": losses[0], "loss_last": losses[-1],
           "peak_mem_gb": torch.cuda.max_memory_allocated() / 2 ** 30}
    # the same iteration replayed from one CUDA graph
    gstep = train.GraphedTrainStep(net, opt, tuple(frames.shape), dev)
    for _ in range(args.warmup):
        gstep(frames, gt)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(args.steps):
        gstep(frames, gt)
    e1.record()
    torch.cuda.synchronize()
    gms = e0.elapsed_time(e1) / args.steps
    out["graph_ms_per_step"] = gms
    out["graph_value"] = B * L / (gms * 1e-3)
    print(json.dumps(out))
    if args.kernels:
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
            phases()
        with open(args.kernels, "w") as f:
            f.write(prof.key_averages().table(sort_by="cuda_time_total", row_limit=40, max_name_column_width=70))


if __name__ == "__main__":
    main()
