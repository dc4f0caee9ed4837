"""Generate tests/golden/infer_golden.npz by running the REFERENCE's own infer_ours_cnt.main() on the CPU (build container
only; needs /root/reference, oracle/_ref (python oracle/build_ref.py) and cv2).

infer_ours_cnt.py is imported unmodified and main() runs with sys.argv set to each case, relative paths under a scratch
working directory.  Stubs:
  * h5py: the in-memory stand-in of make_golden_index.py, holding seeded synthetic columns and grey or BGR `ori_images`
    (make_golden_frames.py's frames); cv2.resize is OpenCV's own;
  * the `_ext` DCNv2 operator as torchvision's deform_conv2d (make_golden_eval.py);
  * myutils.vis_events.matplotlib_plot_events: an event_visualisation that keeps the arrays plot_frame / plot_event_cnt
    receive, and a `plt` whose close does nothing;
  * thop, and `loss`: perceptual_loss returns the mean absolute difference as a stand-in value (the values only have to be
    deterministic here; LPIPS itself is tested elsewhere), ssim_loss / psnr_loss are oracle/metrics.py's restatement of
    loss/restore.py (scikit-image is not installed);
  * MetricTracker restated without pandas (its in-place column writes fail under pandas' copy-on-write) with the frame's
    initial 0 in every column, so that `macs`, never updated, stays the integer 0 as in the original;
  * time.time in the script's namespace returns multiples of 2^-6 s, so `time` is exact in binary and the YAML stable;
  * torch.load maps to the CPU and .to('cuda...') stays on the CPU (the script's default --device is cuda:0).
The recordings' frames, columns and checkpoints are rebuilt by the tests from the seeds stored here.

Kept per case: argv, the dataloader_config passed to infer_body, the text of every inference*.yml (by relative path), and
every gt_img array plot_frame received (by its PNG's relative path).
"""
import os
import sys
import tempfile
import types

import cv2 as _cv2  # the real module, imported before make_golden_index replaces sys.modules["cv2"] with a stub
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)
import make_golden_index as mgi  # noqa: E402  (h5py / cv2 / matplotlib stubs, reference on sys.path)

sys.modules["cv2"].INTER_CUBIC = _cv2.INTER_CUBIC
sys.modules["cv2"].resize = _cv2.resize
sys.modules["myutils"].__path__ = ["/root/reference/myutils"]          # the real utils, stubbed visualisation
sys.modules["myutils.vis_events"].__path__ = []

import torch  # noqa: E402
import torch.nn as nn  # noqa: E402
import torchvision  # noqa: E402

from oracle import metrics as om  # noqa: E402
from oracle import model_ref  # noqa: E402

PLOTS = []


class event_visualisation:
    def plot_event_cnt(self, cnt, is_save=False, path=None, **kw):
        PLOTS.append(("cnt", path, np.array(cnt)))

    def plot_frame(self, img, is_save=False, path=None, **kw):
        PLOTS.append(("frame", path, np.array(img)))


plot = types.ModuleType("myutils.vis_events.matplotlib_plot_events")
plot.event_visualisation = event_visualisation
plot.plt = types.SimpleNamespace(close=lambda *a: None)
sys.modules[plot.__name__] = plot
thop = types.ModuleType("thop")
thop.profile = lambda *a, **k: (0, 0)
sys.modules["thop"] = thop


class perceptual_loss:
    def __init__(self, weight=1.0, net='alex', use_gpu=True, gpu_ids=[0]):
        pass

    def __call__(self, pred, target, normalize=True):
        return (pred - target).abs().mean()


class ssim_loss:
    def __call__(self, pred, tgt):
        return np.float64(om.ssim_loss(pred.numpy(), tgt.numpy()))


class psnr_loss:
    def __call__(self, pred, tgt):
        return np.float64(om.psnr_loss(pred.numpy(), tgt.numpy()))


loss = types.ModuleType("loss")
loss.perceptual_loss, loss.ssim_loss, loss.psnr_loss = perceptual_loss, ssim_loss, psnr_loss
loss.__path__ = []
sys.modules["loss"] = loss
ext = types.ModuleType("_ext")
ext.dcn_v2_forward = lambda inp, w, b, off, m, kh, kw, sh, sw, ph, pw, dh, dw, dg: \
    torchvision.ops.deform_conv2d(inp, off, w, b, stride=(sh, sw), padding=(ph, pw), dilation=(dh, dw), mask=m)
sys.modules["_ext"] = ext

import dataloader.h5dataset as h5ds  # noqa: E402

h5ds.EventRecognition = type("EventRecognition", (), {})
import infer_ours_cnt as ref  # noqa: E402  (the reference script)


class MetricTracker:
    """myutils/utils.py:85-106 without the pandas frame; reset writes 0 into every column as `values[:] = 0` does."""

    def __init__(self, keys, writer=None):
        self.writer, self.keys = writer, list(keys)
        self.reset()

    def reset(self):
        self.total, self.counts, self.average = dict.fromkeys(self.keys, 0), dict.fromkeys(self.keys, 0), dict.fromkeys(self.keys, 0)

    def update(self, key, value, n=1):
        self.total[key] += value * n
        self.counts[key] += n
        self.average[key] = self.total[key] / self.counts[key]

    def result(self):
        return dict(self.average)


ref.MetricTracker = MetricTracker
_clock = [1000.0]


def _time():
    _clock[0] += 2.0 ** -6
    return _clock[0]


ref.time = types.SimpleNamespace(time=_time)
_load, _tensor_to, _module_to = torch.load, torch.Tensor.to, nn.Module.to


def _cpu_load(f, map_location=None, **kw):
    return _load(f, map_location="cpu", **kw)


def _is_cuda(a):
    return (isinstance(a, torch.device) and a.type == "cuda") or (isinstance(a, str) and a.startswith("cuda"))


torch.load = _cpu_load
torch.Tensor.to = lambda self, *a, **k: self if a and _is_cuda(a[0]) else _tensor_to(self, *a, **k)
nn.Module.to = lambda self, *a, **k: self if a and _is_cuda(a[0]) else _module_to(self, *a, **k)
CONFIGS = []
_infer_body = ref.infer_body


def _logged_infer_body(dataloader_config, data_path, *a, **k):
    CONFIGS.append(repr(dataloader_config))
    return _infer_body(dataloader_config, data_path, *a, **k)


ref.infer_body = _logged_infer_body

SENSOR = (128, 192)                       # down16 8 x 12 input, down8 16 x 24 ground truth at the shipped scale 2
# recording name, seed, ori events, channels (grey / BGR frames), image count
# (down16 holds ori / 256 events: 11, 13 and 10 steps of 1024 events)
RECORDINGS = [("rec_a.h5", 61, 256 * 1024 * 11, 1, 12), ("rec_b.h5", 62, 256 * 1024 * 13, 3, 9),
              ("rec_c.h5", 63, 256 * 1024 * 10, 1, 7)]
SHIPPED = ["--model_path", "model.pth", "--data_list", "data.txt", "--infer_mode", "1", "--output_path", "out", "--scale", "2",
           "--seqn", "3", "--seql", "9", "--step_size", "1", "--time_bins", "1", "--ori_scale", "down16", "--mode", "events",
           "--window", "2048", "--sliding_window", "1024", "--need_gt_frame", "--need_gt_events"]


def without(argv, flag, n):
    """argv without `flag` and its n - 1 values."""
    i = argv.index(flag)
    return argv[:i] + argv[i + n:]


def replaced(argv, flag, value):
    i = argv.index(flag)
    return argv[:i + 1] + [value] + argv[i + 2:]


# name, argv, checkpoint (SEQN, weight seed)
CASES = [
    ("shipped", SHIPPED, (3, 5)),
    ("no_step", without(SHIPPED, "--step_size", 2), (3, 5)),
    ("seqn5", replaced(replaced(SHIPPED, "--seqn", "5"), "--model_path", "model5.pth"), (5, 16)),
    ("no_gt_frame", without(SHIPPED, "--need_gt_frame", 1), (3, 5)),
]


def frames(seed, n, shape):
    return np.random.default_rng(seed).integers(0, 256, (n, *shape), dtype=np.uint8)


def recording(name, seed, n_ori, C, n_img):
    cols = mgi.synth_columns(seed, SENSOR, n_ori, {"down8": 8, "down16": 16})
    t0, t1 = cols["down16"]["ts"][0], cols["down16"]["ts"][-1]
    image_ts = np.sort(np.random.default_rng(seed + 100).uniform(t0 + 0.1 * (t1 - t0), t0 + 0.9 * (t1 - t0), n_img))
    imgs = frames(seed + 200, n_img, SENSOR + ((3,) if C == 3 else ()))
    return cols, image_ts, imgs


def checkpoint_config(seqn):
    """The config a trainer checkpoint carries (config/train_ours_enfssyn.yml's model entry and SEQN)."""
    return {"SEQN": seqn, "SCALE": 2, "model": {"name": "DeepRecurrNet", "args": {"inch": 2, "basech": 8, "num_frame": seqn}},
            "experiment": "infer_golden"}


def main():
    torch.set_num_threads(8)
    out = {"names": np.array([c[0] for c in CASES]), "sensor": np.array(SENSOR),
           "recordings": np.array([r[0] for r in RECORDINGS]), "rec_meta": np.array([r[1:] for r in RECORDINGS], np.int64)}
    for name, seed, n_ori, C, n_img in RECORDINGS:
        cols, image_ts, imgs = recording(name, seed, n_ori, C, n_img)
        mgi.fake_file(name, cols, SENSOR, image_ts)
        for i in range(n_img):
            mgi._FILES[name].children["ori_images"].children["image{:09d}".format(i)].value = imgs[i]
    cwd = os.getcwd()
    for case, argv, (seqn, wseed) in CASES:
        with tempfile.TemporaryDirectory() as tmp:
            os.chdir(tmp)
            try:
                with open("data.txt", "w") as f:
                    f.write("".join(r[0] + "\n" for r in RECORDINGS))
                mp = argv[argv.index("--model_path") + 1]
                torch.save({"config": checkpoint_config(seqn), "model": {"name": "DeepRecurrNet",
                            "states": model_ref.seeded_state_dict(wseed, num_frame=seqn)}}, mp)
                CONFIGS.clear()
                PLOTS.clear()
                sys.argv = ["infer_ours_cnt.py"] + argv
                ref.main()                                     # its Logger_yaml objects are written as main returns
                ymls = []
                for d, _, fs in os.walk("out"):
                    ymls += [os.path.join(d, f) for f in fs if f.endswith(".yml")]
                ymls.sort()
                out[f"{case}_argv"] = np.array(argv)
                out[f"{case}_ckpt"] = np.array([seqn, wseed])
                out[f"{case}_config"] = np.array([CONFIGS[0]])
                assert all(c == CONFIGS[0] for c in CONFIGS)
                out[f"{case}_yml_paths"] = np.array(ymls)
                for k, p in enumerate(ymls):
                    with open(p) as f:
                        out[f"{case}_yml_{k}"] = np.array([f.read()])
                gts = [(p, a) for kind, p, a in PLOTS if kind == "frame"]
                out[f"{case}_gt_paths"] = np.array([p for p, _ in gts])
                for k, (_, a) in enumerate(gts):
                    out[f"{case}_gt_{k}"] = a
                print(f"{case}: {len(ymls)} yml, {len(gts)} gt_img, shapes {sorted(set(a.shape for _, a in gts))}")
            finally:
                os.chdir(cwd)
    p = os.path.join(HERE, "infer_golden.npz")
    np.savez_compressed(p, **out)
    print("wrote infer_golden.npz", os.path.getsize(p) // 1024, "KiB")


if __name__ == "__main__":
    main()
