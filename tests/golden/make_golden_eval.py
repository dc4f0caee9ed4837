"""Generate tests/golden/eval_golden.npz: the REFERENCE's evaluation loop body on synthetic recordings (build container only).

Needs /root/reference and oracle/_ref (python oracle/build_ref.py).  The reference's own SequenceDataset
(dataloader/h5dataset.py) reads seeded synthetic columns behind the in-memory h5py stand-in of make_golden_index.py;
InferenceHDF5DataLoaderSequence.custom_collate (dataloader/h5dataloader.py:289-312) builds the windows and window 0
(`inputs_seq[0]`) is evaluated, as infer_body does (infer_ours_cnt.py:55-101); the reference's DeepRecurrNet
(models/model.py, with the DCN stand-in of make_golden_model_nf.py) runs with `oracle.model_ref.seeded_state_dict`
weights and its state reset once per recording.  Per evaluated frame the fixture keeps esr, bicubic and gt[mid], the
dataset indices the window read (logged from H5Dataset.__getitem__), nn.L1Loss / nn.MSELoss, and ssim / psnr from
oracle/metrics.py (the restatement of loss/restore.py; scikit-image is not installed).

Cases (seql, step_size, seqn): (9, 1, 3), (9, None, 3), seql >= the dataset length (clamped to it), (9, 1, 5).
"""
import os
import sys
import types

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F
import torchvision

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE)
import make_golden_index as mgi  # noqa: E402  (stubs h5py / cv2 / matplotlib, puts the reference on sys.path)

sys.path.insert(0, ROOT)
sys.modules["cv2"].INTER_CUBIC = 2
sys.modules["cv2"].resize = lambda img, dsize, interpolation=None: np.zeros((dsize[1], dsize[0]), np.uint8)
sys.modules["myutils.vis_events.matplotlib_plot_events"] = types.ModuleType("stub")
ext = types.ModuleType("_ext")
ext.dcn_v2_forward = lambda inp, w, b, off, m, kh, kw, sh, sw, ph, pw, dh, dw, dg: \
    torchvision.ops.deform_conv2d(inp, off, w, b, stride=(sh, sw), padding=(ph, pw), dilation=(dh, dw), mask=m)
sys.modules["_ext"] = ext

import dataloader.h5dataset as _h5d  # noqa: E402  (the reference)
from dataloader.h5dataset import H5Dataset, SequenceDataset  # noqa: E402

_h5d.EventRecognition = None           # h5dataloader.py:17 imports a name h5dataset.py does not define
from dataloader.h5dataloader import InferenceHDF5DataLoaderSequence  # noqa: E402
from models.model import DeepRecurrNet  # noqa: E402
from oracle import metrics as om  # noqa: E402
from oracle import model_ref  # noqa: E402

SENSOR = (64, 96)                      # down4 input 16 x 24, down2 ground truth 32 x 48
CONFIG = dict(scale=2, ori_scale="down4", time_bins=1, need_gt_frame=False, need_gt_events=True, mode="events", window=160,
              sliding_window=40, data_augment=dict(enabled=False, augment=["Horizontal", "Vertical", "Polarity"],
                                                   augment_prob=[0.5, 0.5, 0.5]),
              hot_filter=dict(enabled=False, max_px=100, min_obvs=5, max_rate=0.8),
              sequence=dict(sequence_length=9, seqn=3, step_size=None,
                            pause=dict(enabled=False, proba_pause_when_running=0.05, proba_pause_when_paused=0.9)))
# name, seql, step_size, seqn, weight seed
CASES = [("s1n3", 9, 1, 3, 3), ("snone", 9, None, 3, 3), ("clamp", 40, None, 3, 3), ("s1n5", 9, 1, 5, 16)]

LOG = []
_getitem = H5Dataset.__getitem__


def _logged_getitem(self, index, Pause=False, seed=None):
    LOG.append(int(index))
    return _getitem(self, index, Pause=Pause, seed=seed)


H5Dataset.__getitem__ = _logged_getitem


def config(seql, step, seqn):
    c = {k: (dict(v) if isinstance(v, dict) else v) for k, v in CONFIG.items()}
    c["sequence"] = dict(CONFIG["sequence"], sequence_length=seql, step_size=step, seqn=seqn)
    return c


def main():
    torch.set_num_threads(8)
    cols = mgi.synth_columns(21, SENSOR, 20 * 120 * 16, {"down2": 2, "down4": 4})
    mgi.fake_file("/fake/eval.h5", cols, SENSOR, np.zeros(0))
    out = {"names": np.array([c[0] for c in CASES]), "sensor": np.array(SENSOR), "config": np.array([repr(CONFIG)])}
    for prex in ("down4", "down2"):
        for k, v in cols[prex].items():
            out[f"{prex}_{k}"] = v
    l1, mse = nn.L1Loss(), nn.MSELoss()
    for name, seql, step, seqn, wseed in CASES:
        cfg = config(seql, step, seqn)
        sd = SequenceDataset("/fake/eval.h5", cfg)
        loader = InferenceHDF5DataLoaderSequence.__new__(InferenceHDF5DataLoaderSequence)
        loader.seqn = seqn
        net = DeepRecurrNet(inch=2, basech=8, num_frame=seqn)
        net.load_state_dict(model_ref.seeded_state_dict(wseed, num_frame=seqn))
        net.eval()
        mid_idx = (seqn - 1) // 2
        rec = {k: [] for k in ("esr", "bicubic", "gt", "frames", "esr_l1", "esr_mse", "esr_ssim", "esr_psnr",
                               "bicubic_l1", "bicubic_mse", "bicubic_ssim", "bicubic_psnr")}
        with torch.no_grad():
            net.reset_states()
            for i in range(len(sd)):
                LOG.clear()
                inputs = loader.custom_collate([sd[i]])[0]
                rec["frames"].append(LOG[:seqn])
                inp_cnt = inputs["inp_cnt"][:, mid_idx]
                gt_cnt = inputs["gt_cnt"][:, mid_idx]
                esr = net(inputs["inp_scaled_cnt"])
                if esr.size()[-2:] != gt_cnt.size()[-2:]:
                    esr = F.interpolate(esr, size=gt_cnt.size()[-2:], mode="bicubic", align_corners=False)
                bic = F.interpolate(inp_cnt, size=sd.gt_sensor_resolution, mode="bicubic", align_corners=False)
                for pre, x in (("esr", esr), ("bicubic", bic)):
                    rec[pre].append(x[0].numpy())
                    rec[f"{pre}_l1"].append(l1(x, gt_cnt).item())
                    rec[f"{pre}_mse"].append(mse(x, gt_cnt).item())
                    rec[f"{pre}_ssim"].append(om.ssim_loss(x.numpy(), gt_cnt.numpy()))
                    rec[f"{pre}_psnr"].append(om.psnr_loss(x.numpy(), gt_cnt.numpy()))
                rec["gt"].append(gt_cnt[0].numpy())
        out[f"{name}_meta"] = np.array([seql, -1 if step is None else step, seqn, wseed, sd.dataset.length, len(sd)])
        for k, v in rec.items():
            out[f"{name}_{k}"] = np.array(v, dtype=np.int64 if k == "frames" else None)
        peak = np.abs(out[f"{name}_esr"]).max()
        print(f"{name}: dataset length {sd.dataset.length}, {len(sd)} windows, frames {out[name + '_frames'][:3].tolist()}..., "
              f"esr peak {peak:.3g}, esr l1 {np.mean(rec['esr_l1']):.4g} ssim {np.mean(rec['esr_ssim']):.4g}")
        assert peak >= 1e-2, f"{name}: esr peaks at {peak:.3g}"
    path = os.path.join(HERE, "eval_golden.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    main()
