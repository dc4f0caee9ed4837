"""GPU: esr_resize_frames_cubic against the numpy restatement (tests/frames_ref.py) bit for bit, and the image entries of
SequenceReader.load_batch and the datalist loader: the gt image of every window, flips, pauses, frame mode, and banks
identical with frames on and off."""
import copy
import random

import numpy as np
import pytest
import torch

from esr_b200 import eventstore, frames, loader
from esr_b200._lib import ESRError
from esr_b200.eventstore import EventStore, SequenceReader
from tests import frames_ref

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")

GEOMS = [((720, 1280), (90, 160), (45, 80)), ((480, 640), (60, 80), (960, 1280)), ((260, 346), (65, 87), (130, 173)),
         ((37, 53), (1, 1), (74, 106)), ((100, 7), (50, 3), (3, 50))]


@pytest.mark.parametrize("where", ["pinned", "device"])
@pytest.mark.parametrize("C", [1, 3])
@pytest.mark.parametrize("geom", GEOMS, ids=lambda g: f"{g[0][0]}x{g[0][1]}")
def test_kernel_equals_restatement(geom, C, where):
    (H, W), s0, s1 = geom
    rng = np.random.default_rng(H * 7 + C)
    imgs = rng.integers(0, 256, (3, H, W) + ((3,) if C == 3 else ()), dtype=np.uint8)
    t = torch.from_numpy(imgs)
    t = t.pin_memory() if where == "pinned" else t.to(DEV)
    index = np.array([2, 0, 1, 2], np.int64)
    flips = np.array([0, 1, 2, 3], np.int32)
    n = len(index)
    o0 = torch.full((n, *s0) + ((3,) if C == 3 else ()), -1.0, device=DEV)
    o1 = torch.full((n, *s1) + ((3,) if C == 3 else ()), -1.0, device=DEV)
    src = np.uint64(t.data_ptr()) + index.astype(np.uint64) * np.uint64(t[0].numel())
    frames.resize_frames(src, flips, frames.row_addresses(o0), frames.row_addresses(o1), (H, W, C), s0, s1, DEV)
    torch.cuda.synchronize()
    for i in range(n):
        for out, s in ((o0, s0), (o1, s1)):
            want = frames_ref.formatted_frame(imgs[index[i]], *s, flips=int(flips[i]))[0]
            np.testing.assert_array_equal(out[i].cpu().numpy(), want, err_msg=f"frame {i} -> {s}")


def _recording(rng, n_img, sensor, C, t_end=1.0):
    H, W = sensor
    cols = {}
    for prex, div in (("down4", 4), ("down2", 2)):
        h, w = round(H / div), round(W / div)
        n = 4000 if div == 4 else 16000
        cols[prex] = {"xs": rng.integers(0, w, n), "ys": rng.integers(0, h, n), "ts": np.sort(rng.uniform(0.0, t_end, n)),
                      "ps": rng.choice([-1.0, 1.0], n)}
    # the images span the middle of the recording: early windows take image 0, late ones are clamped to image n - 1
    image_ts = np.sort(rng.uniform(0.2 * t_end, 0.7 * t_end, n_img))
    images = rng.integers(0, 256, (n_img, H, W) + ((3,) if C == 3 else ()), dtype=np.uint8)
    return cols, image_ts, images


def _config(mode, need_gt_frame=True, augment=True, pause=True):
    return dict(scale=2, ori_scale="down4", time_bins=1, need_gt_frame=need_gt_frame, need_gt_events=True, mode=mode,
                window=0.05, sliding_window=0.0,
                data_augment=dict(enabled=augment, augment=["Horizontal", "Vertical", "Polarity"], augment_prob=[0.5, 0.5, 0.5]),
                sequence=dict(sequence_length=5, seqn=3, step_size=2,
                              pause=dict(enabled=pause, proba_pause_when_running=0.5, proba_pause_when_paused=0.7)))


def _want(store, rd, frames_idx, flips, key):
    """The reference's item entry for every frame of a batch, from the restatement."""
    idx = rd.index
    (H, W), (kH, kW) = idx.inp_res, idx.gt_res
    out = []
    for f, fl in zip(frames_idx, flips):
        if key == "frame":
            out.append(frames_ref.formatted_frame(store.images[f], kH, kW, int(fl)))
            continue
        a, b = idx.event_indices[f]
        g = frames_ref.gt_image_index(store.image_ts, store.columns[idx.inp_prex]["ts"], [a], [b])[0]
        assert g == idx.gt_image_indices[f]
        out.append(frames_ref.formatted_frame(store.images[g], *((kH, kW) if key == "gt_img" else (H, W)), int(fl)))
    return np.stack(out)


@pytest.mark.parametrize("where", ["pinned", "device"])
@pytest.mark.parametrize("mode", ["time", "frame"])
@pytest.mark.parametrize("C,sensor", [(3, (360, 640)), (1, (260, 346))], ids=["bgr", "grey346"])
def test_reader_frames_equal_restatement(tmp_path, C, sensor, mode, where):
    rng = np.random.default_rng(C + len(mode))
    cols, image_ts, images = _recording(rng, 24, sensor, C)
    path = EventStore.write(str(tmp_path / "r.esr"), cols, sensor, image_ts, images)
    store = EventStore(path)
    cfg = _config(mode)
    rd = SequenceReader(store, cfg, where)
    seqs = list(range(len(rd)))
    random.seed(5)
    wins = rd.load_batch(seqs)
    bank = wins[0]["bank"]
    frames_idx, _, gt_xf = eventstore.frame_plan(rd.last_decisions, seqs, rd.step_size)
    assert rd.last_decisions["paused"].any() and len(set(rd.last_decisions["flips"].tolist())) > 2
    B, L = len(seqs), rd.L
    keys = ("gt_img", "gt_inp_size_img") + (("frame",) if mode == "frame" else ())
    assert set(bank) == {"inp_cnt", "inp_scaled_cnt", "gt_cnt", *keys}
    if mode == "time":
        g = rd.index.gt_image_indices
        assert g.min() == 0 and g.max() == len(image_ts) - 1          # clamped at both ends
    for key in keys:
        want = _want(store, rd, frames_idx, gt_xf, key)
        got = bank[key].reshape(B * L, *want.shape[1:]).cpu().numpy()
        np.testing.assert_array_equal(got, want, err_msg=key)
        for w, win in enumerate(wins):
            assert torch.equal(win[key], bank[key][:, w:w + 3])
    # need_gt_frame off gives no gt images and the same count banks for the same decisions (need_gt_frame moves the
    # reference's last reseed, so load_batch would draw different ones: the loader takes them as given)
    (tmp_path / "dl.txt").write_text(path + "\n")
    dec = eventstore.draw_decisions(cfg, len(seqs), L, random.Random(9))
    banks = {}
    for on in (True, False):
        dl = loader.HDF5DataLoaderSequence(dict(use_ddp=False, path_to_datalist_txt=str(tmp_path / "dl.txt"), batch_size=B,
                                                shuffle=False, num_workers=0, pin_memory=where == "pinned", drop_last=False,
                                                dataset=_config(mode, need_gt_frame=on)))
        banks[on] = dl.load([(0, q) for q in seqs], dec)[0]["bank"]
    assert "gt_img" not in banks[False] and "gt_img" in banks[True] and (("frame" in banks[False]) == (mode == "frame"))
    for key in ("inp_cnt", "inp_scaled_cnt", "gt_cnt") + (("frame",) if mode == "frame" else ()):
        assert torch.equal(banks[False][key], banks[True][key]), key
    # a store without images gives today's output, unchanged
    if mode == "time":
        plain = EventStore(EventStore.write(str(tmp_path / "p.esr"), cols, sensor, image_ts))
        random.seed(5)
        pb = SequenceReader(plain, cfg, where).load_batch(seqs)[0]["bank"]
        assert set(pb) == {"inp_cnt", "inp_scaled_cnt", "gt_cnt"}
        for key in pb:
            assert torch.equal(pb[key], bank[key])


def test_loader_frames_equal_reader(tmp_path):
    rng = np.random.default_rng(11)
    sensor = (360, 640)
    paths = []
    for r, n_img in enumerate((20, 26, 23)):
        cols, image_ts, images = _recording(rng, n_img, sensor, 3)
        paths.append(EventStore.write(str(tmp_path / f"rec{r}.esr"), cols, sensor, image_ts, images))
    dl_path = tmp_path / "datalist.txt"
    dl_path.write_text("\n".join(paths) + "\n")
    ds_cfg = _config("time")
    for pin in (True, False):
        cfg = dict(use_ddp=False, path_to_datalist_txt=str(dl_path), batch_size=4, shuffle=True, num_workers=0, pin_memory=pin,
                   drop_last=False, dataset=ds_cfg)
        dl = loader.HDF5DataLoaderSequence(cfg)
        stores = [EventStore(p) for p in paths]
        readers = [SequenceReader(st, ds_cfg, "pinned" if pin else "device") for st in stores]
        batch = [(0, 1), (2, 0), (1, 3), (0, 0), (2, 2)]
        dec = eventstore.draw_decisions(ds_cfg, len(batch), 5, random.Random(3))
        got = dl.load(batch, dec)[0]["bank"]
        for b, (r, s) in enumerate(batch):
            one = {k: v[b:b + 1] for k, v in dec.items()}
            frames_idx, _, gt_xf = eventstore.frame_plan(one, [s], readers[r].step_size)
            for key in ("gt_img", "gt_inp_size_img"):
                want = _want(stores[r], readers[r], frames_idx, gt_xf, key)
                np.testing.assert_array_equal(got[key][b].cpu().numpy(), want, err_msg=f"{key} batch {b}")
    # a batch mixing recordings with and without images is refused
    cols, image_ts, _ = _recording(rng, 20, sensor, 3)
    paths.append(EventStore.write(str(tmp_path / "noimg.esr"), cols, sensor, image_ts))
    dl_path.write_text("\n".join(paths) + "\n")
    cfg = dict(use_ddp=False, path_to_datalist_txt=str(dl_path), batch_size=4, shuffle=False, num_workers=0, pin_memory=True,
               drop_last=False, dataset=copy.deepcopy(ds_cfg))
    dl = loader.HDF5DataLoaderSequence(cfg)
    dec = eventstore.draw_decisions(ds_cfg, 2, 5, random.Random(4))
    with pytest.raises(ESRError):
        dl.load([(0, 0), (3, 0)], dec)


# ---- against the reference's own SequenceDataset with real cv2 (tests/golden/frames_golden.npz) ---------------------------
from tests.test_frames import GOLD, golden_store  # noqa: E402


def _check_golden_bank(name, bank):
    for key in ("gt_img", "gt_inp_size_img", "frame"):
        if f"{name}_{key}" not in GOLD.files:
            assert key not in bank
            continue
        want = GOLD[f"{name}_{key}"]
        got = np.rint(bank[key].cpu().numpy().astype(np.float64) * 255).astype(np.int64)
        d = np.abs(got - want)
        if name == "odd346":          # 346 / 86 is not an integer factor: default cv2 takes IPP's path there (tests/frames_ref.py)
            assert d.max() <= 1 and (d > 0).mean() < 0.08, (key, (d > 0).mean())
        else:
            np.testing.assert_array_equal(got, want, err_msg=f"{name} {key}")


@pytest.mark.parametrize("where", ["pinned", "device"])
@pytest.mark.parametrize("name", [str(n) for n in GOLD["names"]])
def test_reader_frames_equal_reference(tmp_path, name, where):
    store, cfg = golden_store(name, tmp_path)
    rd = SequenceReader(store, cfg, where)
    random.seed(int(GOLD[f"{name}_rseed"][0]))
    wins = rd.load_batch(GOLD[f"{name}_seqs"].tolist())
    assert random.random() == float(GOLD[f"{name}_next"][0])
    frames_idx, _, gt_xf = eventstore.frame_plan(rd.last_decisions, GOLD[f"{name}_seqs"].tolist(), rd.step_size)
    np.testing.assert_array_equal(frames_idx, GOLD[f"{name}_index"].ravel())
    np.testing.assert_array_equal(rd.last_decisions["paused"], GOLD[f"{name}_paused"])
    if cfg["need_gt_frame"]:
        np.testing.assert_array_equal(rd.index.gt_image_indices[frames_idx], GOLD[f"{name}_gt_index"].ravel())
    np.testing.assert_array_equal(gt_xf & 3, GOLD[f"{name}_frame_flips"].ravel())
    _check_golden_bank(name, wins[0]["bank"])


@pytest.mark.parametrize("name", [str(n) for n in GOLD["names"]])
def test_loader_frames_equal_reference(tmp_path, name):
    store, cfg = golden_store(name, tmp_path)
    (tmp_path / "dl.txt").write_text(store.path + "\n")
    dl = loader.HDF5DataLoaderSequence(dict(use_ddp=False, path_to_datalist_txt=str(tmp_path / "dl.txt"), batch_size=2,
                                            shuffle=False, num_workers=0, pin_memory=True, drop_last=False, dataset=cfg))
    seqs = GOLD[f"{name}_seqs"].tolist()
    random.seed(int(GOLD[f"{name}_rseed"][0]))
    dec = eventstore.draw_decisions(cfg, len(seqs), GOLD[f"{name}_index"].shape[1])
    _check_golden_bank(name, dl.load([(0, s) for s in seqs], dec)[0]["bank"])
