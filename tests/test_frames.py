"""CPU: the numpy restatement of cv2.resize(INTER_CUBIC) for uint8 frames (tests/frames_ref.py) against cv2 itself, the
event store's images section, and get_gt_frame's image index rule."""
import ast
import hashlib
import json
import os

import numpy as np
import pytest

from esr_b200.eventstore import HEADER_BYTES, EventStore
from tests import frames_ref

SWEEP = [((720, 1280), [(90, 160), (45, 80), (180, 320), (360, 640), (1440, 2560), (7, 13), (1, 1)]),
         ((480, 640), [(60, 80), (120, 160), (240, 320), (960, 1280), (1, 1)]),
         ((260, 346), [(65, 87), (130, 173), (260, 173), (130, 346), (52, 69), (520, 692), (1, 1)]),
         ((37, 53), [(18, 26), (9, 13), (74, 106), (1, 1)]),
         ((100, 7), [(50, 3), (25, 7), (200, 14), (1, 1)])]


def _cases():
    rng = np.random.default_rng(0)
    for (h, w), outs in SWEEP:
        for cn in (1, 3):
            img = rng.integers(0, 256, (h, w, cn) if cn == 3 else (h, w), dtype=np.uint8)
            for oh, ow in outs:
                yield img, oh, ow


def test_restatement_equals_opencv_generic_resize():
    """OpenCV's own resize code (IPP off) equals the restatement bit for bit over the sweep, downscaling and upscaling."""
    cv2 = pytest.importorskip("cv2")
    opt = cv2.useOptimized()
    cv2.setUseOptimized(False)
    try:
        for img, oh, ow in _cases():
            want = cv2.resize(img, (ow, oh), interpolation=cv2.INTER_CUBIC)
            got = frames_ref.resize_cubic_u8(img, oh, ow)
            if (oh, ow) in ((1440, 2560), (960, 1280), (520, 692), (74, 106), (200, 14)):
                # non-integer upscales: a handful of pixels (< 1e-4) land one level apart in OpenCV's vertical pass
                d = np.abs(want.astype(int) - got)
                assert d.max() <= 1 and (d > 0).mean() < 1e-4, (img.shape, oh, ow)
            else:
                np.testing.assert_array_equal(got, want, err_msg=f"{img.shape} -> {(oh, ow)}")
    finally:
        cv2.setUseOptimized(opt)


def test_restatement_within_one_level_of_default_cv2():
    """cv2 as the reference calls it (IPP where the build has it) is within one level everywhere, and equal at the
    training shapes (720 x 1280 -> 90 x 160 and 45 x 80, 480 x 640 -> 60 x 80)."""
    cv2 = pytest.importorskip("cv2")
    assert cv2.useOptimized()
    for img, oh, ow in _cases():
        want = cv2.resize(img, (ow, oh), interpolation=cv2.INTER_CUBIC)
        got = frames_ref.resize_cubic_u8(img, oh, ow)
        assert np.abs(want.astype(int) - got).max() <= 1, (img.shape, oh, ow)
        if img.shape[:2] in ((720, 1280), (480, 640)) and (oh, ow) in ((90, 160), (45, 80), (60, 80)):
            np.testing.assert_array_equal(got, want)


def test_flip_is_applied_before_the_resize():
    """The coefficients are not mirror-symmetric: flipping the output differs from resizing the flipped source."""
    rng = np.random.default_rng(3)
    img = rng.integers(0, 256, (60, 346), dtype=np.uint8)
    a = frames_ref.formatted_frame(img, 30, 87, flips=1)[0]
    b = np.flip(frames_ref.formatted_frame(img, 30, 87)[0], 1)
    assert not np.array_equal(a, b)
    assert a.dtype == np.float32 and a.max() <= 1.0


@pytest.mark.parametrize("shape", [(5, 12, 17), (4, 9, 14, 3)], ids=["grey", "bgr"])
def test_store_round_trip_with_images(tmp_path, shape):
    rng = np.random.default_rng(1)
    images = rng.integers(0, 256, shape, dtype=np.uint8)
    n = shape[0]
    cols = {"ori": {"xs": [1, 2, 3], "ys": [0, 1, 2], "ts": [0.0, 0.5, 1.0], "ps": [1.0, -1.0, 1.0]}}
    path = EventStore.write(str(tmp_path / "r.esr"), cols, shape[1:3], np.linspace(0, 1, n), images)
    st = EventStore(path)
    assert st.images.shape == shape and st.images.dtype == np.uint8
    np.testing.assert_array_equal(np.asarray(st.images), images)
    off = st.meta["images"][0]
    assert off % 4096 == 0 and off >= st.meta["image_ts"][0] + 8 * n
    np.testing.assert_array_equal(np.asarray(st.columns["ori"]["xs"]), [1, 2, 3])


def test_store_rejects_bad_images(tmp_path):
    from esr_b200._lib import ESRError
    cols = {"ori": {"xs": [1], "ys": [0], "ts": [0.0], "ps": [1.0]}}
    with pytest.raises(ESRError):
        EventStore.write(str(tmp_path / "a.esr"), cols, (4, 4), [0.0, 1.0], np.zeros((3, 4, 4), np.uint8))
    with pytest.raises(ESRError):
        EventStore.write(str(tmp_path / "b.esr"), cols, (4, 4), [0.0], np.zeros((1, 4, 4, 2), np.uint8))
    with pytest.raises(ESRError):
        EventStore.write(str(tmp_path / "c.esr"), cols, (4, 4), [0.0], np.zeros((1, 4, 4), np.float32))


def test_store_without_images_is_laid_out_as_before(tmp_path):
    """A file written without images has no images entry and ends where image_ts ends, as files written before the
    images section existed; it opens with images None."""
    cols = {"ori": {"xs": [1, 2], "ys": [0, 1], "ts": [0.0, 1.0], "ps": [1.0, -1.0]}}
    path = EventStore.write(str(tmp_path / "old.esr"), cols, (4, 4), [0.25, 0.75])
    with open(path, "rb") as f:
        raw = f.read()
    n = int.from_bytes(raw[8:12], "little")
    meta = json.loads(raw[12:12 + n].decode())
    assert set(meta) == {"sensor_resolution", "columns", "image_ts"}
    o, cnt = meta["image_ts"]
    assert len(raw) == max(o + 8 * cnt, HEADER_BYTES)
    st = EventStore(path)
    assert st.images is None
    np.testing.assert_array_equal(np.asarray(st.image_ts), [0.25, 0.75])


def test_gt_image_index_rule():
    """bisection at the middle input event, exact hits return the probed index, clamped to [0, n - 1]."""
    image_ts = np.array([1.0, 2.0, 3.0, 4.0])
    inp_ts = np.array([0.0, 0.5, 1.5, 2.0, 3.0, 3.5, 9.0, 10.0])
    idx0 = np.array([0, 2, 3, 4, 6, 0])
    idx1 = np.array([1, 2, 4, 6, 7, 7])
    # middles: 0 -> 0.0 (before all: 0), 2 -> 1.5 (1), 3 -> 2.0 (hit: 1), 5 -> 3.5 (3), 6 -> 9.0 (past the end: 3), 3 -> 2.0
    np.testing.assert_array_equal(frames_ref.gt_image_index(image_ts, inp_ts, idx0, idx1), [0, 1, 1, 3, 3, 1])


# ---- against the reference's own SequenceDataset with real cv2 (tests/golden/make_golden_frames.py) ----------------------
GOLD = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "frames_golden.npz"))
NAMES = [str(n) for n in GOLD["names"]]


def golden_frames(name):
    shape = tuple(GOLD[f"{name}_sensor"].tolist()) + ((3,) if int(GOLD[f"{name}_channels"][0]) == 3 else ())
    n = len(GOLD[f"{name}_image_ts"])
    imgs = np.random.default_rng(int(GOLD[f"{name}_frames_seed"][0])).integers(0, 256, (n, *shape), dtype=np.uint8)
    assert hashlib.sha256(imgs.tobytes()).hexdigest() == str(GOLD[f"{name}_frames_sha256"][0])
    return imgs


def golden_store(name, tmp_path):
    cols = {p: {k: GOLD[f"{name}_{p}_{k}"] for k in ("xs", "ys", "ts", "ps")} for p in ("down4", "down2")}
    path = EventStore.write(str(tmp_path / f"{name}.esr"), cols, GOLD[f"{name}_sensor"].tolist(), GOLD[f"{name}_image_ts"],
                            golden_frames(name))
    return EventStore(path), ast.literal_eval(str(GOLD[f"{name}_cfg"][0]))


@pytest.mark.parametrize("name", NAMES)
def test_gt_image_index_rule_against_reference(name):
    cfg = ast.literal_eval(str(GOLD[f"{name}_cfg"][0]))
    if not cfg["need_gt_frame"]:
        pytest.skip("no gt image")
    win = GOLD[f"{name}_win"].reshape(-1, 2)
    got = frames_ref.gt_image_index(GOLD[f"{name}_image_ts"], GOLD[f"{name}_down4_ts"], win[:, 0], win[:, 1])
    np.testing.assert_array_equal(got, GOLD[f"{name}_gt_index"].ravel())


@pytest.mark.parametrize("name", NAMES)
def test_restatement_against_reference(name):
    """The reference's entries rebuilt from its recorded image choices and flips with the restatement."""
    cfg = ast.literal_eval(str(GOLD[f"{name}_cfg"][0]))
    imgs = golden_frames(name)
    H, W = GOLD[f"{name}_sensor"].tolist()
    inp = (round(H / 4), round(W / 4))
    gt = (round(H / 2), round(W / 2))
    flips = GOLD[f"{name}_frame_flips"].ravel()
    entries = {"gt_img": (GOLD[f"{name}_gt_index"].ravel(), gt), "gt_inp_size_img": (GOLD[f"{name}_gt_index"].ravel(), inp),
               "frame": (GOLD[f"{name}_index"].ravel(), gt)}
    checked = 0
    for key, (idx, size) in entries.items():
        if f"{name}_{key}" not in GOLD.files:
            continue
        want = GOLD[f"{name}_{key}"].reshape(len(idx), *GOLD[f"{name}_{key}"].shape[2:]).astype(np.int64)
        got = np.stack([frames_ref.resize_cubic_u8(frames_ref.augment_frame(imgs[i], int(f)), *size)[None]
                        for i, f in zip(idx, flips)]).astype(np.int64)
        d = np.abs(got - want)
        if name == "odd346":          # a non-integer factor: default cv2 uses IPP's path, within one level
            assert d.max() <= 1
        else:
            np.testing.assert_array_equal(got, want, err_msg=key)
        checked += 1
    assert checked == 2 * cfg["need_gt_frame"] + (cfg["mode"] == "frame")
