"""numpy restatement of cv2.resize(img, (oW, oH), interpolation=cv2.INTER_CUBIC) for uint8 images, as OpenCV's generic
resize computes it (imgproc resize: interpolateCubic, HResizeCubic, VResizeCubic and its SIMD vertical pass
VResizeCubicVec_32s8u), and the dataset's frame formatting around it.  It is the reference the GPU kernel
(esr_resize_frames_cubic) is held to bit for bit.

What OpenCV does, step by step:
  * scale = 1. / (dst / src) in double; source position fx = (float)((d + 0.5) * scale - 0.5); sx = floor(fx), x = fx - sx;
  * coefficients: interpolateCubic's fp32 polynomials (A = -0.75, the fourth = 1 - c0 - c1 - c2), each rounded to nearest
    even at 2^11 (saturate_cast<short>);
  * taps sx - 1 .. sx + 2, clamped to the image (replicated border);
  * horizontal pass: exact int32 sums;
  * vertical pass: for the first floor(oW * C / 8) * 8 elements of a row, fp32 t = h3 * b3, then t = fma(h_k, b_k, t) for
    k = 2, 1, 0 with b_k = beta_k * 2^-22, rounded to nearest even; for the rest, (sum h_k * beta_k + 2^21) >> 22;
    saturated to uint8.
Where OpenCV is built with IPP (the opencv-python wheels), cv2.resize hands some geometries -- non-integer scale factors --
to IPP, whose result differs from this by at most one level on a few per cent of pixels; tests/test_frames.py holds that.
"""
import numpy as np


def cubic_taps(dst, src):
    """-> (tap indices int64 [dst, 4] clamped to [0, src), 11-bit coefficients int64 [dst, 4])."""
    scale = np.float64(1.0) / (np.float64(dst) / np.float64(src))
    fx = ((np.arange(dst, dtype=np.float64) + 0.5) * scale - 0.5).astype(np.float32)
    fl = np.floor(fx)
    x = (fx - fl).astype(np.float32)
    f = np.float32
    A, one = f(-0.75), f(1)
    x1, y = x + one, one - x
    c0 = ((A * x1 - f(5) * A) * x1 + f(8) * A) * x1 - f(4) * A
    c1 = ((A + f(2)) * x - (A + f(3))) * x * x + one
    c2 = ((A + f(2)) * y - (A + f(3))) * y * y + one
    c3 = one - c0 - c1 - c2
    coef = np.rint(np.stack([c0, c1, c2, c3], 1).astype(np.float32) * f(2048)).astype(np.int64)
    idx = np.clip(fl.astype(np.int64)[:, None] + np.arange(-1, 3)[None, :], 0, src - 1)
    return idx, coef


def resize_cubic_u8(img, oH, oW):
    """uint8 [H, W] or [H, W, C] -> uint8 [oH, oW(, C)], equal to OpenCV's generic INTER_CUBIC resize."""
    img = np.asarray(img, np.uint8)
    H, W = img.shape[:2]
    C = img.shape[2] if img.ndim == 3 else 1
    xi, xc = cubic_taps(oW, W)
    yi, yc = cubic_taps(oH, H)
    s = img.reshape(H, W, C).astype(np.int64)
    hs = (s[:, xi] * xc[None, :, :, None]).sum(2).reshape(H, oW * C)        # [H, oW * C]
    rows = hs[yi]                                                              # [oH, 4, oW * C]
    b = (yc.astype(np.float32) * np.float32(2.0 ** -22)).astype(np.float64)
    t = (rows[:, 3] * b[:, 3:4]).astype(np.float32)
    for k in (2, 1, 0):                                                        # fma: exact in float64, one fp32 rounding
        t = (rows[:, k] * b[:, k:k + 1] + t.astype(np.float64)).astype(np.float32)
    vf = np.rint(t).astype(np.int64)
    vi = ((rows * yc[:, :, None]).sum(1) + (1 << 21)) >> 22
    end = oW * C // 8 * 8
    v = np.concatenate([vf[:, :end], vi[:, end:]], 1)
    out = np.clip(v, 0, 255).astype(np.uint8)
    return out.reshape((oH, oW, C) if img.ndim == 3 else (oH, oW))


def augment_frame(img, flips):
    """H5Dataset.augment_frame's result for flip bits (1: Horizontal = np.flip(img, 1), 2: Vertical = np.flip(img, 0))."""
    if flips & 1:
        img = np.flip(img, 1)
    if flips & 2:
        img = np.flip(img, 0)
    return np.ascontiguousarray(img)


def formatted_frame(img, oH, oW, flips=0):
    """frame_formatting(cv2.resize(augment_frame(img), (oW, oH), INTER_CUBIC)) as numpy: fp32 [1, oH, oW(, C)]."""
    u = resize_cubic_u8(augment_frame(img, flips), oH, oW)
    return (u.astype(np.float32) / np.float32(255))[None]


def gt_image_index(image_ts, inp_ts, idx0, idx1):
    """H5Dataset.get_gt_frame's image index (h5dataset.py:477-487): bisection of the image timestamps at the input event in
    the middle of the window, clamped to [0, n - 1].  binary_search_h5_dset returns the probed index on an exact hit."""
    image_ts = np.asarray(image_ts, np.float64)
    out = []
    for a, b in zip(np.atleast_1d(idx0), np.atleast_1d(idx1)):
        x = float(inp_ts[int((int(a) + int(b)) // 2)])
        lo, hi, res = 0, len(image_ts) - 1, -1
        while lo <= hi:
            mid = lo + (hi - lo) // 2
            if image_ts[mid] == x:
                res = mid
                break
            if image_ts[mid] < x:
                lo = mid + 1
            else:
                hi = mid - 1
        i = res if res >= 0 else lo
        out.append(min(max(i, 0), len(image_ts) - 1))
    return np.asarray(out, np.int64)
