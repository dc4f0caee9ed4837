"""A live event stream in, SR events out as each window completes: esr_b200.superresolve for a recording that is still arriving.

    s = EventStream(model, lr_size=(H, W), scale=k, window=2048, chunk=8)
    s.push(xs, ys, ts, ps)        # any number of events, 0 or part of a frame included
    out = s.pull()                # {'xs', 'ys': int16, 'ts', 'ps': float64} numpy columns ready so far (maybe empty); never blocks
    out = s.pull(wait=True)       # waits for everything pushed so far that can be emitted
    out = s.close()               # ends the stream; returns the rest

The contract is superresolve's (see its module docstring) for config mode 'events', sliding_window 0, sequence_length = seqn,
step_size 1:
  * frame f = input events [f * W, (f + 1) * W) (W = window); window i = frames i .. i + N - 1 (N = model._cfg['num_frame']);
    window i emits the events of its middle frame m = i + (N - 1) // 2: cnt2event(round-half-even(SR counts), 'linear') in
    cnt2event's order, no padding, no zero row for an empty window, t = t0 + float64(t32) * (t1 - t0) with t0, t1 the raw
    timestamps of frame m's first and last input event.
  * The reference clamps a frame's end to num_events - 1 (h5dataset.py:204-208), so when a recording's length is a multiple of
    W its last frame loses its last event.  Frame f is therefore final only once more than (f + 1) * W events have arrived,
    or at close(), where the stream has n // W frames and the clamp applies (frame_rows).  Fewer than N frames emit nothing.
  * Whatever the push sizes, everything pull() and close() return, concatenated, equals byte for byte the columns
    super_resolve_recordings writes for the same events stored as one recording.
  * Refused with ESRError: sliding_window > 0 (consecutive middle frames would overlap), a model whose plan refuses its
    configuration, an HR size above int16, timestamps that decrease within or across pushes, coordinates outside the LR size,
    columns of unequal length, push after close.
  * The stream owns its model object's carried ConvGRU state: it calls reset_states() at construction, and a model object
    serves one stream at a time.  Two streams need two model objects (which may load one state_dict).

Per push, on the current CUDA stream: the events go through a reused pinned staging buffer into an HBM ring of int16 xs / ys
and float64 ps holding the frames not encoded yet; the ring's capacity is a multiple of W, so every frame is contiguous in it
and esr_encode_frames_multi encodes newly final frames straight from it (one recording, start = position mod capacity).  The
HR frames go to a bank of chunk + N - 1 frames whose last N - 1 are the next call's context.  Only each frame's (t0, t1) is
taken from ts, on the host.  k ready windows run as forward_sequence calls of descending powers of two no larger than chunk
(so at most log2(chunk) + 1 plans per shape; DeepRecurrNet.carry_states hands the ConvGRU state from one length to the next),
never padded, because a padded window would advance the carried state.  Each call's events are emitted as superresolve
emits them (superresolve.emit_call) and copied out of pinned memory without waiting once the device has written them.
Device and pinned memory are bounded by window, chunk and the largest call's events, not by the stream's length.
"""
from collections import deque

import numpy as np
import torch

from . import _lib, superresolve as sr

_COLUMNS = (("xs", np.int16), ("ys", np.int16), ("ts", np.float64), ("ps", np.float64))


def final_frames(n, closed, window):
    """The number of final frames after n events: those f with (f + 1) * window < n, or n // window once closed."""
    return n // window if closed else max(n - 1, 0) // window


def frame_rows(n, closed, window, first=0):
    """(idx0, idx1) of the final frames first, first + 1, ... after n events (closed: the stream has ended): int64 [F, 2],
    rows of WindowIndex.event_indices for mode 'events', sliding_window 0 (compute_k_indices, h5dataset.py:196-208)."""
    idx0 = np.arange(first, final_frames(n, closed, window), dtype=np.int64) * window
    return np.stack([idx0, np.minimum(idx0 + window, n - 1)], 1)


def _empty():
    return {c: np.zeros(0, dt) for c, dt in _COLUMNS}


class EventStream:
    """Super-resolve one live event stream (see the module docstring).  `frames`: the final frames so far; `windows_returned`:
    the windows whose events pull() and close() have returned so far (windows that emit no events included)."""

    def __init__(self, model, lr_size, scale, window, chunk=8, sliding_window=0):
        if sliding_window != 0:
            raise _lib.ESRError(f"stream: sliding_window {sliding_window} makes consecutive middle frames overlap: merging "
                                "overlapping windows is not implemented (sliding_window must be 0)")
        model._check_supported()
        H, W = (int(v) for v in lr_size)
        if H < 1 or W < 1 or int(scale) != scale or scale < 1 or window < 1 or chunk < 1:
            raise ValueError(f"stream: lr_size {tuple(lr_size)}, scale {scale}, window {window} and chunk {chunk} must be positive "
                             "integers")
        scale = int(scale)
        sr.check_resolution((H * scale, W * scale))
        self.model, self.res, self.hr = model, (H, W), (H * scale, W * scale)
        self.window, self.chunk, self.N = int(window), int(chunk), model._cfg["num_frame"]
        model.reset_states()
        self.cap = (self.chunk + self.N) * self.window           # ring events; a multiple of W keeps every frame contiguous
        self.bank_frames = self.chunk + self.N - 1
        self.dev = None             # the device buffers are made when the first events leave the staging buffer
        self._stage_np = [np.zeros(self.cap, dt) for dt in (np.int16, np.int16, np.float64)]
        self._ts = np.zeros(self.cap, np.float64)                # host ring of timestamps, same positions as the HBM ring
        self._times = np.zeros((self.bank_frames, 2), np.float64)  # (t0, t1) of frame f at row f % bank_frames
        self._n = 0                 # events pushed
        self._staged = 0            # events [staged, n) wait in the staging buffer; [enc * W, staged) are in the ring
        self._copy = None           # CUDA event after the last staging -> ring copy
        self._enc = 0               # frames encoded: frames [win, enc) are in bank 0 at rows f - win
        self._win = 0               # the next window to run
        self._key = None            # the plan shape of the last call
        self._last_t = -np.inf
        self._closed = False
        self._pinned, self._pending, self._ready = [], deque(), []
        self._collected = 0
        self.frames = 0
        self.windows_returned = 0

    def _allocate(self):
        """The HBM ring, the pinned staging buffer (which takes over what the host-side one holds) and the frame banks."""
        self.dev = torch.device("cuda", torch.cuda.current_device())
        (H, W), (kH, kW) = self.res, self.hr
        with torch.cuda.device(self.dev):
            self._ring = self._views(torch.empty((12 * self.cap,), dtype=torch.uint8, device=self.dev))
            self._stage = self._views(torch.empty((12 * self.cap,), dtype=torch.uint8).pin_memory())
            host = self._stage_np
            self._stage_np = [v.numpy() for v in self._stage]
            for dst, src in zip(self._stage_np, host):
                dst[:] = src
            self._cols = torch.tensor([[v.data_ptr() for v in self._ring]], dtype=torch.int64).to(self.dev)
            self._banks = [torch.zeros((self.bank_frames, 2, kH, kW), dtype=torch.float32, device=self.dev) for _ in range(2)]
            self._lr = torch.empty((self.bank_frames, 2, H, W), dtype=torch.float32, device=self.dev)

    @staticmethod
    def _views(buf):
        c = buf.numel() // 12
        return (buf[:2 * c].view(torch.int16), buf[2 * c:4 * c].view(torch.int16), buf[4 * c:].view(torch.float64))

    # ---- input -------------------------------------------------------------------------------------------------------
    def push(self, xs, ys, ts, ps):
        """Append events (1-D array-likes of one length: x, y in the LR size, ts non-decreasing across pushes, p).  Runs the
        windows they complete; their events become available to pull()."""
        if self._closed:
            raise _lib.ESRError("stream: push after close")
        cols = [np.asarray(c) for c in (xs, ys, ts, ps)]
        if any(c.ndim != 1 for c in cols) or len({len(c) for c in cols}) != 1:
            raise _lib.ESRError(f"stream: xs, ys, ts, ps must be 1-D columns of one length, got shapes {[c.shape for c in cols]}")
        xs, ys, ts, ps = cols
        n = len(ts)
        if n == 0:
            return
        ts = ts.astype(np.float64)
        down = np.flatnonzero(np.diff(ts, prepend=self._last_t) < 0)
        if len(down):
            i = int(down[0])
            prev = ts[i - 1] if i > 0 else self._last_t
            raise _lib.ESRError(f"stream: timestamps decrease at event {self._n + i} ({prev!r} -> {ts[i]!r})")
        H, W = self.res
        out = np.flatnonzero((xs < 0) | (xs >= W) | (ys < 0) | (ys >= H))
        if len(out):
            i = int(out[0])
            raise _lib.ESRError(f"stream: event {self._n + i} at x {xs[i]}, y {ys[i]} is outside the LR size {H} x {W}")
        k = 0
        while k < n:                                              # pieces that fit the ring's free space
            take = min(n - k, self.cap - (self._n - self._enc * self.window))
            if self._copy is not None:                            # the staging buffer is still being read
                self._copy.synchronize()
                self._copy = None
            o = self._n - self._staged
            for dst, src in zip(self._stage_np, (xs, ys, ps)):
                dst[o:o + take] = src[k:k + take]
            pos = (self._n + np.arange(take)) % self.cap
            self._ts[pos] = ts[k:k + take]
            self._n += take
            k += take
            self._advance(False)
        self._last_t = ts[-1]

    def close(self):
        """End the stream: the last frame becomes final (with the reference's clamp), its windows run, and everything not yet
        returned is returned, as pull(wait=True) would.  A second close() returns nothing."""
        if not self._closed:
            self._closed = True
            self._advance(True)
        return self.pull(wait=True)

    # ---- output ------------------------------------------------------------------------------------------------------
    def pull(self, wait=False):
        """The SR events of the windows completed since the last pull, as numpy columns {'xs', 'ys': int16, 'ts', 'ps':
        float64}, in window order.  wait False returns what the device has finished (maybe nothing); True waits for all."""
        self._collect(wait)
        ready, self._ready = self._ready, []
        self.windows_returned = self._collected
        if not ready:
            return _empty()
        return {c: np.concatenate([r[j] for r in ready]) for j, (c, _) in enumerate(_COLUMNS)}

    def _collect(self, wait):
        while self._pending and (wait or self._pending[0][0].query()):
            done, buf, total, nw = self._pending.popleft()
            done.synchronize()
            self._ready.append([v.numpy().copy() for v in sr._segment_views(buf, total)])
            self._pinned.append(buf)
            self._collected += nw

    # ---- the device side ---------------------------------------------------------------------------------------------
    def _flush(self):
        """Staged events -> the HBM ring (split where the ring wraps)."""
        m = self._n - self._staged
        if m == 0:
            return
        if self.dev is None:
            self._allocate()
        p = self._staged % self.cap
        a = min(m, self.cap - p)
        with torch.cuda.device(self.dev):
            for dst, src in zip(self._ring, self._stage):
                dst[p:p + a].copy_(src[:a], non_blocking=True)
                if m > a:
                    dst[:m - a].copy_(src[a:m], non_blocking=True)
            self._copy = torch.cuda.Event()
            self._copy.record()
        self._staged = self._n

    def _advance(self, closed):
        """Encode the final frames that fit the bank, run the ready windows, repeat until neither is possible."""
        N, Wn = self.N, self.window
        self.frames = final_frames(self._n, closed, Wn)
        while True:
            rows = frame_rows(self._n, closed, Wn, self._enc)[:self._win + self.bank_frames - self._enc]
            if len(rows):
                self._encode(rows)
            ready = self._enc - (N - 1) - self._win
            if ready > 0:
                with torch.cuda.device(self.dev):
                    self._run(ready)
            elif not len(rows):
                return

    def _encode(self, rows):
        self._flush()
        with torch.cuda.device(self.dev):
            self._encode_frames(rows)

    def _encode_frames(self, rows):
        e, a = len(rows), self._enc - self._win
        lens = rows[:, 1] - rows[:, 0]
        desc = np.zeros((e, 3), np.int64)                        # esr_frame_desc: start, len, rec 0 | xform 0
        desc[:, 0] = rows[:, 0] % self.cap
        desc[:, 1] = lens
        H, W = self.res
        kH, kW = self.hr
        _lib.check(_lib.lib().esr_encode_frames_multi(_lib.ptr(self._cols), _lib.ptr(torch.from_numpy(desc).to(self.dev)), e,
                                                      int(lens.max()), H, W, kH, kW, _lib.ptr(self._lr),
                                                      _lib.ptr(self._banks[0][a:a + e]), _lib.stream_ptr()),
                   "esr_encode_frames_multi")
        t0 = self._ts[rows[:, 0] % self.cap]
        t1 = np.where(lens > 0, self._ts[(rows[:, 1] - 1) % self.cap], t0)
        f = np.arange(self._enc, self._enc + e)
        self._times[f % self.bank_frames] = np.stack([t0, t1], 1)
        self._enc += e

    def _run(self, ready):
        """`ready` windows from bank row 0 on, as forward_sequence calls of descending powers of two; then the frames left
        move to the front of the other bank."""
        N, (kH, kW) = self.N, self.hr
        off = 0
        while off < ready:
            s = 1 << ((ready - off).bit_length() - 1)
            L = s + N - 1
            key = (1, L, kH, kW)
            if self._key is not None and self._key != key:
                self.model.carry_states(self._key, key, self.dev)
            self._key = key
            with torch.no_grad():
                esr = self.model.forward_sequence(self._banks[0][off:off + L].unsqueeze(0))
            mids = (self._win + off + (N - 1) // 2 + np.arange(s)) % self.bank_frames
            t0, t1 = self._times[mids, 0], self._times[mids, 1]
            done, buf, total, _ = sr.emit_call(esr, t0, t1, self._pinned, self._collect)
            self._pending.append((done, buf, total, s))
            off += s
        self._win += ready
        left = self._enc - self._win
        if left:
            self._banks[1][:left].copy_(self._banks[0][ready:ready + left])
        self._banks.reverse()
