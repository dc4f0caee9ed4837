"""Live event streams in, SR events out as each window completes: esr_b200.superresolve for recordings that are still arriving.

One stream:

    s = EventStream(model, lr_size=(H, W), scale=k, window=2048, chunk=8)
    s.push(xs, ys, ts, ps)        # any number of events, 0 or part of a frame included
    out = s.pull()                # {'xs', 'ys': int16, 'ts', 'ps': float64} numpy columns ready so far (maybe empty); never blocks
    out = s.pull(wait=True)       # waits for everything pushed so far that can be emitted
    out = s.close()               # ends the stream; returns the rest

Many streams on one model object, their ready windows batched into shared calls:

    pool = EventStreamPool(model, lr_size=(H, W), scale=k, window=2048, slots=16, chunk=8, capacity=256)
    sid = pool.open()             # a new stream with a zero state; ESRError when `capacity` streams are open
    pool.push(sid, xs, ys, ts, ps)  # stages the events; runs nothing unless the stream's ring is full (then a round runs)
    pool.run()                    # one round: every ready window of every open stream, batched across streams
    out = pool.pull(sid, wait=False)
    out = pool.close(sid)         # the stream's last frame becomes final, its windows run, the rest is returned

The contract is superresolve's (see its module docstring) for config mode 'events', sliding_window 0, sequence_length = seqn,
step_size 1:
  * frame f = input events [f * W, (f + 1) * W) (W = window); window i = frames i .. i + N - 1 (N = model._cfg['num_frame']);
    window i emits the events of its middle frame m = i + (N - 1) // 2: cnt2event(round-half-even(SR counts), 'linear') in
    cnt2event's order, no padding, no zero row for an empty window, t = t0 + float64(t32) * (t1 - t0) with t0, t1 the raw
    timestamps of frame m's first and last input event.
  * The reference clamps a frame's end to num_events - 1 (h5dataset.py:204-208), so when a recording's length is a multiple of
    W its last frame loses its last event.  Frame f is therefore final only once more than (f + 1) * W events have arrived,
    or at close(), where the stream has n // W frames and the clamp applies (frame_rows).  Fewer than N frames emit nothing.
  * Whatever the push sizes, everything pull() and close() return for a stream, concatenated, equals byte for byte the columns
    super_resolve_recordings writes for the same events stored as one recording.  In a pool this holds per stream whatever
    the interleaving of pushes, runs and pulls across streams, the number of slots, and which streams share a call: every
    plan kernel works per image, so a sample's output does not depend on its batch-mates.
  * Refused with ESRError: sliding_window > 0 (consecutive middle frames would overlap), a model whose plan refuses its
    configuration, an HR size above int16, timestamps that decrease within or across pushes, coordinates outside the LR size,
    columns of unequal length, push after close; in a pool also an unknown or closed stream and opening past `capacity`.
  * A stream or pool owns its model object's carried ConvGRU state: it calls reset_states() at construction, and a model
    object serves one stream or pool at a time.  All streams of a pool share one (lr_size, scale, window).

On the device, on the current CUDA stream.  Each stream has a ring of int16 xs / ys and float64 ps in HBM, (chunk + N) * W
events, holding its frames from the next window's first on; the capacity is a multiple of W, so every frame is contiguous in
it.  Pushed events wait in a host mirror of the ring.  A round that runs windows first uploads every stream's new events:
they are packed into one pinned buffer, moved by one host-to-device copy, and esr_events_append_rings scatters each stream's
segment into its ring in one launch.  Only each frame's (t0, t1) is taken from ts, on the host.  The round's calls come from
plan_round: each stream's ready windows in descending powers of two no larger than chunk, pieces of one size sharing calls of
at most `slots` streams.  A call of s windows over B slots (B a power of two, at most slots) encodes its [B, s + N - 1]
frames from the rings with one esr_encode_frames_multi launch, loads the slots' ConvGRU states from the pool's state rows
(esr_net_gather_states), runs forward_sequence and stores them back (esr_net_scatter_states).  Its events are emitted as
superresolve emits them (superresolve.emit_call) in stream-major order and copied out of pinned memory without waiting once the
device has written them.  Device and pinned memory depend on capacity, slots, chunk, window and the largest call, not on how
long the streams run.
"""
from collections import deque

import numpy as np
import torch

from . import _lib, superresolve as sr

_COLUMNS = (("xs", np.int16), ("ys", np.int16), ("ts", np.float64), ("ps", np.float64))
RING_DESC = np.dtype([("xs", "<u8"), ("ys", "<u8"), ("ps", "<u8"), ("capacity", "<i8"), ("position", "<i8"), ("count", "<i8"),
                      ("src", "<i8")])                                                    # esr_ring_desc
FRAME_DESC = np.dtype([("start", "<i8"), ("len", "<i8"), ("rec", "<i4"), ("xform", "<i4")])   # esr_frame_desc


def final_frames(n, closed, window):
    """The number of final frames after n events: those f with (f + 1) * window < n, or n // window once closed."""
    return n // window if closed else max(n - 1, 0) // window


def frame_rows(n, closed, window, first=0):
    """(idx0, idx1) of the final frames first, first + 1, ... after n events (closed: the stream has ended): int64 [F, 2],
    rows of WindowIndex.event_indices for mode 'events', sliding_window 0 (compute_k_indices, h5dataset.py:196-208)."""
    idx0 = np.arange(first, final_frames(n, closed, window), dtype=np.int64) * window
    return np.stack([idx0, np.minimum(idx0 + window, n - 1)], 1)


def plan_round(ready, slots, chunk):
    """The calls of one round: ready = {stream: ready windows} (or a sequence indexed by stream) -> [(s, [stream, ...]), ...].
    Each stream's windows are split into descending powers of two no larger than chunk; calls are issued in descending s, so
    each stream's windows stay in order.  The pieces of one size share calls of at most `slots` streams, and a call never holds
    one stream twice: with n_s pieces of size s over all streams and at most m_s of them in one stream, size s takes exactly
    max(ceil(n_s / slots), m_s) calls."""
    items = ready.items() if hasattr(ready, "items") else enumerate(ready)
    top = 1 << (int(chunk).bit_length() - 1)
    pieces = {}                                                    # s -> [stream, ...], a stream's pieces adjacent
    for sid, n in sorted(items, key=lambda kv: kv[0]):
        n = int(n)
        while n > 0:
            s = min(top, 1 << (n.bit_length() - 1))
            pieces.setdefault(s, []).append(sid)
            n -= s
    calls = []
    for s in sorted(pieces, reverse=True):
        p = pieces[s]
        m = max(-(-len(p) // slots), max(p.count(sid) for sid in set(p)))
        # piece t goes to call t mod m: a stream's (at most m) adjacent pieces land in distinct calls, and no call holds more
        # than ceil(n_s / m) <= slots pieces
        calls += [(s, p[c::m]) for c in range(m)]
    return calls


def _empty():
    return {c: np.zeros(0, dt) for c, dt in _COLUMNS}


def _join(parts):
    if not parts:
        return _empty()
    return {c: np.concatenate([r[j] for r in parts]) for j, (c, _) in enumerate(_COLUMNS)}


class _Stream:
    """One open stream of a pool.  Events [win * W, n) are in the host mirror (ring positions mod cap); [win * W, up) are
    also in the device ring."""

    def __init__(self, row, mirror):
        self.row, self.mirror = row, mirror        # mirror: xs, ys, ps, ts numpy columns of the ring's capacity
        self.n = self.up = self.win = 0
        self.fresh = True                          # no call has run yet: the state row holds nothing of this stream
        self.closed = False
        self.last_t = -np.inf
        self.parts, self.collected, self.returned = [], 0, 0


class EventStreamPool:
    """Super-resolve many live event streams of one shape on one model object, batching their ready windows into shared
    calls (see the module docstring).  slots: the largest batch of a call; chunk: the most windows of one stream in a call;
    capacity: the most streams open at once."""

    def __init__(self, model, lr_size, scale, window, slots=16, chunk=8, capacity=256, sliding_window=0):
        if sliding_window != 0:
            raise _lib.ESRError(f"stream: sliding_window {sliding_window} makes consecutive middle frames overlap: merging "
                                "overlapping windows is not implemented (sliding_window must be 0)")
        model._check_supported()
        H, W = (int(v) for v in lr_size)
        if (H < 1 or W < 1 or int(scale) != scale or scale < 1 or window < 1 or chunk < 1 or int(slots) != slots or slots < 1
                or int(capacity) != capacity or capacity < 1):
            raise ValueError(f"stream: lr_size {tuple(lr_size)}, scale {scale}, window {window}, chunk {chunk}, slots {slots} "
                             f"and capacity {capacity} must be positive integers")
        scale = int(scale)
        sr.check_resolution((H * scale, W * scale))
        self.model, self.res, self.hr = model, (H, W), (H * scale, W * scale)
        self.window, self.chunk, self.slots, self.capacity = int(window), int(chunk), int(slots), int(capacity)
        self.N = model._cfg["num_frame"]
        model.reset_states()
        self.cap = (self.chunk + self.N) * self.window           # ring events per stream; a multiple of W
        self.dev = None                                          # device buffers are made by the first round that runs windows
        self._streams, self._next_sid = {}, 0
        self._free = list(range(self.capacity - 1, -1, -1))     # free rows (ring, state row, host mirror); pop() takes row 0 first
        self._mirrors = [None] * self.capacity
        self._stage, self._uploaded = None, None                 # pinned upload buffer; CUDA event after the last upload's copy
        self._pinned, self._pending = [], deque()                # idle emission buffers; (event, buffer, total, [(sid, a, b, nw)])

    # ---- streams ------------------------------------------------------------------------------------------------------
    def open(self):
        """A new stream with a zero ConvGRU state -> its id."""
        if not self._free:
            raise _lib.ESRError(f"stream pool: {self.capacity} streams are open (capacity {self.capacity})")
        row = self._free.pop()
        if self._mirrors[row] is None:
            self._mirrors[row] = [np.zeros(self.cap, dt) for dt in (np.int16, np.int16, np.float64, np.float64)]
        sid = self._next_sid
        self._next_sid += 1
        self._streams[sid] = _Stream(row, self._mirrors[row])
        return sid

    def _get(self, sid, what):
        st = self._streams.get(sid)
        if st is None:
            if isinstance(sid, (int, np.integer)) and 0 <= sid < self._next_sid:
                raise _lib.ESRError(f"stream pool: {what} after close (stream {sid})")
            raise _lib.ESRError(f"stream pool: {what}: no stream {sid!r}")
        return st

    def frames(self, sid):
        """The final frames of stream sid so far."""
        st = self._get(sid, "frames")
        return final_frames(st.n, st.closed, self.window)

    def windows_returned(self, sid):
        """The windows whose events pull(sid) has returned so far (windows that emit no events included)."""
        return self._get(sid, "windows_returned").returned

    # ---- input --------------------------------------------------------------------------------------------------------
    def push(self, sid, xs, ys, ts, ps):
        """Append events to stream sid (1-D array-likes of one length: x, y in the LR size, ts non-decreasing across pushes,
        p).  Runs nothing, unless the stream's ring is full: then a round runs (other streams' ready windows join it)."""
        st = self._get(sid, "push")
        cols = [np.asarray(c) for c in (xs, ys, ts, ps)]
        if any(c.ndim != 1 for c in cols) or len({len(c) for c in cols}) != 1:
            raise _lib.ESRError(f"stream: xs, ys, ts, ps must be 1-D columns of one length, got shapes {[c.shape for c in cols]}")
        xs, ys, ts, ps = cols
        n = len(ts)
        if n == 0:
            return
        ts = ts.astype(np.float64)
        down = np.flatnonzero(np.diff(ts, prepend=st.last_t) < 0)
        if len(down):
            i = int(down[0])
            prev = ts[i - 1] if i > 0 else st.last_t
            raise _lib.ESRError(f"stream: timestamps decrease at event {st.n + i} ({prev!r} -> {ts[i]!r})")
        H, W = self.res
        out = np.flatnonzero((xs < 0) | (xs >= W) | (ys < 0) | (ys >= H))
        if len(out):
            i = int(out[0])
            raise _lib.ESRError(f"stream: event {st.n + i} at x {xs[i]}, y {ys[i]} is outside the LR size {H} x {W}")
        k = 0
        while k < n:                                              # pieces that fit the ring's free space
            take = min(n - k, self.cap - (st.n - st.win * self.window))
            if take == 0:
                self.run()                                        # frees at least chunk * W events of this ring
                continue
            p = st.n % self.cap
            a = min(take, self.cap - p)
            for dst, src in zip(st.mirror, (xs, ys, ps, ts)):
                dst[p:p + a] = src[k:k + a]
                dst[:take - a] = src[k + a:k + take]
            st.n += take
            k += take
        st.last_t = ts[-1]

    def run(self):
        """One round: every open stream's ready windows run, batched across streams (plan_round).  Their events become
        available to pull()."""
        N, Wn = self.N, self.window
        ready = {sid: max(final_frames(st.n, st.closed, Wn) - (N - 1) - st.win, 0) for sid, st in self._streams.items()}
        calls = plan_round({sid: r for sid, r in ready.items() if r}, self.slots, self.chunk)
        if not calls:
            return
        if self.dev is None:
            self._allocate()
        with torch.cuda.device(self.dev):
            self._upload()
            at = {sid: self._streams[sid].win for sid in ready}   # each stream's next window in this round
            for s, sids in calls:
                self._call(s, sids, at)
        for sid, r in ready.items():
            self._streams[sid].win += r

    def close(self, sid):
        """End stream sid: its last frame becomes final (with the reference's clamp), its windows run, and everything not
        yet returned is returned, as pull(sid, wait=True) would.  Its ring and state row go to the next open()."""
        return self._close(sid)[0]

    def _close(self, sid):
        st = self._get(sid, "close")
        st.closed = True
        self.run()
        out = self.pull(sid, wait=True)
        del self._streams[sid]
        self._free.append(st.row)
        return out, st

    # ---- output -------------------------------------------------------------------------------------------------------
    def pull(self, sid, wait=False):
        """The SR events of stream sid's windows completed since its last pull, as numpy columns {'xs', 'ys': int16, 'ts',
        'ps': float64}, in window order.  wait False returns what the device has finished (maybe nothing); True waits for
        all of this stream's windows that have run."""
        st = self._get(sid, "pull")
        last = max((i for i, p in enumerate(self._pending) if any(r[0] == sid for r in p[3])), default=-1) if wait else -1
        self._collect(last)
        parts, st.parts = st.parts, []
        st.returned = st.collected
        return _join(parts)

    def _collect(self, upto=-1):
        """Hand the finished calls' segments to their streams: calls [0, upto] whether finished or not, then every finished
        one."""
        while self._pending and (upto >= 0 or self._pending[0][0].query()):
            done, buf, total, runs = self._pending.popleft()
            upto -= 1
            done.synchronize()
            cols = [v.numpy() for v in sr._segment_views(buf, total)]
            for sid, a, b, nw in runs:
                st = self._streams[sid]
                st.parts.append([c[a:b].copy() for c in cols])
                st.collected += nw
            self._pinned.append(buf)

    # ---- the device side ----------------------------------------------------------------------------------------------
    def _allocate(self):
        """The rings, their column table, the state rows and the frame banks of the largest call."""
        self.dev = torch.device("cuda", torch.cuda.current_device())
        (H, W), (kH, kW) = self.res, self.hr
        top = 1 << (self.chunk.bit_length() - 1)
        frames = self.slots * (top + self.N - 1)
        with torch.cuda.device(self.dev):
            c, R = self.cap, self.capacity
            rings = torch.empty((12 * R * c,), dtype=torch.uint8, device=self.dev)
            self._rings = (rings[:2 * R * c].view(torch.int16).view(R, c), rings[2 * R * c:4 * R * c].view(torch.int16).view(R, c),
                           rings[4 * R * c:].view(torch.float64).view(R, c))
            self._ring_addr = np.stack([[v[r].data_ptr() for v in self._rings] for r in range(R)]).astype(np.uint64)  # [R, 3]
            self._cols = torch.from_numpy(self._ring_addr.view(np.int64)).to(self.dev)
            self._state_bytes = _lib.lib().esr_net_state_bytes(kH, kW)
            self._states = torch.empty((R * self._state_bytes,), dtype=torch.uint8, device=self.dev)
            self._bank = torch.empty((frames, 2, kH, kW), dtype=torch.float32, device=self.dev)
            self._lr = torch.empty((frames, 2, H, W), dtype=torch.float32, device=self.dev)

    def _upload(self):
        """Every stream's events not yet on the device -> one pinned buffer (int16 xs | int16 ys | float64 ps) -> one
        host-to-device copy -> the rings, one esr_events_append_rings launch.  (Measured on an H100 at 64 streams of 2048
        events, the copy and the kernel reading device memory take 0.050 ms, the kernel reading the pinned buffer directly
        0.066-0.071 ms: tools/bench_stream_pool.py.)"""
        segs = [st for st in self._streams.values() if st.n > st.up]
        if not segs:
            return
        total = sum(st.n - st.up for st in segs)
        total += total & 1                                        # even: ps starts 8-byte aligned
        if self._uploaded is not None:                            # the last upload's copy may still read the pinned buffer
            self._uploaded.synchronize()
        if self._stage is None or self._stage.numel() < 12 * total:
            self._stage = torch.empty((12 * max(total, 1 << 16),), dtype=torch.uint8).pin_memory()
            self._stage_d = torch.empty_like(self._stage, device=self.dev)
        host = [v.numpy() for v in self._columns(self._stage, total)]
        desc = np.zeros(len(segs), RING_DESC)
        o = 0
        for i, st in enumerate(segs):
            m, p = st.n - st.up, st.up % self.cap
            a = min(m, self.cap - p)
            for dst, col in zip(host, st.mirror[:3]):
                dst[o:o + a] = col[p:p + a]
                dst[o + a:o + m] = col[:m - a]
            desc[i] = (*self._ring_addr[st.row], self.cap, st.up, m, o)
            o += m
            st.up = st.n
        self._stage_d[:12 * total].copy_(self._stage[:12 * total], non_blocking=True)
        self._uploaded = torch.cuda.Event()
        self._uploaded.record()
        desc_d = torch.from_numpy(desc.view(np.uint8)).to(self.dev)
        _lib.check(_lib.lib().esr_events_append_rings(_lib.ptr(desc_d), len(segs), int(desc["count"].max()),
                                                      *map(_lib.ptr, self._columns(self._stage_d, total)), _lib.stream_ptr()),
                   "esr_events_append_rings")

    @staticmethod
    def _columns(buf, T):
        """The xs, ys, ps columns of T events at the front of a byte buffer: int16 xs | int16 ys | float64 ps."""
        return buf[:2 * T].view(torch.int16), buf[2 * T:4 * T].view(torch.int16), buf[4 * T:12 * T].view(torch.float64)

    def _call(self, s, sids, at):
        """One forward_sequence call of s windows for the streams sids, each from window at[sid] on.  B, the smallest power of
        two >= len(sids) (at most slots): padding slots repeat the last stream's frames and state, so they emit as many events
        as it does and never enlarge cnt2event's rows; they emit nothing and their state is not stored."""
        N, Wn, (H, W), (kH, kW) = self.N, self.window, self.res, self.hr
        nb, L = len(sids), s + N - 1
        B = min(1 << (nb - 1).bit_length(), self.slots)
        slot = [self._streams[sid] for sid in sids] + [self._streams[sids[-1]]] * (B - nb)
        first = np.array([at[sid] for sid in sids] + [at[sids[-1]]] * (B - nb), np.int64)
        for sid in sids:
            at[sid] += s
        f = first[:, None] + np.arange(L)                                      # [B, L] frames
        n = np.array([st.n for st in slot], np.int64)[:, None]
        idx0 = f * Wn
        idx1 = np.minimum(idx0 + Wn, n - 1)
        desc = np.zeros(B * L, FRAME_DESC)
        desc["start"] = (idx0 % self.cap).ravel()
        desc["len"] = (idx1 - idx0).ravel()
        desc["rec"] = np.repeat([st.row for st in slot], L)
        rows = np.array([[-1 if st.fresh else st.row for st in slot], [st.row for st in slot[:nb]] + [-1] * (B - nb)], np.int32)
        tables = torch.from_numpy(np.concatenate([desc.view(np.uint8), rows.view(np.uint8).ravel()])).to(self.dev)
        gather, scatter = tables[B * L * FRAME_DESC.itemsize:].view(torch.int32).view(2, B)
        bank = self._bank[:B * L]
        lib = _lib.lib()
        _lib.check(lib.esr_encode_frames_multi(_lib.ptr(self._cols), _lib.ptr(tables), B * L, int(desc["len"].max()), H, W, kH, kW,
                                               _lib.ptr(self._lr), _lib.ptr(bank), _lib.stream_ptr()), "esr_encode_frames_multi")
        plan = self.model._plan(B, L, kH, kW, self.dev)
        _lib.check(lib.esr_net_gather_states(plan.handle, _lib.ptr(self._states), _lib.ptr(gather), _lib.stream_ptr()),
                   "esr_net_gather_states")
        with torch.no_grad():
            esr = self.model.forward_sequence(bank.view(B, L, 2, kH, kW))       # window-major: row j * B + b
        _lib.check(lib.esr_net_scatter_states(plan.handle, _lib.ptr(self._states), _lib.ptr(scatter), _lib.stream_ptr()),
                   "esr_net_scatter_states")
        for st in slot[:nb]:
            st.fresh = False
        # middle frames' (t0, t1), window-major like esr; the segment is written stream-major, padding left out
        m = (first[None, :] + np.arange(s)[:, None] + (N - 1) // 2)             # [s, B]
        mirror_ts = [st.mirror[3] for st in slot]
        m0 = m * Wn
        m1 = np.minimum(m0 + Wn, n.T - 1)
        t0 = np.array([[mirror_ts[b][m0[j, b] % self.cap] for b in range(B)] for j in range(s)])
        t1 = np.array([[mirror_ts[b][(m1[j, b] - 1) % self.cap] if m1[j, b] > m0[j, b] else t0[j, b] for b in range(B)]
                       for j in range(s)])
        order = (np.arange(nb)[:, None] + np.arange(s)[None, :] * B).ravel()   # stream b's windows j = 0 .. s - 1
        done, buf, total, cd = sr.emit_call(esr, t0.ravel(), t1.ravel(), self._pinned, lambda wait: self._collect(), order)
        runs = []
        for b, sid in enumerate(sids):
            a = int(cd["dst"][b])
            runs.append((sid, a, a + int(cd["valid"][b + np.arange(s) * B].sum()), s))
        self._pending.append((done, buf, total, runs))


class EventStream:
    """Super-resolve one live event stream (see the module docstring): a pool of one stream, whose push runs a round.
    `frames`: the final frames so far; `windows_returned`: the windows whose events pull() and close() have returned so far
    (windows that emit no events included)."""

    def __init__(self, model, lr_size, scale, window, chunk=8, sliding_window=0):
        self._pool = EventStreamPool(model, lr_size, scale, window, slots=1, chunk=chunk, capacity=1,
                                     sliding_window=sliding_window)
        self._sid = self._pool.open()
        self._closed = False
        self.frames = 0
        self.windows_returned = 0

    def push(self, xs, ys, ts, ps):
        """Append events (1-D array-likes of one length: x, y in the LR size, ts non-decreasing across pushes, p).  Runs the
        windows they complete; their events become available to pull()."""
        if self._closed:
            raise _lib.ESRError("stream: push after close")
        self._pool.push(self._sid, xs, ys, ts, ps)
        self._pool.run()
        self.frames = self._pool.frames(self._sid)

    def pull(self, wait=False):
        """The SR events of the windows completed since the last pull, as numpy columns {'xs', 'ys': int16, 'ts', 'ps':
        float64}, in window order.  wait False returns what the device has finished (maybe nothing); True waits for all."""
        if self._closed:
            return _empty()
        out = self._pool.pull(self._sid, wait)
        self.windows_returned = self._pool.windows_returned(self._sid)
        return out

    def close(self):
        """End the stream: the last frame becomes final (with the reference's clamp), its windows run, and everything not yet
        returned is returned, as pull(wait=True) would.  A second close() returns nothing."""
        if self._closed:
            return _empty()
        self._closed = True
        out, st = self._pool._close(self._sid)
        self.frames = final_frames(st.n, True, self._pool.window)
        self.windows_returned = st.returned
        return out
