"""Host side of the dense-counts -> event-list kernels (esr_expand_count / esr_expand_emit).

Shared by esr_b200.cnt2event (cnt2event.pyx:18-116) and esr_b200.event_redistribute
(event_redistribute.pyx:17-153).  The one host synchronisation (reading the per-sample statistics) is
inherent: the output length is data dependent, exactly like the reference's np.zeros([batch, maxlen, 4]).
"""
import ctypes
import os

import numpy as np
import torch

from . import _lib


def _numpy_stream(n):
    """The reference reseeds numpy's GLOBAL legacy RNG on every call (cnt2event.pyx:25) and then draws one
    float64 per event in emission order; reproduce both the values and the side effect."""
    np.random.seed(123)
    return np.random.random([int(n)])


_RANK_CACHE = {}


def _rank_table(m, dev):
    """Compact sort keys for cnt2event/linear timestamps: rank of float32(np.linspace(0,1,n)[j]) among all distinct
    timestamps that counts 1..m can produce (numpy's own linspace = the reference's arithmetic).  Cached per (m, device)."""
    key = (m, str(dev))
    if key not in _RANK_CACHE:
        vals = [np.linspace(0, 1, n).astype(np.float32) for n in range(1, m + 1)]
        uniq = np.unique(np.concatenate(vals))
        table = np.zeros((m + 1, m), dtype=np.uint16)
        for n in range(1, m + 1):
            table[n, :n] = np.searchsorted(uniq, vals[n - 1])
        bits = max(1, int(np.ceil(np.log2(max(2, len(uniq))))))
        _RANK_CACHE[key] = (torch.from_numpy(table.view(np.int16)).to(dev), bits)
    return _RANK_CACHE[key]


_XF_MAXN = 64                 # largest per-pixel count the fused path ranks (csrc/expand_fused.cu XF_MAXN)
_XF_TABLES = {}
_XF_SLACK = 4096
_XF_ROWS = {}                 # (device, B, H, W) -> (rows, largest count) of the last call: sizes the next call's guesses


def _xf_tables_host():
    """Key tables of the fused cnt2event path for m = 1, 2, 4 .. 64, built with numpy.linspace (the reference's arithmetic,
    cnt2event.pyx:74): per m a rank table uint16 [(m+1), m] -- rank[n, j] = index of float32(linspace(0, 1, n)[j]) among the K(m)
    distinct timestamps counts <= m can produce -- and those timestamps, ascending.  Returns (blob bytes, desc int32 [7, 3] =
    rank byte offset, timestamps byte offset, K)."""
    blob = bytearray()
    desc = np.zeros((7, 3), dtype=np.int32)
    for i in range(7):
        m = 1 << i
        vals = [np.linspace(0, 1, n).astype(np.float32) for n in range(1, m + 1)]
        uniq = np.unique(np.concatenate(vals))
        table = np.zeros((m + 1, m), dtype=np.uint16)
        for n in range(1, m + 1):
            table[n, :n] = np.searchsorted(uniq, vals[n - 1])
        for j, arr in enumerate((table, uniq.astype(np.float32))):
            blob.extend(b"\0" * (-len(blob) % 16))
            desc[i, j] = len(blob)
            blob.extend(arr.tobytes())
        desc[i, 2] = len(uniq)
    return bytes(blob), np.ascontiguousarray(desc)


def _xf_tables(dev):
    """One device copy of _xf_tables_host() per device."""
    key = str(dev)
    if key not in _XF_TABLES:
        blob, desc = _xf_tables_host()
        _XF_TABLES[key] = (torch.from_numpy(np.frombuffer(blob, dtype=np.uint8).copy()).to(dev), desc)
    return _XF_TABLES[key]


class _ExpandCtx:
    __slots__ = ("vals", "kind", "dims", "counts", "stats", "stats_host", "event", "parts", "fused_out", "fused_cap", "fused_mcap", "ev")


_PINNED = {}                  # rows -> idle pinned [rows, 4] int64 buffers (cudaHostAlloc per call costs more than the kernels)


def _stats_to_host(ctx, dev):
    free = _PINNED.setdefault(int(ctx.stats.shape[0]), [])
    ctx.stats_host = free.pop() if free else torch.empty(tuple(ctx.stats.shape), dtype=torch.int64).pin_memory()
    ctx.stats_host.copy_(ctx.stats, non_blocking=True)
    ctx.event = torch.cuda.Event()
    ctx.event.record()


def _count_begin(ctx):
    """General chain, phase 1: round / count every slot (esr_expand_count), statistics on their way to the host."""
    vals = ctx.vals
    B, P, C, H, W = ctx.dims
    dev = vals.device
    ctx.stats = torch.empty((B, 4), dtype=torch.int64, device=dev)
    ctx.counts = torch.empty((B * P * C * H * W,), dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().esr_expand_count(_lib.ptr(vals), B, P, C, H, W, ctx.kind, _lib.ptr(ctx.stats), _lib.ptr(ctx.counts),
                                               _lib.stream_ptr()), "esr_expand_count")
        _stats_to_host(ctx, dev)


def _fused_begin(ctx):
    """cnt2event / linear in three launches (esr_cnt2event_fused): the padded rows are written before the host knows maxlen,
    into a buffer sized from the previous call of this shape (x1.25; first call: 4 rows per pixel slot), with per-key counters
    sized for twice the previous call's largest count (first call: 64).  expand_finish checks the statistics and falls back to
    the general chain when a guess was too small or the data is outside the fused path."""
    vals = ctx.vals
    B, _, _, H, W = ctx.dims
    dev = vals.device
    L = _lib.lib()
    last = _XF_ROWS.get((str(dev), B, H, W))
    slots = B * 2 * H * W
    cap = int(last[0] * 1.25) + _XF_SLACK if last is not None else 4 * slots
    cap = max(B, min(cap, (1 << 32) - 1, slots * _XF_MAXN))
    mcap = _XF_MAXN if last is None else min(_XF_MAXN, 1 << max(0, int(2 * last[1] - 1).bit_length()))
    tables, desc = _xf_tables(dev)
    ctx.stats = torch.empty((B, 4), dtype=torch.int64, device=dev)
    ctx.fused_cap, ctx.fused_mcap = cap, mcap
    ctx.fused_out = torch.empty((cap * 4,), dtype=torch.float32, device=dev)
    nbytes = L.esr_cnt2event_fused_workspace_bytes(B, H, W)
    ws = torch.empty((nbytes,), dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        _lib.check(L.esr_cnt2event_fused(_lib.ptr(vals), B, H, W, _lib.ptr(tables), desc.ctypes.data_as(ctypes.c_void_p), mcap,
                                         _lib.ptr(ctx.stats), _lib.ptr(ctx.fused_out), cap, _lib.ptr(ws), nbytes, _lib.stream_ptr()),
                   "esr_cnt2event_fused")
        _stats_to_host(ctx, dev)


class FusedCnt2Event:
    """cnt2event / linear with every buffer allocated up front, so that enqueue() can be recorded into a CUDA graph behind the
    network (esr_b200.pipeline): three kernels, two memsets and the 32 B-per-sample statistics copy, no host work per step.
    result() applies the reference's sizing rules (cnt2event.pyx:33-60) to the statistics once the caller has synchronised and
    returns a [B, maxlen, 4] view of the static output, or None when this call was outside the fused path (a count above
    `max_count`, more rows than `cap_rows`): the caller then runs expand() on the same values."""

    def __init__(self, B, H, W, dev, cap_rows, max_count):
        L = _lib.lib()
        self.B, self.H, self.W, self.dev = B, H, W, dev
        self.cap = int(max(B, min(cap_rows, (1 << 32) - 1)))
        self.mcap = min(_XF_MAXN, 1 << max(0, int(max_count - 1).bit_length()))
        self.tables, self.desc = _xf_tables(dev)
        self.stats = torch.zeros((B, 4), dtype=torch.int64, device=dev)
        self.stats_host = torch.zeros((B, 4), dtype=torch.int64).pin_memory()
        self.out = torch.empty((self.cap * 4,), dtype=torch.float32, device=dev)
        self.nbytes = L.esr_cnt2event_fused_workspace_bytes(B, H, W)
        self.ws = torch.empty((self.nbytes,), dtype=torch.uint8, device=dev)

    def enqueue(self, vals):
        assert vals.is_cuda and vals.dtype == torch.float32 and vals.is_contiguous() and tuple(vals.shape) == (self.B, 2, self.H, self.W)
        _lib.check(_lib.lib().esr_cnt2event_fused(_lib.ptr(vals), self.B, self.H, self.W, _lib.ptr(self.tables),
                                                   self.desc.ctypes.data_as(ctypes.c_void_p), self.mcap, _lib.ptr(self.stats),
                                                   _lib.ptr(self.out), self.cap, _lib.ptr(self.ws), self.nbytes, _lib.stream_ptr()),
                   "esr_cnt2event_fused")
        self.stats_host.copy_(self.stats, non_blocking=True)

    def result(self):
        """After the enqueueing stream has been synchronised.  Returns (events or None, rows needed, largest count)."""
        h = self.stats_host.numpy()
        sums, nev, neg = h[:, 0], h[:, 1], h[:, 2]
        np.random.seed(123)                                   # visible side effect of every reference call (cnt2event.pyx:25)
        active = sums != 0
        if not active.any():
            return torch.zeros((self.B, 1, 4), dtype=torch.float32, device=self.dev), self.B, 1
        if bool((active & (neg != 0)).any()):
            raise ValueError("negative dimensions are not allowed")     # np.zeros([-n, 4]) in the reference
        maxlen = int(np.where(active, nev, 1).max())
        mx = int(h[:, 3][active].max())
        rows = self.B * maxlen
        if mx > self.mcap or rows > self.cap:
            return None, rows, mx
        return self.out[:rows * 4].view(self.B, maxlen, 4), rows, mx


def expand_begin(vals, kind, mode=None):
    """Phase 1 (asynchronous): round / count every slot, per-sample statistics -> pinned host memory.  Returns a context for
    expand_finish; nothing here waits for the GPU, so a caller can enqueue more work (the next batch's network) before it
    pays for the host side of phase 2.  A caller that already knows the timestamp mode passes it: cnt2event with linear timestamps
    (kind 0, mode 0) then runs the fused path, which also writes the output rows here."""
    if not vals.is_cuda:
        raise _lib.ESRError("esr_b200.expand needs a CUDA tensor (no CPU fallback)")
    vals = vals.contiguous().float()
    if kind == 0:
        assert vals.dim() == 4 and vals.shape[1] == 2, "Wrong event count data!"
        B, P, H, W = vals.shape
        C = 1
    elif vals.dim() == 5:
        B, P, C, H, W = vals.shape
    elif vals.dim() == 4:
        B, C, H, W = vals.shape
        P = 1
    else:
        raise Exception("wrong event stack")
    ctx = _ExpandCtx()
    ctx.vals, ctx.kind, ctx.dims, ctx.parts = vals, kind, (B, P, C, H, W), None
    ctx.counts = ctx.fused_out = None
    ctx.fused_cap = ctx.fused_mcap = 0
    if B > 256:   # the radix sort carries the sample index in one 8-bit digit
        ctx.parts = [expand_begin(vals[i:i + 256], kind, mode) for i in range(0, B, 256)]
        return ctx
    if kind == 0 and mode == 0 and B * 2 * H * W < (1 << 32) and os.environ.get("ESR_EXPAND_FUSED", "1") != "0":
        _fused_begin(ctx)
    else:
        _count_begin(ctx)
    return ctx


def _host_plan(ctx):
    """Wait for a (sub-)batch's statistics -- the one inherent host synchronisation: the output length is data dependent -- and size
    its output on the host.  Returns None for an all-empty batch (`if event_cnt_round.sum() != 0`, cnt2event.pyx:56)."""
    ctx.event.synchronize()
    h = ctx.stats_host.numpy().copy()
    _PINNED[h.shape[0]].append(ctx.stats_host)
    ctx.stats_host = None
    sums, nev, neg = h[:, 0], h[:, 1], h[:, 2]
    if int(sums.sum()) == 0:
        return None
    active = (sums != 0)
    if ctx.kind == 0 and bool((active & (neg != 0)).any()):
        np.random.seed(123)
        raise ValueError("negative dimensions are not allowed")     # np.zeros([-n, 4]) in the reference
    ev = np.where(active, nev, 0).astype(np.int64)
    return {"active": active, "lens": np.where(active, nev, 1).astype(np.int64), "ev": ev, "total": int(ev.sum()),
            "mx": int(h[:, 3][active].max()) if active.any() else 0}


def _emit(ctx, plan, mode, rnd):
    vals, kind = ctx.vals, ctx.kind
    B, P, C, H, W = ctx.dims
    L = _lib.lib()
    dev = vals.device
    if plan is None:
        return torch.zeros((B, 1, 4), dtype=torch.float32, device=dev)
    if ctx.fused_out is not None:
        rows = B * int(plan["lens"].max())
        _XF_ROWS[(str(dev), B, H, W)] = (rows, max(1, plan["mx"]))
        if mode == 0 and plan["mx"] <= ctx.fused_mcap and rows <= ctx.fused_cap:
            return ctx.fused_out[:rows * 4].view(B, -1, 4)         # the kernels already wrote exactly this (padding included)
        ctx.fused_out = None                                        # outside the fused path: general chain, same statistics
        _count_begin(ctx)
    active, ev, total, mx = plan["active"], plan["ev"], plan["total"], plan["mx"]
    maxlen = int(plan["lens"].max())
    start = np.concatenate([[0], np.cumsum(ev)[:-1]]).astype(np.int64)
    with torch.cuda.device(dev):
        st = _lib.stream_ptr()
        out = torch.zeros((B, maxlen, 4), dtype=torch.float32, device=dev)
        rank, rank_m, rank_bits = None, 0, 0
        if kind == 0 and mode == 0 and 1 <= mx <= 255:
            rank_m = 1 << max(0, (mx - 1).bit_length())            # few distinct table sizes: 1, 2, 4, ... 256
            rank_m = min(rank_m, 255)
            rank, rank_bits = _rank_table(rank_m, dev)
        nbytes = L.esr_expand_workspace_bytes(B, P, C, H, W, total)
        ws = torch.empty((nbytes,), dtype=torch.uint8, device=dev)
        act32 = np.ascontiguousarray(active.astype(np.int32))
        _lib.check(L.esr_expand_emit(_lib.ptr(vals), _lib.ptr(ctx.counts), B, P, C, H, W, kind, int(mode), _lib.ptr(rnd),
                                     _lib.ptr(rank), rank_m, rank_bits,
                                     act32.ctypes.data_as(ctypes.c_void_p), start.ctypes.data_as(ctypes.c_void_p),
                                     total, maxlen, _lib.ptr(out), _lib.ptr(ws), nbytes, st), "esr_expand_emit")
    return out


def expand_finish(ctx, mode):
    """Phase 2: wait for the statistics, size the output, emit and sort.  Returns CUDA fp32 [B, maxlen, 4] and leaves in ctx.ev
    (numpy int64 [B]) every sample's number of events: its rows before the padding, 0 for an empty sample (one zero row).

    Random mode (mode 1): the reference seeds numpy ONCE per call and draws one continuous stream over all samples in emission
    order (cnt2event.pyx:25,74; event_redistribute.pyx:24) -- also when the batch is processed in 256-sample parts here (the radix
    sort carries the sample index in one 8-bit digit): the parts receive consecutive slices of that one stream."""
    B = ctx.dims[0]
    dev = ctx.vals.device
    parts = ctx.parts if ctx.parts is not None else [ctx]
    plans = [_host_plan(c) for c in parts]
    ctx.ev = np.concatenate([np.zeros(c.dims[0], np.int64) if pl is None else pl["ev"] for c, pl in zip(parts, plans)])
    rnds = [None] * len(parts)
    if mode == 1:
        totals = [0 if pl is None else pl["total"] for pl in plans]
        if sum(totals) > 0:
            stream = torch.from_numpy(_numpy_stream(sum(totals))).to(dev)
            off = 0
            for i, t in enumerate(totals):
                rnds[i] = stream[off:off + t] if t > 0 else None
                off += t
        else:
            np.random.seed(123)
    else:
        np.random.seed(123)                         # visible side effect of every reference call
    outs = [_emit(c, pl, mode, r) for c, pl, r in zip(parts, plans, rnds)]
    if ctx.parts is None:
        return outs[0]
    if all(pl is None for pl in plans):             # the whole batch is empty: [B, 1, 4] zeros like one reference call
        return torch.zeros((B, 1, 4), dtype=torch.float32, device=dev)
    maxlen = max(o.shape[1] for o in outs)
    out = ctx.vals.new_zeros((B, maxlen, 4))
    for i, o in enumerate(outs):
        out[i * 256:i * 256 + o.shape[0], :o.shape[1]] = o
    return out


def expand(vals, kind, mode):
    """vals: CUDA fp32 tensor [B,2,H,W] (kind 0) or [B,P,C,H,W] / [B,C,H,W] (kind 1) -> CUDA fp32 [B,maxlen,4]."""
    return expand_finish(expand_begin(vals, kind, mode), mode)
