"""GPU: esr_b200.stream.EventStreamPool -- every stream's joined output byte-equal to EventStream alone and to
super_resolve_recordings' file, whatever the interleaving, the slots and the sharing -- and its new device entries: the state
rows (esr_net_gather_states / esr_net_scatter_states) against torch indexing of the same bytes, esr_events_append_rings
against a numpy model, and device memory that grows neither with the streams' length nor with the streams opened."""
import gc

import numpy as np
import pytest
import torch

from esr_b200 import _lib
from esr_b200.stream import RING_DESC, EventStream, EventStreamPool
from tests.test_stream_gpu import (LR, W, _assert_bytes_equal, _columns, _join, _offline, _sizes, _store, _streamed,  # noqa: F401
                                   stores)
from tests.test_superresolve_gpu import _model

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def net():
    return _model(3, 0.6)


@pytest.fixture(scope="module")
def want(net, stores, tmp_path_factory):
    d = tmp_path_factory.mktemp("pool_offline")
    return [_offline(net, s, d) for s in stores]


def _drive(pool, streams, run=True):
    """streams: {key: (columns, sizes)}; round i pushes piece i of every stream that has one (sizes[i] None: idle), runs a
    round, pulls every open stream; then closes all.  -> {key: joined columns}"""
    rounds = max(len(sizes) for _, sizes in streams.values())
    sid = {k: pool.open() for k in streams}
    outs, at = {k: [] for k in streams}, {k: 0 for k in streams}
    for i in range(rounds):
        for k, (cols, sizes) in streams.items():
            if i < len(sizes) and sizes[i] is not None:
                a, b = at[k], at[k] + sizes[i]
                pool.push(sid[k], *(c[a:b] for c in cols))
                at[k] = b
        if run:
            pool.run()
        for k in streams:
            outs[k].append(pool.pull(sid[k]))
    for k, (cols, _) in streams.items():
        assert at[k] == len(cols[2])
        outs[k].append(pool.close(sid[k]))
    return {k: _join(v) for k, v in outs.items()}


def _random(store, seed):
    cols = _columns(store)
    return cols, _sizes("random", len(cols[2]), seed=seed)


@pytest.mark.parametrize("slots", [1, 2, 3, 8])
def test_interleaved_streams_equal_each_alone(net, stores, want, slots):
    streams = {k: _random(s, k) for k, s in enumerate(stores)}
    got = _drive(EventStreamPool(net, LR, 2, W, slots=slots, chunk=4, capacity=5), streams)
    for k in streams:
        _assert_bytes_equal(got[k], want[k])
        if slots == 2:
            _assert_bytes_equal(got[k], _streamed(_model(3, 0.6), stores[k], streams[k][1])[0])


def test_an_idle_stream_keeps_its_state(net, stores, want):
    cols, sizes = _random(stores[1], 1)
    idle = [sizes[0]] + [None] * 10 + sizes[1:]                     # ten rounds without events while the others run
    streams = {1: (cols, idle), **{k: _random(stores[k], k) for k in (0, 2, 4)}}
    got = _drive(EventStreamPool(net, LR, 2, W, slots=4, chunk=4, capacity=4), streams)
    for k in streams:
        _assert_bytes_equal(got[k], want[k])


def test_reused_rows_start_from_zero(net, stores, want):
    """capacity 2, five recordings over time: every open() after the second takes a row another stream used"""
    pool = EventStreamPool(net, LR, 2, W, slots=2, chunk=4, capacity=2)
    for ks in ((0, 1), (2, 3), (4, 0)):
        got = _drive(pool, {k: _random(stores[k], k + 7) for k in ks})
        for k in ks:
            _assert_bytes_equal(got[k], want[k])


def test_counts_above_64_take_the_general_chain(stores, tmp_path):
    hot = _model(5, 70.0)
    ref = {k: _offline(hot, stores[k], tmp_path) for k in (2, 3)}
    assert all(len(r["ts"]) > 64 * 2 * 32 * 48 for r in ref.values())
    got = _drive(EventStreamPool(hot, LR, 2, W, slots=2, chunk=4, capacity=2), {k: _random(stores[k], k) for k in (2, 3)})
    for k in (2, 3):
        _assert_bytes_equal(got[k], ref[k])


def test_streams_shorter_than_n_frames(net, stores, want, tmp_path):
    lengths = (0, 1, W, 2 * W, 3 * W - 1, 3 * W)
    short = {n: _store(str(tmp_path / f"short{n}.esr"), n, max(n, 1)) for n in lengths}
    streams = {n: ([c[:n] for c in _columns(s)], [n // 2, n - n // 2]) for n, s in short.items()}
    streams["long"] = _random(stores[0], 0)                         # sharing calls with one that does emit
    got = _drive(EventStreamPool(net, LR, 2, W, slots=4, chunk=4, capacity=8), streams)
    for n in lengths:
        if n < 3 * W:
            assert all(len(v) == 0 for v in got[n].values())
        else:
            _assert_bytes_equal(got[n], _offline(net, short[n], tmp_path))
    _assert_bytes_equal(got["long"], want[0])


def test_pushes_larger_than_the_ring_force_rounds(net, stores, want):
    """whole recordings in one push each, no run() of our own: the pushes run the rounds, taking the other streams along"""
    streams = {k: (_columns(stores[k]), [len(_columns(stores[k])[2])]) for k in (0, 1, 3)}
    got = _drive(EventStreamPool(net, LR, 2, W, slots=2, chunk=2, capacity=3), streams, run=False)
    for k in streams:
        _assert_bytes_equal(got[k], want[k])


# ---- the device entries ---------------------------------------------------------------------------------------------------------
def test_state_rows_are_bit_exact_copies():
    net = _model(3, 0.6)
    dev = torch.device("cuda")
    lib = _lib.lib()
    B, L, H, Wd = 4, 3, 32, 48
    plan = net._plan(B, L, H, Wd, dev)
    nbytes = lib.esr_net_state_bytes(H, Wd)
    assert nbytes == 4 * (H // 8) * (Wd // 8) * 64 * 2 and lib.esr_net_state_bytes(0, 5) == 0
    g = torch.Generator(device=dev).manual_seed(0)
    R = 6
    pool = torch.randint(0, 256, (R, nbytes), dtype=torch.uint8, device=dev, generator=g)

    def rows(v):
        return torch.tensor(v, dtype=torch.int32, device=dev)

    def run(fn, p, tbl):
        _lib.check(getattr(lib, fn)(plan.handle, _lib.ptr(p), _lib.ptr(tbl), _lib.stream_ptr()), fn)

    for gat in ([2, 0, 2, -1], [5, 4, 3, 1], [-1, -1, -1, -1], [1, 1, 1, 1]):
        run("esr_net_gather_states", pool, rows(gat))
        out = torch.randint(0, 256, (R, nbytes), dtype=torch.uint8, device=dev, generator=g)
        keep = out.clone()
        sca = [3, -1, 0, 5]                                          # a permutation with a skipped slot
        run("esr_net_scatter_states", out, rows(sca))
        src = torch.where(rows(gat)[:, None] >= 0, pool[rows(gat).clamp_min(0).long()], torch.zeros_like(pool[:B]))
        for b, r in enumerate(sca):
            if r >= 0:
                keep[r] = src[b]
        torch.cuda.synchronize()
        assert torch.equal(out, keep), gat
    # the row holds the sample's whole state: both directions, both planes
    h = torch.randn((2, B, 64, H // 8, Wd // 8), device=dev)
    _lib.check(lib.esr_net_set_states(plan.handle, _lib.ptr(h), _lib.stream_ptr()), "esr_net_set_states")
    want = torch.stack(net.states(B, L, H, Wd))
    run("esr_net_scatter_states", pool, rows([4, 2, 0, 1]))
    net.reset_states()
    run("esr_net_gather_states", pool, rows([4, 2, 0, 1]))
    assert torch.equal(torch.stack(net.states(B, L, H, Wd)), want)
    run("esr_net_gather_states", pool, rows([1, 0, -1, 4]))
    got = torch.stack(net.states(B, L, H, Wd))
    assert torch.equal(got[:, 0], want[:, 3]) and torch.equal(got[:, 1], want[:, 2]) and torch.equal(got[:, 3], want[:, 0])
    assert not got[:, 2].any()


@pytest.mark.parametrize("pinned", [True, False])
def test_append_rings_equals_a_numpy_model(pinned):
    dev = torch.device("cuda")
    rng = np.random.default_rng(1)
    R, cap = 7, 5 * 64
    rings = [torch.zeros((R, cap), dtype=dt, device=dev) for dt in (torch.int16, torch.int16, torch.float64)]
    model = [np.zeros((R, cap), dt) for dt in (np.int16, np.int16, np.float64)]
    pos = np.zeros(R, np.int64)
    for _ in range(60):
        counts = rng.choice([0, 0, 1, 17, 64, 200, cap], R)          # streams that push nothing, and whole rings
        live = np.flatnonzero(counts)
        total = int(counts.sum())
        src = [rng.integers(-2000, 2000, total).astype(np.int16), rng.integers(0, 500, total).astype(np.int16),
               rng.standard_normal(total)]
        srct = [torch.from_numpy(s) for s in src]
        srct = [s.pin_memory() for s in srct] if pinned else [s.to(dev) for s in srct]
        desc = np.zeros(len(live), RING_DESC)
        o = 0
        for i, r in enumerate(live):
            m = int(counts[r])
            desc[i] = (*[v[r].data_ptr() for v in rings], cap, pos[r], m, o)
            j = (pos[r] + np.arange(m)) % cap
            for mc, s in zip(model, src):
                mc[r, j] = s[o:o + m]
            pos[r] += m
            o += m
        if len(live) == 0:
            continue
        desc_d = torch.from_numpy(desc.view(np.uint8)).to(dev)
        _lib.check(_lib.lib().esr_events_append_rings(_lib.ptr(desc_d), len(live), int(counts.max()), *map(_lib.ptr, srct),
                                                      _lib.stream_ptr()), "esr_events_append_rings")
        torch.cuda.synchronize()
        for ring, mc in zip(rings, model):
            assert np.array_equal(ring.cpu().numpy(), mc)
    assert pos.max() > 4 * cap                                       # every ring wrapped several times


def test_device_memory_grows_neither_with_length_nor_with_streams(net, tmp_path):
    short, long = _store(str(tmp_path / "s.esr"), 1, 12 * W + 5), _store(str(tmp_path / "l.esr"), 2, 120 * W + 5)
    pool = EventStreamPool(net, LR, 2, W, slots=2, chunk=4, capacity=2)

    def replay(stores, step):
        cols = [_columns(s) for s in stores]
        sids = [pool.open() for _ in stores]
        for a in range(0, max(len(c[2]) for c in cols), step):
            for sid, c in zip(sids, cols):
                pool.push(sid, *(v[a:a + step] for v in c))
            pool.run()
            for sid in sids:
                pool.pull(sid)
        for sid in sids:
            pool.close(sid)

    def used():
        gc.collect()
        torch.cuda.synchronize()
        return torch.cuda.memory_allocated()

    for step in (W + 1, 3 * W, 9 * W):                               # every plan and cnt2event shape exists after this
        replay([short, short], step)
    base = used()
    replay([long, long], W + 1)                                      # streams ten times longer
    assert used() <= base
    for _ in range(10):                                              # ten times capacity streams opened and closed
        replay([short, short], W + 1)
    assert used() <= base


def test_event_stream_is_a_pool_of_one(net, stores, want):
    s = EventStream(net, LR, 2, W, chunk=4)
    assert s._pool.slots == 1 and s._pool.capacity == 1
    cols = _columns(stores[4])
    s.push(*cols)
    _assert_bytes_equal(_join([s.pull(wait=True), s.close()]), want[4])
