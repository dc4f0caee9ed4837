"""End-to-end hot path on one GPU: raw events -> count tensors -> DeepRecurrNet over sliding windows (state carried)
-> SR count tensors -> time-sorted SR event lists.

This is the per-batch body of the reference's inference loop (infer_ours_cnt.py:54-75) together with the dataloader
encodings it depends on (dataloader/h5dataset.py:508-528 `inp_scaled_cnt`, dataloader/h5dataloader.py:229-231
sliding windows) and the redistribution API (dataloader/cython_cnt2event/cnt2event_api.py:25-35), with every stage
on the GPU and no intermediate host round trip:

    host events (pinned) --H2D--> esr_scatter_cnt (LR->HR lift fused) --> frame bank [B*L,2,kH,kW]
        --> L-N+1 x esr_net_forward (N = the model's num_frame; windows addressed by index into the bank; ConvGRU state carried)
        --> esr_expand_count / esr_expand_emit on all window outputs --> events [B*(L-N+1), maxlen, 4] --D2H--> host
"""
import torch

from . import encodings
from .expand import FusedCnt2Event, expand, expand_begin, expand_finish


class EventSRPipeline:
    def __init__(self, model, B, L, lr_size, scale, device):
        self.model, self.B, self.L, self.scale, self.dev = model, B, L, scale, device
        self.lr_size = (int(lr_size[0]), int(lr_size[1]))
        self.hr_size = (self.lr_size[0] * scale, self.lr_size[1] * scale)
        N = model._cfg["num_frame"]                  # frames per window (the config's SEQN)
        if L < N:
            raise ValueError(f"EventSRPipeline: L={L} frames per sequence is fewer than the model's num_frame={N}")
        self.num_frame = N
        self.window_index = [
            torch.tensor([b * L + w + n for b in range(B) for n in range(N)], dtype=torch.int32, device=device)
            for w in range(L - N + 1)]
        self.sr_bias = None      # optional synthetic counts added to the SR output before redistribution (bench only)
        self.bank = torch.zeros((B * L, 2, self.hr_size[0], self.hr_size[1]), dtype=torch.float32, device=device)
        self._graph = None
        self._graph_sr = None
        self._graphs = []
        self._host_events = None
        self._copy_stream = None
        self.sequence_plan = True
        self.graph_launches = 0

    def _windows(self):
        self.model.reset_states()                    # per sequence batch (train_ours_cnt_seq.py:213-216)
        if self.sequence_plan:
            sr = self.model.forward_sequence(self.bank.view(self.B, self.L, 2, self.hr_size[0], self.hr_size[1]))
        else:                                        # the reference's loop: one forward per window
            sr = torch.cat([self.model(self.bank, frame_index=idx) for idx in self.window_index], 0)
        if self.sr_bias is not None:
            sr = sr + self.sr_bias
        return sr

    @torch.no_grad()
    def capture(self, slots=2, fused_rows=None, fused_max_count=None):
        """Capture the whole window chain AND the redistribution of its output (cnt2event with linear timestamps, the mode the
        reference's inference uses) into CUDA graphs: the plan allocates nothing and never synchronises, the fused redistribution
        (csrc/expand_fused.cu) sizes its output on the device, so one replay = one launch from the host and the only
        synchronisation of a step is the final one.  `slots` graphs with their own output buffers are recorded so that batch i's
        event list can drain to the host while batch i+1 is being computed (submit_host / finish / collect).
        The row capacity / largest count the fused kernels are recorded with come from an eager run on the data currently in the
        frame bank (x1.5 / x2); a step that exceeds them is finished by the general chain and the graphs are re-recorded larger."""
        from . import _lib
        sr = self._windows()                         # warm-up: packs parameters, builds the plan, sets smem attributes
        ev = expand(sr, 0, 0)
        if fused_rows is None:
            fused_rows = int(ev.shape[0] * ev.shape[1] * 1.5) + 65536
        if fused_max_count is None:
            fused_max_count = 2 * max(4, int(torch.round(sr).max().item()))
        torch.cuda.synchronize()
        self._graphs = []
        for _ in range(slots):
            g = torch.cuda.CUDAGraph()
            fused = FusedCnt2Event(sr.shape[0], sr.shape[2], sr.shape[3], self.dev, fused_rows, fused_max_count)
            s = torch.cuda.Stream(device=self.dev)
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                fused.enqueue(self._windows())
            torch.cuda.current_stream().wait_stream(s)
            c0 = _lib.lib().esr_launch_count()
            with torch.cuda.graph(g):
                out_sr = self._windows()
                fused.enqueue(out_sr)
            self.graph_launches = int(_lib.lib().esr_launch_count() - c0)   # kernels of ours inside one replay
            self._graphs.append({"graph": g, "sr": out_sr, "fused": fused, "busy": None})
        self._graph, self._graph_sr = self._graphs[0]["graph"], self._graphs[0]["sr"]

    def _grow(self, rows, mx):
        """A step fell outside the recorded capacity: record the graphs again, larger (takes effect from the next step)."""
        f = self._graphs[0]["fused"]
        if rows <= f.cap and f.mcap >= 64:
            return                                   # a count above 64: outside the fused path whatever the graphs were recorded with
        self.capture(len(self._graphs), max(int(rows * 1.5) + 65536, f.cap), max(2 * mx, f.mcap))

    def _replay(self, slot, mode):
        """One replay of graph `slot`; returns (sr, events or None) once the device has finished it."""
        gs = self._graphs[slot]
        if gs["busy"] is not None:
            torch.cuda.current_stream().wait_event(gs["busy"])     # the previous event list of this slot is still draining
            gs["busy"] = None
        gs["graph"].replay()
        return gs

    @torch.no_grad()
    def run_device(self, xs, ys, ps, frame_off, n_max_frame, mode=0):
        """All inputs already on the GPU.  Returns (sr_cnt [B*(L-N+1),2,kH,kW], events [B*(L-N+1),maxlen,4]) on the GPU.
        Sample order of the outputs: window-major (w * B + b).  With captured graphs both tensors are views of the graph's static
        buffers: valid until the next call."""
        encodings.encode_frames(xs, ys, ps, frame_off, lr_size=self.lr_size, hr_size=self.hr_size,
                                n_max_frame=n_max_frame, out=self.bank)
        if self._graph is None:
            sr = self._windows()
            return sr, expand(sr, 0, mode)
        gs = self._replay(0, mode)
        sr = gs["sr"]
        if mode != 0:
            return sr, expand(sr, 0, mode)
        torch.cuda.current_stream().synchronize()
        events, rows, mx = gs["fused"].result()
        if events is None:
            events = expand(sr, 0, 0)
            self._grow(rows, mx)
        return sr, events

    # ---- asynchronous end-to-end API, software-pipelined in three stages ------------------------------------------
    #   submit_host(i) : H2D of the events, encode, network + redistribution (one CUDA graph replay), statistics -> pinned host
    #                    memory; returns at once
    #   finish(i)      : waits for batch i, reads its size from the statistics, starts the D2H of the event list on a side
    #                    stream into one of two pinned buffers
    #   collect(i)     : wait for that copy
    # Calling submit_host(i+1) BEFORE finish(i) keeps the GPU busy with batch i+1 while the host handles batch i (bench.py's
    # e2e loop); submit / collect alone (finish implied) is the simple two-in-flight form.
    @torch.no_grad()
    def submit_host(self, xs_h, ys_h, ps_h, off_h, n_max_frame, mode=0):
        if self._copy_stream is None:
            self._copy_stream = torch.cuda.Stream(device=self.dev)
            self._host_pool = [None, None]
            self._slot = 0
        xs = xs_h.to(self.dev, non_blocking=True)
        ys = ys_h.to(self.dev, non_blocking=True)
        ps = ps_h.to(self.dev, non_blocking=True)
        off = off_h.to(self.dev, non_blocking=True)
        encodings.encode_frames(xs, ys, ps, off, lr_size=self.lr_size, hr_size=self.hr_size, n_max_frame=n_max_frame, out=self.bank)
        slot = self._slot
        self._slot ^= 1
        handle = {"ctx": None, "gs": None, "mode": mode, "slot": slot, "host": None, "done": None}
        if self._graph is not None and mode == 0 and len(self._graphs) > slot:
            handle["gs"] = self._replay(slot, mode)
            handle["ready"] = torch.cuda.Event()
            handle["ready"].record()
        else:
            if self._graph is not None:
                gs = self._replay(0, mode)
                sr = gs["sr"].clone()                # the graph's output buffer is overwritten by the next replay
            else:
                sr = self._windows()
            handle["ctx"] = expand_begin(sr, 0, mode)
        return handle

    @torch.no_grad()
    def finish(self, handle):
        if handle["done"] is not None:
            return handle
        gs = handle["gs"]
        if gs is not None:
            handle["ready"].synchronize()
            events, rows, mx = gs["fused"].result()
            if events is None:                       # outside the recorded capacity: general chain on the same SR counts
                events = expand(gs["sr"], 0, 0)
                handle["grow"] = (rows, mx)
        else:
            events = expand_finish(handle["ctx"], handle["mode"])
            handle["ctx"] = None
        slot = handle["slot"]
        n = events.numel()
        buf = self._host_pool[slot]
        if buf is None or buf.numel() < n:
            buf = torch.empty((int(n * 1.25) + 1024,), dtype=torch.float32).pin_memory()
            self._host_pool[slot] = buf
        host = buf[:n].view(events.shape)
        if gs is not None and handle.get("grow") is None:
            ready = handle["ready"]                  # the rows were complete when the replay ended: do not queue behind later batches
        else:
            ready = torch.cuda.Event()
            ready.record()
        with torch.cuda.stream(self._copy_stream):
            self._copy_stream.wait_event(ready)
            host.copy_(events, non_blocking=True)
            done = torch.cuda.Event()
            done.record()
        events.record_stream(self._copy_stream)
        if gs is not None:
            gs["busy"] = done                        # the next replay of this slot overwrites the static event buffer
        handle["host"], handle["done"] = host, done
        return handle

    def collect(self, handle):
        self.finish(handle)
        handle["done"].synchronize()
        if handle.get("grow") is not None:           # nothing of the old graphs is in flight any more on this handle's slot
            rows, mx = handle.pop("grow")
            torch.cuda.synchronize()
            self._grow(rows, mx)
        return handle["host"]

    @torch.no_grad()
    def run_host(self, xs_h, ys_h, ps_h, off_h, n_max_frame, mode=0):
        """Pinned host buffers in, host event tensor out (the e2e path: H2D and D2H inside)."""
        xs = xs_h.to(self.dev, non_blocking=True)
        ys = ys_h.to(self.dev, non_blocking=True)
        ps = ps_h.to(self.dev, non_blocking=True)
        off = off_h.to(self.dev, non_blocking=True)
        _, events = self.run_device(xs, ys, ps, off, n_max_frame, mode)
        # D2H into a reusable pinned buffer (pageable `.cpu()` copies run at a fraction of the link rate)
        n = events.numel()
        if self._host_events is None or self._host_events.numel() < n:
            self._host_events = torch.empty((int(n * 1.25) + 1024,), dtype=torch.float32).pin_memory()
        host = self._host_events[:n].view(events.shape)
        host.copy_(events, non_blocking=True)
        torch.cuda.current_stream().synchronize()
        return host
