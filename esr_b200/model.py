"""H100 implementation of the reference's `models/model.py` network class.

`DeepRecurrNet` keeps the reference's constructor signature, `forward(BxNx2xHxW) -> Bx2xHxW`, `reset_states()` and
state_dict key names (models/model.py:294-344; 68 tensors, SURVEY 8b), so a reference checkpoint loads with
`load_state_dict` and `infer_ours_cnt.py` can instantiate it through `eval(config['model']['name'])(**args)`.
The parameters are ordinary `nn.Parameter`s (DDP-wrappable); the forward pass is the C++/CUDA plan behind
`esr_net_*` (include/esr_b200.h).  There is no PyTorch/CPU fallback: a CPU tensor or a missing library raises.

Two execution paths, both sm_90a kernels behind the C ABI:
  * torch.no_grad(): the fused inference plan (esr_net_*), states kept inside the plan's workspace;
  * gradients enabled (training, train_ours_cnt_seq.py:217-232): esr_b200.train.forward_window -- the same network
    composed from differentiable operators (esr_conv2d_forward/backward, esr_dcn_v2_forward/backward), with the
    carried ConvGRU states kept as graph tensors so that backward runs through time like the reference's.
"""
import ctypes
import math

import torch
import torch.nn as nn

from . import _lib


class _Conv(nn.Module):
    """parameter holder with the reference ConvLayer's attribute name (`conv2d`)  (models/submodules.py:159-200)"""

    def __init__(self, cin, cout, k):
        super().__init__()
        self.conv2d = nn.Conv2d(cin, cout, k, 1, k // 2)


class _Res(nn.Module):
    """ResidualBlock parameter holder: conv1, conv2 (models/submodules.py:347-409)"""

    def __init__(self, c):
        super().__init__()
        self.conv1 = nn.Conv2d(c, c, 3, 1, 1)
        self.conv2 = nn.Conv2d(c, c, 3, 1, 1)


class _GRU(nn.Module):
    """ConvGRU parameter holder with the reference's init (models/submodules.py:474-494)"""

    def __init__(self, c):
        super().__init__()
        self.reset_gate = nn.Conv2d(2 * c, c, 3, padding=1)
        self.update_gate = nn.Conv2d(2 * c, c, 3, padding=1)
        self.out_gate = nn.Conv2d(2 * c, c, 3, padding=1)
        for g in (self.reset_gate, self.update_gate, self.out_gate):
            nn.init.orthogonal_(g.weight)
            nn.init.constant_(g.bias, 0.0)


class _Recurrent(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.conv = _Conv(c, c, 3)
        self.recurrent_block = _GRU(c)


class _DCN(nn.Module):
    """DCN_sep parameter holder with the reference's init (models/DCNv2/dcn_v2.py:98-132,197-212)"""

    def __init__(self, c, groups=8):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(c, c, 3, 3))
        self.bias = nn.Parameter(torch.zeros(c))
        stdv = 1.0 / math.sqrt(c * 9)
        self.weight.data.uniform_(-stdv, stdv)
        self.conv_offset_mask = nn.Conv2d(c, groups * 3 * 9, 3, 1, 1, bias=True)
        self.conv_offset_mask.weight.data.zero_()
        self.conv_offset_mask.bias.data.zero_()


class _MLP(nn.Module):
    def __init__(self, i, h, o):
        super().__init__()
        self.layers = nn.ModuleList([nn.Linear(i, h), nn.Linear(h, o)])


class _FeatsExtract(nn.Module):
    def __init__(self, b):
        super().__init__()
        self.convblock = nn.ModuleList([_Conv(b, 2 * b, 3), _Conv(2 * b, 4 * b, 3), _Conv(4 * b, 8 * b, 3)])


class _TimePropagation(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.pred_map = nn.Sequential(_Conv(2 * c, c, 3), _Conv(c, 1, 3))
        self.local_fusion = nn.Sequential(_Res(3 * c), _Conv(3 * c, c, 3))
        self.lstm = _Recurrent(c)
        self.global_fusion = _Conv(2 * c, c, 1)


class _STFusion(nn.Module):
    def __init__(self, c, num_frame):
        super().__init__()
        self.offset = nn.Sequential(_Conv(2 * c, c, 3), _Conv(c, c, 3))
        self.dcn = _DCN(c, 8)
        self.convblock = nn.Sequential(_Conv(2 * c, c, 3), _Conv(c, c, 3))
        self.kernel = _Conv(c, 2, 1)
        self.fc = nn.Sequential(_MLP(c, c // 2, 2 * c), nn.Sigmoid())
        self.dcn_fusion = nn.Sequential(_Conv(2 * c, c, 3), _Conv(c, c, 3))
        self.dense_fusion = nn.Sequential(_Conv(num_frame * c, c, 3), _Conv(c, c, 3))
        self.attens = nn.ModuleList([_Conv(c, 1, 3), _Conv(c // 2, 1, 3), _Conv(c // 4, 1, 3)])
        self.recons = nn.ModuleList([_Conv(c, c // 2, 3), _Conv(c // 2, c // 4, 3), _Conv(c // 4, c // 8, 3)])


class _Plan:
    """One esr_net_t for a (B, L, H, W, device) with its workspace (L = num_frame: the reference's single-window forward)."""

    def __init__(self, B, N, L, H, W, blob, device):
        lib = _lib.lib()
        self.key = (B, L, H, W)
        nbytes = lib.esr_net_workspace_bytes(B, N, L, H, W)
        self.ws = torch.empty((nbytes,), dtype=torch.uint8, device=device)
        self.handle = ctypes.c_void_p()
        _lib.check(lib.esr_net_create(ctypes.byref(self.handle), B, N, L, H, W, _lib.ptr(blob), _lib.ptr(self.ws), nbytes,
                                      _lib.stream_ptr()), "esr_net_create")

    def close(self):
        if self.handle:
            _lib.lib().esr_net_destroy(self.handle)
            self.handle = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def load_checkpoint(path, weights_only=True):
    """A checkpoint file on the CPU -> (the loaded object, the model's state_dict): {'model': {'states': ...}} as the
    reference's trainer and esr_b200.trainer save it (infer_ours_cnt.py:118-127), or a bare state_dict.
    weights_only=False unpickles anything (the reference's checkpoints may hold numpy scalars): only for trusted files."""
    cpt = torch.load(path, map_location="cpu", weights_only=weights_only)
    return cpt, (cpt["model"]["states"] if "model" in cpt else cpt)


class DeepRecurrNet(nn.Module):
    def __init__(self, inch=2, basech=16, num_frame=3, norm=None, activation='relu',
                 has_ltc=True, has_gtc=True, gtc_frozen=False,
                 has_dcnatten=True, has_scaleaggre=True):
        super().__init__()
        self.down_scale = 8
        self._cfg = dict(inch=inch, basech=basech, num_frame=num_frame, norm=norm, activation=activation, has_ltc=has_ltc,
                         has_gtc=has_gtc, gtc_frozen=gtc_frozen, has_dcnatten=has_dcnatten, has_scaleaggre=has_scaleaggre)
        self.head = _Conv(inch, basech, 3)
        self.feat_extract = _FeatsExtract(basech)
        self.time_propagate = _TimePropagation(8 * basech)
        self.spacetime_fuse = _STFusion(8 * basech, num_frame)
        self.tail = _Conv(basech, inch, 3)
        self._plans = {}
        self._blob = None
        self._blob_sig = None
        self._train_states = None          # [h_fwd, h_rev] with autograd history (training path)

    # ------------------------------------------------------------------------------------------
    def _check_supported(self):
        c = self._cfg
        nf = c["num_frame"]
        ok = (c["inch"] == 2 and c["basech"] == 8 and isinstance(nf, int) and nf >= 3 and nf % 2 == 1 and c["norm"] is None
              and c["activation"] == "relu" and c["has_ltc"] and c["has_gtc"] and not c["gtc_frozen"] and c["has_dcnatten"]
              and c["has_scaleaggre"])
        if not ok:
            raise _lib.ESRError("esr_b200.DeepRecurrNet: the sm_90a plan implements the shipped configuration "
                                "(inch=2, basech=8, norm=None, relu, all blocks on; config/train_ours_enfssyn.yml:21-26) "
                                f"with an odd num_frame >= 3 (models/model.py:163-166); got {c}")

    def _packed_params(self, device):
        params = list(self.state_dict(keep_vars=True).values())
        sig = tuple((p.data_ptr(), p._version) for p in params) + (str(device),)
        if self._blob is None or sig != self._blob_sig:
            L = _lib.lib()
            tensors = [p.detach().to(device=device, dtype=torch.float32).contiguous() for p in params]
            arr = (ctypes.c_void_p * len(tensors))(*[t.data_ptr() for t in tensors])
            if self._blob is None or self._blob.device != device:
                self._blob = torch.empty((L.esr_net_param_bytes_n(self._cfg["num_frame"]),), dtype=torch.uint8, device=device)
                for p in self._plans.values():
                    p.close()
                self._plans = {}
            _lib.check(L.esr_net_pack_params_n(self._cfg["num_frame"], arr, _lib.ptr(self._blob), _lib.stream_ptr()),
                       "esr_net_pack_params_n")
            torch.cuda.current_stream().synchronize()      # `tensors` may be temporaries
            self._blob_sig = sig
        return self._blob

    def _plan(self, B, L, H, W, device):
        blob = self._packed_params(device)
        key = (B, L, H, W)
        if key not in self._plans:
            self._plans[key] = _Plan(B, self._cfg["num_frame"], L, H, W, blob, device)
        return self._plans[key]

    # ------------------------------------------------------------------------------------------
    def reset_states(self):
        """models/model.py:311-312: forget the carried ConvGRU states (of every cached shape)."""
        self._train_states = None
        for p in self._plans.values():
            with torch.cuda.device(p.ws.device):
                _lib.check(_lib.lib().esr_net_reset_states(p.handle, _lib.stream_ptr()), "esr_net_reset_states")

    def reset_sample_states(self, indices):
        """Forget the carried ConvGRU states of the batch samples `indices` only (of every cached inference plan whose batch
        holds them); the other samples keep theirs.  Lets a batch of independent recordings start a new one in one slot."""
        idx = [int(i) for i in indices]
        for p in self._plans.values():
            B = p.key[0]
            with torch.cuda.device(p.ws.device):
                for b in idx:
                    if not 0 <= b < B:
                        continue
                    _lib.check(_lib.lib().esr_net_reset_sample_states(p.handle, b, _lib.stream_ptr()), "esr_net_reset_sample_states")

    def states(self, B, L, H, W):
        """The carried states [h_fwd, h_rev] (each Bx64xhxw) of the plan for this shape -- the reference's
        `time_propagate.states`."""
        p = self._plans[(B, L, H, W)]
        h, w = (H + 7) // 8, (W + 7) // 8
        out = torch.empty((2, B, 64, h, w), dtype=torch.float32, device=p.ws.device)
        with torch.cuda.device(p.ws.device):
            _lib.check(_lib.lib().esr_net_get_states(p.handle, _lib.ptr(out), _lib.stream_ptr()), "esr_net_get_states")
        return [out[0], out[1]]

    def forward(self, input, frame_index=None):
        """input: BxNx2xHxW fp32 CUDA tensor -> Bx2xHxW.  (frame_index: optional int32 [B*N] selecting frames out of a
        [n_frames,2,H,W] bank instead -- zero-copy sliding windows; not part of the reference signature.)"""
        self._check_supported()
        if not input.is_cuda:
            raise _lib.ESRError("esr_b200.DeepRecurrNet.forward needs a CUDA tensor (there is no CPU path)")
        if torch.is_grad_enabled() and (input.requires_grad or any(p.requires_grad for p in self.parameters())):
            if frame_index is not None:
                raise _lib.ESRError("esr_b200.DeepRecurrNet: frame banks are an inference feature")
            from . import train
            # L == num_frame: the reference's single window; L > num_frame: all sliding windows in one graph (window-major)
            out, self._train_states = train.forward_sequence(self, input, self._train_states)
            return out
        if frame_index is None and input.dim() == 5 and input.shape[1] > self._cfg["num_frame"]:
            return self.forward_sequence(input)
        x = input.detach()
        if x.dtype != torch.float32 or not x.is_contiguous():
            x = x.float().contiguous()
        if frame_index is None:
            B, N, C, H, W = x.shape
        else:
            _, C, H, W = x.shape
            N = self._cfg["num_frame"]
            B = frame_index.numel() // N
        assert C == 2
        with torch.cuda.device(x.device):
            plan = self._plan(B, N, H, W, x.device)
            out = torch.empty((B, 2, H, W), dtype=torch.float32, device=x.device)
            _lib.check(_lib.lib().esr_net_forward(plan.handle, _lib.ptr(x), _lib.ptr(frame_index), _lib.ptr(out),
                                                  _lib.stream_ptr()), "esr_net_forward")
        return out

    def forward_sequence(self, frames):
        """frames: BxLx2xHxW (L >= N = num_frame) -> (L-N+1)*B x 2 x H x W, window-major (w*B + b): the L-N+1
        sliding-window forwards of the reference's loop (train_ours_cnt_seq.py:217-231) in ONE plan -- per-frame layers run
        once per frame, state-independent layers once for all windows, only the ConvGRU chain is serial.  The carried state
        is read at the start and left as after the last window, exactly as L-N+1 successive forward() calls would."""
        self._check_supported()
        if not frames.is_cuda:
            raise _lib.ESRError("esr_b200.DeepRecurrNet.forward_sequence needs a CUDA tensor (there is no CPU path)")
        if torch.is_grad_enabled() and (frames.requires_grad or any(p.requires_grad for p in self.parameters())):
            return self.forward(frames)
        x = frames.detach()
        if x.dtype != torch.float32 or not x.is_contiguous():
            x = x.float().contiguous()
        B, L, C, H, W = x.shape
        N = self._cfg["num_frame"]
        assert C == 2 and L >= N
        with torch.cuda.device(x.device):
            plan = self._plan(B, L, H, W, x.device)
            out = torch.empty(((L - N + 1) * B, 2, H, W), dtype=torch.float32, device=x.device)
            _lib.check(_lib.lib().esr_net_forward(plan.handle, _lib.ptr(x), None, _lib.ptr(out), _lib.stream_ptr()),
                       "esr_net_forward")
        return out
