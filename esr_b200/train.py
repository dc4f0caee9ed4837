"""Training step of the hot path (SURVEY.md 8a row 17; train_ours_cnt_seq.py:206-235, 767-782).

The reference sums MSELoss(pred, gt) over the L-N+1 windows of a sequence (ConvGRU state carried, so gradients flow back
through time across windows), calls backward once, lets DDP all-reduce the 1 813 120 gradients and steps
Adam(lr, weight_decay, amsgrad).  Here

  * every ConvLayer (models/submodules.py:159-200) is `conv2d` below: an autograd.Function whose forward AND backward
    are the sm_90a operators esr_conv2d_forward / esr_conv2d_backward (wgmma implicit GEMM for the 64-multiple
    layers incl. dx and dw, CUDA-core kernels for the narrow full-resolution layers; include/esr_b200.h);
  * DCN_sep (models/DCNv2/dcn_v2.py:17-68) is `dcn_v2`: esr_dcn_v2_forward / esr_dcn_v2_backward;
  * the loss and the optimizer are esr_mse_loss / esr_adam_step (one launch over the flat parameter buffer);
  * autograd itself, the concatenations / gating products / bilinear x2 / global max / 64-32-128 MLP between those
    operators are torch on the GPU -- plumbing, < 2 % of the step's FLOPs.

`forward_window` is the differentiable counterpart of esr_b200.DeepRecurrNet.forward (which runs the fused inference
plan and cannot be differentiated); DeepRecurrNet.forward dispatches here when gradients are enabled.
"""
import contextlib
import math

import torch
import torch.nn.functional as F

from . import _lib, dcn_v2_ext

_ACT = {None: 0, "none": 0, "relu": 1, "sigmoid": 2, "tanh": 3}


def _ws(nbytes, device):
    return torch.empty((max(int(nbytes), 256),), dtype=torch.uint8, device=device)


def deterministic():
    """True when the training operators must be bitwise reproducible: torch.use_deterministic_algorithms(True) or
    torch.backends.cudnn.deterministic = True (the reference trainer's init_seeds sets the latter, train_ours_cnt_seq.py:30-46).
    Read at every call.  In this mode every gradient / loss reduction runs from per-block partials in a fixed order (or in
    int64 fixed point for the DCN grad_input), and paths that have no such variant raise ESRError."""
    return torch.are_deterministic_algorithms_enabled() or bool(torch.backends.cudnn.deterministic)


def _flags():
    return _lib.DETERMINISTIC if deterministic() else 0


_DEFERRED = None        # None: off.  dict key -> [sink, [(x, y, dy), ...]] while a train_step collects weight-shared layers


class _defer_weight_grads:
    """Inside this context, convolutions called with `defer=(key, sink)` return only dx from backward and stash (x, y, dy);
    flush() then computes dw / db of each key ONCE over the concatenated batch (the ConvGRU applies the same weights at
    every step of every window: 18 small weight-gradient launches + 18 x 6 M atomics become one) and hands them to sink."""

    def __enter__(self):
        global _DEFERRED
        self.prev, _DEFERRED = _DEFERRED, {}
        return self

    def __exit__(self, *exc):
        global _DEFERRED
        _DEFERRED = self.prev

    @staticmethod
    def flush():
        for key, (sink, items, cfg) in list(_DEFERRED.items()):
            if not items:
                continue
            y = torch.cat([t[3] for t in items], 0)
            dy = torch.cat([t[4] for t in items], 0)
            shp = items[0][2]
            shape = (sum(t[2][0] for t in items),) + tuple(shp[1:])
            if items[0][1] is not None:                           # split operands [2 planes][B][...]: concatenate per plane
                x, xs = None, torch.cat([t[1].view(2, t[2][0], -1) for t in items], 1).reshape(-1)
            else:
                x, xs = torch.cat([t[0] for t in items], 0), None
            w, stride, act = cfg
            dw, db = _conv2d_backward_raw(x, w, y, dy, stride, act, need_dx=False, need_dw=True, x_split=xs, x_shape=shape)[1:]
            sink(dw, db)
            items.clear()


def _conv2d_backward_raw(x, w, y, dy, stride, act, need_dx=True, need_dw=True, x_split=None, x_shape=None):
    B, Cin, H, W = x_shape if x is None else x.shape
    Cout, _, k, _ = w.shape
    L = _lib.lib()
    dx = torch.empty((B, Cin, H, W), dtype=torch.float32, device=w.device) if need_dx else None
    dw = torch.empty_like(w) if need_dw else None
    db = torch.empty((Cout,), dtype=torch.float32, device=w.device) if need_dw else None
    flags = _flags()
    with torch.cuda.device(w.device):
        nbytes = L.esr_conv2d_workspace_bytes_ex(B, Cin, H, W, Cout, k, stride, flags)
        ws = _ws(nbytes, w.device)
        _lib.check(L.esr_conv2d_backward_ex(_lib.ptr(x), _lib.ptr(x_split), _lib.ptr(w), _lib.ptr(y), _lib.ptr(dy), B, Cin, H, W, Cout, k,
                                            stride, act, _lib.ptr(dx), _lib.ptr(dw), _lib.ptr(db), flags, _lib.ptr(ws), nbytes,
                                            _lib.stream_ptr()), "esr_conv2d_backward")
    return dx, dw, db


class _Conv2dFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, b, stride, act, defer=None):
        ctx.defer = defer if (_DEFERRED is not None and defer is not None) else None
        if not x.is_cuda:
            raise _lib.ESRError("esr_b200.train.conv2d needs CUDA tensors (there is no CPU path)")
        x, w, b = x.contiguous().float(), w.contiguous().float(), b.contiguous().float()
        B, Cin, H, W = x.shape
        Cout, _, k, _ = w.shape
        pad = k // 2
        Ho, Wo = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
        L = _lib.lib()
        y = torch.empty((B, Cout, Ho, Wo), dtype=torch.float32, device=x.device)
        with torch.cuda.device(x.device):
            nbytes = L.esr_conv2d_workspace_bytes(B, Cin, H, W, Cout, k, stride)
            ws = _ws(nbytes, x.device)
            # layers whose dw also runs on the tensor cores keep x in the split-bf16 operand format for the backward
            # (same bytes as fp32; the backward then needs neither x nor a second conversion)
            nsplit = L.esr_conv2d_split_bytes(B, Cin, H, W, Cout, k, stride) if ctx.needs_input_grad[1] else 0
            xs = torch.empty((nsplit,), dtype=torch.uint8, device=x.device) if nsplit else None
            _lib.check(L.esr_conv2d_forward(_lib.ptr(x), _lib.ptr(w), _lib.ptr(b), B, Cin, H, W, Cout, k, stride, act,
                                            _lib.ptr(y), _lib.ptr(xs), _lib.ptr(ws), nbytes, _lib.stream_ptr()), "esr_conv2d_forward")
        ctx.has_split = xs is not None
        ctx.save_for_backward(xs if xs is not None else x, w, y)
        ctx.x_shape = tuple(x.shape)
        ctx.cfg = (stride, act)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, w, y = ctx.saved_tensors
        stride, act = ctx.cfg
        dy = dy.contiguous().float()
        xs = x if ctx.has_split else None                              # saved split operand instead of x itself
        x = None if ctx.has_split else x
        if ctx.defer is not None and _DEFERRED is not None and ctx.needs_input_grad[0]:
            key, sink = ctx.defer
            _DEFERRED.setdefault(key, [sink, [], (w, stride, act)])[1].append((x, xs, ctx.x_shape, y, dy))
            dx = _conv2d_backward_raw(x, w, y, dy, stride, act, need_dx=True, need_dw=False, x_split=xs, x_shape=ctx.x_shape)[0]
            return dx, None, None, None, None, None
        dx, dw, db = _conv2d_backward_raw(x, w, y, dy, stride, act, need_dx=ctx.needs_input_grad[0], x_split=xs, x_shape=ctx.x_shape)
        return dx, dw, db, None, None, None


def conv2d(x, w, b, stride=1, act=None, defer=None):
    """act(conv2d(x, w, b, stride, padding=k//2)), differentiable; k = 3 or 1 (ConvLayer, models/submodules.py:159-200).
    defer=(key, sink): see _defer_weight_grads."""
    return _Conv2dFn.apply(x, w, b, int(stride), _ACT[act], defer)


class _DCNFn(torch.autograd.Function):
    """_DCNv2 (models/DCNv2/dcn_v2.py:17-68): same save_for_backward set, same five gradients."""

    @staticmethod
    def forward(ctx, inp, offset, mask, weight, bias, dg):
        ctx.dg = dg
        ctx.save_for_backward(inp, offset, mask, weight, bias)
        return dcn_v2_ext.dcn_v2_forward(inp, weight, bias, offset, mask, 3, 3, 1, 1, 1, 1, 1, 1, dg)

    @staticmethod
    def backward(ctx, grad_output):
        inp, offset, mask, weight, bias = ctx.saved_tensors
        gi, go, gm, gw, gb = dcn_v2_ext.dcn_v2_backward(inp, weight, bias, offset, mask, grad_output.contiguous(), 3, 3, 1, 1,
                                                        1, 1, 1, 1, ctx.dg)
        return gi, go, gm, gw, gb, None


def dcn_v2(inp, offset, mask, weight, bias, dg=8):
    return _DCNFn.apply(inp.contiguous(), offset.contiguous(), mask.contiguous(), weight, bias, dg)


class _Up2Fn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        x = x.contiguous().float()
        B, C, H, W = x.shape
        y = torch.empty((B, C, 2 * H, 2 * W), dtype=torch.float32, device=x.device)
        with torch.cuda.device(x.device):
            _lib.check(_lib.lib().esr_upsample2x_forward(_lib.ptr(x), B * C, H, W, _lib.ptr(y), _lib.stream_ptr()), "esr_upsample2x_forward")
        return y

    @staticmethod
    def backward(ctx, dy):
        dy = dy.contiguous().float()
        B, C, H2, W2 = dy.shape
        dx = torch.empty((B, C, H2 // 2, W2 // 2), dtype=torch.float32, device=dy.device)
        with torch.cuda.device(dy.device):
            _lib.check(_lib.lib().esr_upsample2x_backward(_lib.ptr(dy), B * C, H2 // 2, W2 // 2, _lib.ptr(dx), _lib.stream_ptr()),
                       "esr_upsample2x_backward")
        return dx


def upsample2x(x):
    """F.interpolate(x, scale_factor=2, mode='bilinear', align_corners=False) (UpsampleConvLayer, models/submodules.py:290)."""
    return _Up2Fn.apply(x)


class _GruHRFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, h, zr):
        h, zr = h.contiguous(), zr.contiguous()
        out = torch.empty_like(h)
        B, chw = h.shape[0], h[0].numel()
        with torch.cuda.device(h.device):
            _lib.check(_lib.lib().esr_gru_hr(_lib.ptr(h), _lib.ptr(zr), B, chw, _lib.ptr(out), _lib.stream_ptr()), "esr_gru_hr")
        ctx.save_for_backward(h, zr)
        return out

    @staticmethod
    def backward(ctx, g):
        h, zr = ctx.saved_tensors
        g = g.contiguous()
        dh, dzr = torch.empty_like(h), torch.empty_like(zr)
        with torch.cuda.device(h.device):
            _lib.check(_lib.lib().esr_gru_hr_backward(_lib.ptr(h), _lib.ptr(zr), _lib.ptr(g), h.shape[0], h[0].numel(), _lib.ptr(dh),
                                                      _lib.ptr(dzr), _lib.stream_ptr()), "esr_gru_hr_backward")
        return dh, dzr


class _GruBlendFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, h, zr, o):
        h, zr, o = h.contiguous(), zr.contiguous(), o.contiguous()
        out = torch.empty_like(h)
        with torch.cuda.device(h.device):
            _lib.check(_lib.lib().esr_gru_blend(_lib.ptr(h), _lib.ptr(zr), _lib.ptr(o), h.shape[0], h[0].numel(), _lib.ptr(out),
                                                _lib.stream_ptr()), "esr_gru_blend")
        ctx.save_for_backward(h, zr, o)
        return out

    @staticmethod
    def backward(ctx, g):
        h, zr, o = ctx.saved_tensors
        g = g.contiguous()
        dh, dzr, do = torch.empty_like(h), torch.empty_like(zr), torch.empty_like(o)
        with torch.cuda.device(h.device):
            _lib.check(_lib.lib().esr_gru_blend_backward(_lib.ptr(h), _lib.ptr(zr), _lib.ptr(o), _lib.ptr(g), h.shape[0], h[0].numel(),
                                                         _lib.ptr(dh), _lib.ptr(dzr), _lib.ptr(do), _lib.stream_ptr()),
                       "esr_gru_blend_backward")
        return dh, dzr, do


class _MSEFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pred, target):
        pred, target = pred.contiguous().float(), target.contiguous().float()
        loss = torch.empty((1,), dtype=torch.float32, device=pred.device)
        grad = torch.empty_like(pred)
        flags, L = _flags(), _lib.lib()
        with torch.cuda.device(pred.device):
            nbytes = L.esr_mse_loss_workspace_bytes_ex(pred.numel(), flags)
            ws = _ws(nbytes, pred.device) if nbytes else None
            _lib.check(L.esr_mse_loss_ex(_lib.ptr(pred), _lib.ptr(target), pred.numel(), _lib.ptr(loss), _lib.ptr(grad), 1.0, flags,
                                         _lib.ptr(ws), nbytes, _lib.stream_ptr()), "esr_mse_loss")
        ctx.save_for_backward(grad)
        return loss[0]

    @staticmethod
    def backward(ctx, g):
        (grad,) = ctx.saved_tensors
        return grad * g, None


def mse_loss(pred, target):
    """nn.MSELoss() (train_ours_cnt_seq.py:774): mean over all elements; value and gradient from one kernel."""
    return _MSEFn.apply(pred, target)


# ------------------------------------------------------------------------------------------------------------------
# the differentiable window forward (structure of models/model.py:314-344 and the sub-blocks it calls)
# ------------------------------------------------------------------------------------------------------------------
def _cl(m, x, stride=1, act=None):
    return conv2d(x, m.conv2d.weight, m.conv2d.bias, stride, act)


def _accumulate(param, grad):
    if param.grad is None:
        param.grad = grad.detach().clone().view_as(param)
    else:
        param.grad.add_(grad.view_as(param))


def forward_sequence(model, frames, states=None):
    """frames BxLx2xHxW (L >= N = num_frame) -> ((L-N+1)*B x 2 x H x W window-major, [h_fwd, h_rev]).

    The L-N+1 sliding-window forwards of the reference's training loop (train_ours_cnt_seq.py:217-231) as ONE differentiable
    graph with the same batching as the inference plan (DESIGN.md 5): head / encoder / attention maps once per frame,
    every state-independent layer once for all windows, only the ConvGRU chain serial (both directions batched as 2B).
    Per image the arithmetic is that of models/model.py:314-344; gradients w.r.t. parameters, frames and `states`."""
    cfg = model._cfg
    N = cfg["num_frame"]
    B, L, Cin, H, W = frames.shape
    assert L >= N
    Wn = L - N + 1
    Hc, Wc = 8 * math.ceil(H / 8), 8 * math.ceil(W / 8)
    x = frames.float().transpose(0, 1).reshape(L * B, Cin, H, W)          # frame-major: image l*B + b
    if (Hc, Wc) != (H, W):                                               # CropSize.pad (models/model_util.py:148-152)
        pt, pb = math.ceil(0.5 * (Hc - H)), math.floor(0.5 * (Hc - H))
        pl, pr = math.ceil(0.5 * (Wc - W)), math.floor(0.5 * (Wc - W))
        x = F.pad(x, (pl, pr, pt, pb))
    x = _cl(model.head, x, act="relu")
    pyramid = []
    for blk in model.feat_extract.convblock:                              # FeatsExtract (models/model.py:20-45)
        x = _cl(blk, x, stride=2, act="relu")
        pyramid.append(x)
    pyramid.reverse()
    C, h, w = pyramid[0].shape[1:]
    f = pyramid[0].view(L, B, C, h, w).unbind(0)                          # unbind / split: one stack / cat in backward
    #                                                                       (indexing would zero-fill a full tensor per use)
    # ---- TimePropagation.local_time_corre (models/model.py:77-89, 133-146) for every (window, slot)
    tp = model.time_propagate
    # the (frame, frame) pairs the LTC index rule touches: (w, w) and (w+N-1, w+N-1) at a window's edges, neighbours inside
    pairs = sorted({(j, j) for j in range(Wn)} | {(j + N - 1, j + N - 1) for j in range(Wn)} | {(j, j + 1) for j in range(L - 1)})
    pm_in = torch.cat([torch.cat([f[a], f[b]], 1) for a, b in pairs], 0)
    pm = _cl(tp.pred_map[1], _cl(tp.pred_map[0], pm_in, act="relu"), act="sigmoid").view(len(pairs), B, 1, h, w).unbind(0)
    gate = {p: pm[k] for k, p in enumerate(pairs)}
    cat_in = []
    for wi in range(Wn):
        for i in range(N):
            a, b, c = wi + max(i - 1, 0), wi + i, wi + min(i + 1, N - 1)
            cat_in.append(torch.cat([f[a] * gate[(a, b)], f[b], f[c] * gate[(b, c)]], 1))
    xcat = torch.cat(cat_in, 0)                                           # [(Wn*N*B), 192, h, w]
    rb = tp.local_fusion[0]                                               # ResidualBlock (models/submodules.py:391-409)
    r = conv2d(xcat, rb.conv1.weight, rb.conv1.bias, 1, "relu")
    r = torch.relu(conv2d(r, rb.conv2.weight, rb.conv2.bias, 1, None) + xcat)
    mid_feat = torch.cat([f[wi + i] for wi in range(Wn) for i in range(N)], 0)
    ltc = _cl(tp.local_fusion[1], r) + mid_feat
    # ---- TimePropagation.global_time_corre: RecurrentConvLayer + ConvGRU (models/submodules.py:340-344, 496-514)
    gx = _cl(tp.lstm.conv, ltc, act="relu").view(Wn * N, B, C, h, w).unbind(0)   # the x-side conv of every step at once
    gru = tp.lstm.recurrent_block
    w_zr = torch.cat([gru.update_gate.weight, gru.reset_gate.weight], 0)   # both gates in one 128 -> 128 convolution
    b_zr = torch.cat([gru.update_gate.bias, gru.reset_gate.bias], 0)

    def sink_zr(dw, db):                                                   # batched weight gradient of all steps (train_step)
        for p, gpart in ((gru.update_gate.weight, dw[:C]), (gru.reset_gate.weight, dw[C:]), (gru.update_gate.bias, db[:C]),
                         (gru.reset_gate.bias, db[C:])):
            _accumulate(p, gpart)

    def sink_o(dw, db):
        _accumulate(gru.out_gate.weight, dw)
        _accumulate(gru.out_gate.bias, db)

    h_f, h_r = states if states is not None else (None, None)
    hs = None if h_f is None else torch.cat([h_f, h_r], 0)                # forward and reverse chains batched as 2B
    fwd, rev = [], []
    for wi in range(Wn):
        rev_w = [None] * N
        for i in range(N):
            if cfg["gtc_frozen"]:
                hs = None
            xi = torch.cat([gx[wi * N + i], gx[wi * N + N - 1 - i]], 0)
            if hs is None:
                hs = torch.zeros_like(xi)
            zr = conv2d(torch.cat([xi, hs], 1), w_zr, b_zr, 1, "sigmoid", defer=("gru_zr", sink_zr))
            o = conv2d(torch.cat([xi, _GruHRFn.apply(hs, zr)], 1), gru.out_gate.weight, gru.out_gate.bias, 1, "tanh",
                       defer=("gru_o", sink_o))
            hs = _GruBlendFn.apply(hs, zr, o)                          # h (1 - z) + o z   (models/submodules.py:511-512)
            hf, hr = hs.split(B, 0)
            fwd.append(hf)
            rev_w[N - 1 - i] = hr
        rev.extend(rev_w)
    new_states = [None, None] if cfg["gtc_frozen"] else list(hs.split(B, 0))
    both = torch.cat([torch.cat(fwd, 0), torch.cat(rev, 0)], 1)           # [(Wn*N*B), 128, h, w]
    prop = (_cl(tp.global_fusion, both, act="relu") + mid_feat).view(Wn, N, B, C, h, w).unbind(1)

    # ---- STFusion (models/model.py:208-291): both neighbours of all windows at once
    sf = model.spacetime_fuse
    mid = (N - 1) // 2
    center = prop[mid].reshape(Wn * B, C, h, w)
    others = [i for i in range(N) if i != mid]
    nb = torch.cat([prop[i].reshape(Wn * B, C, h, w) for i in others], 0)
    ctr = torch.cat([center] * len(others), 0)
    off_feat = _cl(sf.offset[1], _cl(sf.offset[0], torch.cat([nb, ctr], 1), act="relu"))
    om = conv2d(off_feat, sf.dcn.conv_offset_mask.weight, sf.dcn.conv_offset_mask.bias, 1, None)
    o1, o2, msk = torch.chunk(om, 3, dim=1)                               # DCN_sep.forward (models/DCNv2/dcn_v2.py:214-227)
    aligned = torch.relu(dcn_v2(nb, torch.cat((o1, o2), 1), torch.sigmoid(msk), sf.dcn.weight, sf.dcn.bias, 8))
    ft = _cl(sf.convblock[1], _cl(sf.convblock[0], torch.cat([aligned, ctr], 1), act="relu"))
    sk = _cl(sf.kernel, ft, act="sigmoid")
    mlp = sf.fc[0].layers
    ck = torch.relu(F.linear(ft.flatten(2).max(dim=2)[0], mlp[0].weight, mlp[0].bias))
    ck = torch.sigmoid(F.linear(ck, mlp[1].weight, mlp[1].bias))
    sk0, sk1 = sk.split(1, 1)
    ck0, ck1 = ck.split(C, 1)
    y = torch.cat([aligned * sk0 * ck0[:, :, None, None], ctr * sk1 * ck1[:, :, None, None]], 1)
    fz = _cl(sf.dcn_fusion[1], _cl(sf.dcn_fusion[0], y, act="relu")).view(len(others), Wn * B, C, h, w).unbind(0)
    x = torch.cat(list(fz) + [center], 1)
    x = _cl(sf.dense_fusion[1], _cl(sf.dense_fusion[0], x, act="relu"))
    for lvl, ft in enumerate(pyramid):                                    # scale_aggre + recons (models/model.py:253-291)
        prod = (ft * _cl(sf.attens[lvl], ft, act="sigmoid")).view(L, B, *ft.shape[1:]).unbind(0)
        agg = torch.cat([_window_sum(prod, wi, N) / N for wi in range(Wn)], 0)   # mean over the window's N frames
        x = upsample2x(x + agg)
        x = _cl(sf.recons[lvl], x, act="relu")
    x = _cl(model.tail, x, act="relu")
    if (Hc, Wc) != (H, W):                                               # CropSize.crop (models/model_util.py:154-164)
        cy, cx = Hc // 2, Wc // 2
        x = x[..., cy - H // 2: cy + math.ceil(H / 2), cx - W // 2: cx + math.ceil(W / 2)].contiguous()
    return x, new_states


def _window_sum(prod, wi, N):
    """prod[wi] + prod[wi + 1] + ... + prod[wi + N - 1], added in frame order."""
    s = prod[wi]
    for i in range(1, N):
        s = s + prod[wi + i]
    return s


def forward_window(model, inp, states=None):
    """inp BxNx2xHxW -> (Bx2xHxW, [h_fwd, h_rev]): the reference's single-window forward, differentiable."""
    assert inp.shape[1] == model._cfg["num_frame"]
    return forward_sequence(model, inp, states)


# ------------------------------------------------------------------------------------------------------------------
# optimizer and the step
# ------------------------------------------------------------------------------------------------------------------
class Adam(torch.optim.Optimizer):
    """torch.optim.Adam(params, lr, betas, eps, weight_decay, amsgrad) semantics (the reference's optimizer,
    train_ours_cnt_seq.py:781 + config optimizer args) with one kernel launch per step: parameters and gradients are
    re-homed as views of two flat fp32 buffers (so the gradient exchange and the update see contiguous memory); the step
    counter and the hyper-parameters live on the device (the kernel reads them when it runs), so a captured CUDA graph of the
    step stays correct on replay AND follows a learning-rate schedule.

    `param_groups` is the single group torch schedulers read and write (`torch.optim.lr_scheduler.*` only touch
    `optimizer.param_groups[i]['lr']`, `initial_lr`): every step() / graph replay uploads lr, betas, eps and weight_decay from
    it.  `log_slots` extra floats ride at the tail of the gradient buffer (`exchange`): the trainer's logging scalars
    (train_ours_cnt_seq.py:238-239: last-window MSE, summed loss) take part in the ONE all-reduce of the iteration instead of
    two extra barrier + all-reduce pairs (myutils/utils.py:43-54) and the per-step dist.barrier (:339)."""

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, amsgrad=False, log_slots=2):
        self.params = [p for p in params if p.requires_grad]
        if not self.params or not self.params[0].is_cuda:
            raise _lib.ESRError("esr_b200.train.Adam needs CUDA parameters")
        dev = self.params[0].device
        n = sum(p.numel() for p in self.params)
        self.flat = torch.empty((n,), dtype=torch.float32, device=dev)
        self.exchange = torch.zeros((n + int(log_slots),), dtype=torch.float32, device=dev)   # gradients | logging scalars
        self.flat_grad = self.exchange[:n]
        self.log = self.exchange[n:]
        off = 0
        for p in self.params:
            k = p.numel()
            self.flat[off:off + k].copy_(p.data.reshape(-1))
            p.data = self.flat[off:off + k].view_as(p.data)
            p.grad = self.flat_grad[off:off + k].view_as(p.data)
            off += k
        self.exp_avg, self.exp_avg_sq = torch.zeros_like(self.flat), torch.zeros_like(self.flat)
        self.max_exp_avg_sq = torch.zeros_like(self.flat) if amsgrad else None
        self.step_dev = torch.zeros((1,), dtype=torch.int32, device=dev)   # step counter lives on the device (graph replays)
        # torch.optim.Optimizer base: param_groups / defaults / hooks, so torch.optim.lr_scheduler.* attach to it
        # (train_ours_cnt_seq.py:784); the per-parameter `state` of the base class stays empty, the moments are flat buffers
        super().__init__(self.params, dict(lr=lr, betas=tuple(betas), eps=eps, weight_decay=weight_decay, amsgrad=amsgrad))
        self.hyper = torch.zeros((5,), dtype=torch.float32, device=dev)
        self._hyper_host = torch.zeros((5,), dtype=torch.float32).pin_memory()
        self._hyper_sig = None
        self.upload_hyper()

    # the attributes torch's schedulers / older callers read
    @property
    def lr(self):
        return self.param_groups[0]["lr"]

    def upload_hyper(self):
        """param_groups[0] -> device (called before every step / graph replay; 20 bytes, only when something changed)."""
        g = self.param_groups[0]
        sig = (float(g["lr"]), float(g["betas"][0]), float(g["betas"][1]), float(g["eps"]), float(g["weight_decay"]))
        if sig != self._hyper_sig:
            for i, v in enumerate(sig):
                self._hyper_host[i] = v
            self.hyper.copy_(self._hyper_host, non_blocking=True)
            self._hyper_sig = sig

    def zero_grad(self, set_to_none=False):
        self.exchange.zero_()
        off = 0
        for p in self.params:                                    # keep the views if something replaced .grad
            k = p.numel()
            if p.grad is None or p.grad.data_ptr() != self.flat_grad.data_ptr() + 4 * off:
                p.grad = self.flat_grad[off:off + k].view_as(p.data)
            off += k

    def step(self, closure=None):
        if not torch.cuda.is_current_stream_capturing():
            self.upload_hyper()
        with torch.cuda.device(self.flat.device):
            _lib.check(_lib.lib().esr_adam_step_dev(_lib.ptr(self.flat), _lib.ptr(self.flat_grad), _lib.ptr(self.exp_avg),
                                                    _lib.ptr(self.exp_avg_sq), _lib.ptr(self.max_exp_avg_sq), self.flat.numel(),
                                                    _lib.ptr(self.step_dev), _lib.ptr(self.hyper), _lib.stream_ptr()), "esr_adam_step_dev")
        torch._C._increment_version(self.params)                  # the kernel wrote the parameters behind autograd's back:
        #                                                           bump their versions so cached inference blobs repack

    def state_dict(self):
        return {"step": int(self.step_dev.item()), "exp_avg": self.exp_avg, "exp_avg_sq": self.exp_avg_sq,
                "max_exp_avg_sq": self.max_exp_avg_sq, "param_groups": [{k: v for k, v in self.param_groups[0].items() if k != "params"}]}

    def load_state_dict(self, sd):
        self.step_dev.fill_(int(sd["step"]))
        self.exp_avg.copy_(sd["exp_avg"]); self.exp_avg_sq.copy_(sd["exp_avg_sq"])
        if self.max_exp_avg_sq is not None and sd.get("max_exp_avg_sq") is not None:
            self.max_exp_avg_sq.copy_(sd["max_exp_avg_sq"])
        self.param_groups[0].update(sd["param_groups"][0])
        self.upload_hyper()

    def _offsets(self, named_params):
        """Flat-buffer offset of every (name, parameter) in `named_params`' order (matched by identity, not by this
        optimizer's own parameter order)."""
        at, off = {}, 0
        for p in self.params:
            at[id(p)] = off
            off += p.numel()
        try:
            return [at[id(p)] for _, p in named_params]
        except KeyError:
            raise _lib.ESRError("Adam: a named parameter is not one this optimizer updates") from None

    def torch_state_dict(self, named_params):
        """This state in torch.optim.Adam.state_dict()'s layout, parameter index i = named_params[i] (the reference's
        optimizer sees the model's parameters in its state_dict key order, train_ours_cnt_seq.py:778)."""
        named_params = list(named_params)
        shapes = [tuple(p.shape) for _, p in named_params]
        return to_torch_adam(shapes, self._offsets(named_params), int(self.step_dev.item()), self.exp_avg.cpu(),
                             self.exp_avg_sq.cpu(), None if self.max_exp_avg_sq is None else self.max_exp_avg_sq.cpu(),
                             self.param_groups[0])

    def load_torch_state_dict(self, sd, named_params):
        """Load a torch.optim.Adam.state_dict() (a reference checkpoint's optimizer states) whose parameter index i is
        named_params[i]."""
        named_params = list(named_params)
        shapes = [tuple(p.shape) for _, p in named_params]
        flat = from_torch_adam(sd, shapes, self._offsets(named_params), self.flat.numel(), self.max_exp_avg_sq is not None)
        self.step_dev.fill_(flat["step"])
        self.exp_avg.copy_(flat["exp_avg"])
        self.exp_avg_sq.copy_(flat["exp_avg_sq"])
        if self.max_exp_avg_sq is not None:
            self.max_exp_avg_sq.copy_(flat["max_exp_avg_sq"])
        self.param_groups[0].update(flat["group"])
        self.upload_hyper()


def to_torch_adam(shapes, offsets, step, exp_avg, exp_avg_sq, max_exp_avg_sq, group):
    """Flat Adam moments -> torch.optim.Adam.state_dict(): {'state': {i: {'step', 'exp_avg', 'exp_avg_sq'[,
    'max_exp_avg_sq']}}, 'param_groups': [{..., 'params': [0..n-1]}]}.  Parameter i has shape shapes[i] and starts at
    offsets[i] of the flat buffers.  No entry per parameter before the first step, as torch's own."""
    ref = torch.optim.Adam([torch.zeros(1)]).state_dict()["param_groups"][0]
    g = dict(ref, **{k: v for k, v in group.items() if k != "params"})
    g["betas"] = tuple(g["betas"])
    g["params"] = list(range(len(shapes)))
    state = {}
    if step > 0:
        for i, (shp, off) in enumerate(zip(shapes, offsets)):
            k = math.prod(shp)
            st = {"step": torch.tensor(float(step)), "exp_avg": exp_avg[off:off + k].reshape(shp).clone(),
                  "exp_avg_sq": exp_avg_sq[off:off + k].reshape(shp).clone()}
            if g["amsgrad"]:
                st["max_exp_avg_sq"] = max_exp_avg_sq[off:off + k].reshape(shp).clone()
            state[i] = st
    return {"state": state, "param_groups": [g]}


def from_torch_adam(sd, shapes, offsets, n, amsgrad):
    """torch.optim.Adam.state_dict() -> {'step', 'exp_avg', 'exp_avg_sq', 'max_exp_avg_sq', 'group'} with flat CPU fp32
    moments of n elements (the inverse of to_torch_adam).  'step' may be a tensor or, from older torch, an int."""
    if len(sd["param_groups"]) != 1 or len(sd["param_groups"][0]["params"]) != len(shapes):
        raise _lib.ESRError(f"Adam: the checkpoint's optimizer has {[len(g['params']) for g in sd['param_groups']]} parameters "
                            f"in its groups; the model has {len(shapes)} in one")
    out = {"exp_avg": torch.zeros(n), "exp_avg_sq": torch.zeros(n), "max_exp_avg_sq": torch.zeros(n) if amsgrad else None}
    steps = set()
    for i, (shp, off) in enumerate(zip(shapes, offsets)):
        st = sd["state"].get(i)
        if st is None:
            steps.add(0)
            continue
        k = math.prod(shp)
        keys = ("exp_avg", "exp_avg_sq", "max_exp_avg_sq") if amsgrad else ("exp_avg", "exp_avg_sq")
        if amsgrad and "max_exp_avg_sq" not in st:
            raise _lib.ESRError("Adam: the checkpoint's optimizer ran with amsgrad=False (no max_exp_avg_sq); the config asks "
                                "for amsgrad=True")
        for key in keys:
            t = st[key]
            if tuple(t.shape) != tuple(shp):
                raise _lib.ESRError(f"Adam: parameter {i}: {key} has shape {tuple(t.shape)}, the model's is {tuple(shp)}")
            out[key][off:off + k] = t.detach().reshape(-1).float().cpu()
        steps.add(int(st["step"]))
    if len(steps) > 1:
        raise _lib.ESRError(f"Adam: the checkpoint's parameters were stepped different numbers of times {sorted(steps)}")
    out["step"] = steps.pop() if steps else 0
    out["group"] = {k: v for k, v in sd["param_groups"][0].items() if k not in ("params", "amsgrad")}
    return out


def _step_body(model, optimizer, frames, gt, num_frame, all_reduce):
    Wn = frames.shape[1] - num_frame + 1
    mid = (num_frame - 1) // 2
    optimizer.zero_grad()
    net = model.module if hasattr(model, "module") else model
    net.reset_states()
    # the ConvGRU weight gradients are batched over all steps (one launch per gate; measured -1.5 ms per cfg2 iteration).
    # Not under DDP: its reducer must see every gradient inside backward.
    defer = not hasattr(model, "module")
    with _defer_weight_grads() if defer else contextlib.nullcontext() as deferred:
        pred = model(frames)                                      # all windows, window-major [(Wn*B), 2, H, W]
        target = gt[:, mid:mid + Wn].transpose(0, 1).reshape(pred.shape)
        loss = Wn * mse_loss(pred, target)                        # = sum over windows of MSELoss(pred_w, gt[:, w + mid])
        loss.backward()
        if deferred is not None:
            deferred.flush()                                      # ConvGRU weight gradients: one launch per gate over all steps
    if optimizer.log.numel() >= 2:
        # the trainer's two logging scalars (train_ours_cnt_seq.py:238-239): MSE of the last window and the summed loss; they
        # travel at the tail of the gradient bucket, so the single exchange below reduces them too
        B = frames.shape[0]
        with torch.no_grad():
            optimizer.log[0:1].copy_(mse_loss(pred.detach()[-B:], target[-B:]).reshape(1))
            optimizer.log[1:2].copy_(loss.detach().reshape(1))
    if all_reduce is not None:
        all_reduce(optimizer.exchange)
    optimizer.step()
    return loss.detach(), pred.detach()


def _model_num_frame(model, num_frame):
    """The model's num_frame (model._cfg, or model.module._cfg under DDP); an explicit value must agree with it."""
    net = model.module if hasattr(model, "module") else model
    n = net._cfg["num_frame"]
    if num_frame is not None and int(num_frame) != n:
        raise _lib.ESRError(f"esr_b200.train: num_frame={num_frame} but the model was built with num_frame={n}")
    return n


def train_step(model, optimizer, frames, gt, num_frame=None, all_reduce=None):
    """One reference training iteration (train_ours_cnt_seq.py:209-235) on a batch of sequences.

    frames: BxLx2xHxW input count tensors (inp_scaled_cnt of each frame); gt: BxLx2xHxW target count tensors.
    Windows of num_frame frames (default and required: the model's) slide by one frame (dataloader/h5dataloader.py:229-231);
    the loss is the sum over windows of
    MSE(pred, gt[:, window middle]) with the ConvGRU state carried from window to window; one backward; optional
    `all_reduce(exchange)` over the flat gradient bucket + the two logging scalars (DDP's role when the model is not
    DDP-wrapped; after it `optimizer.log` holds the rank-reduced last-window MSE and summed loss, which is everything
    train_ours_cnt_seq.py:238-239 + :339 need -- no extra barrier or collective); one Adam step.  Returns the local summed loss."""
    return _step_body(model, optimizer, frames, gt, _model_num_frame(model, num_frame), all_reduce)[0]


class GraphedTrainStep:
    """train_step captured once into a CUDA graph (forward, backward, all-reduce hook and the Adam kernel) and replayed:
    no Python / launch overhead per iteration.  Shapes are fixed at construction; data is copied into static buffers.
    `exchanges` is the number of all_reduce calls the captured graph holds (1 with a hook, 0 without).
    After a replay `pred` holds the iteration's prediction of every window (window-major [(L-N+1)*B, 2, H, W], the static
    output of the graph; the trainer's images read the last window from it).
    The graph holds the kernels of the mode it was captured in (`deterministic()` or not); replaying it after the mode has
    changed raises ESRError instead of running the other mode's kernels."""

    def __init__(self, model, optimizer, frames_shape, device, num_frame=None, all_reduce=None, warmup=2):
        self.model, self.opt = model, optimizer
        self.deterministic = deterministic()
        num_frame = _model_num_frame(model, num_frame)
        self.frames = torch.zeros(frames_shape, dtype=torch.float32, device=device)
        self.gt = torch.zeros(frames_shape, dtype=torch.float32, device=device)
        keep = [t.clone() for t in (optimizer.flat, optimizer.exp_avg, optimizer.exp_avg_sq)]
        keep_max = None if optimizer.max_exp_avg_sq is None else optimizer.max_exp_avg_sq.clone()
        keep_step = optimizer.step_dev.clone()
        side = torch.cuda.Stream(device)
        side.wait_stream(torch.cuda.current_stream(device))
        with torch.cuda.stream(side):                             # warm-up: lazy inits + allocator, outside the capture
            for _ in range(warmup):
                _step_body(model, optimizer, self.frames, self.gt, num_frame, all_reduce)
        torch.cuda.current_stream(device).wait_stream(side)
        # capture; with an NCCL all-reduce inside, the FIRST capture on a fresh capture stream can be invalidated by the process
        # group's first-use bookkeeping (seen at N = 2: first attempt fails, second succeeds) -> one retry; the optimizer state
        # touched by the warm-up iterations is restored whatever happens
        def restore():
            for dst, src in zip((optimizer.flat, optimizer.exp_avg, optimizer.exp_avg_sq), keep):
                dst.copy_(src)
            if keep_max is not None:
                optimizer.max_exp_avg_sq.copy_(keep_max)
            optimizer.step_dev.copy_(keep_step)

        calls = [0]

        def counted(flat):
            calls[0] += 1
            all_reduce(flat)

        err = None
        for attempt in range(2):
            calls[0] = 0
            try:
                self.graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(self.graph):
                    self.loss, self.pred = _step_body(model, optimizer, self.frames, self.gt, num_frame,
                                                      None if all_reduce is None else counted)
                err = None
                break
            except Exception as e:                                # noqa: BLE001 -- rethrown below
                err = e
                torch.cuda.synchronize(device)
        restore()
        if err is not None:
            raise err
        self.exchanges = calls[0]                                 # all_reduce calls in the graph: each replay issues them

    def __call__(self, frames, gt):
        if deterministic() != self.deterministic:
            raise _lib.ESRError(f"GraphedTrainStep was captured with deterministic mode {'on' if self.deterministic else 'off'}; "
                                "restore torch.use_deterministic_algorithms / torch.backends.cudnn.deterministic to that "
                                "setting or capture a new GraphedTrainStep")
        self.frames.copy_(frames)
        self.gt.copy_(gt)
        self.opt.upload_hyper()                                   # a scheduler may have changed param_groups[0]['lr']
        self.graph.replay()
        torch._C._increment_version(self.opt.params)
        return self.loss
