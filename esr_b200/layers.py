"""Layer-level host wrappers over the C ABI (esr_conv_tc & friends).  Used by the tests and by tools; the
network itself is driven from C++ (esr_net_*), not from here."""
import ctypes

import torch

from . import _lib

ACT = {None: 0, "none": 0, "relu": 1, "sigmoid": 2, "tanh": 3}


class Split:
    """A split-bf16 NHWC activation tensor [2][n_img][H][W][C] living in a torch bf16 buffer."""

    def __init__(self, n_img, C, H, W, device):
        self.n_img, self.C, self.H, self.W = n_img, C, H, W
        self.buf = torch.zeros((2, n_img, H, W, C), dtype=torch.bfloat16, device=device)

    @staticmethod
    def from_nchw(x):
        x = x.contiguous().float()
        n, C, H, W = x.shape
        s = Split(n, C, H, W, x.device)
        _lib.check(_lib.lib().esr_split_from_nchw(_lib.ptr(x), n, C, H, W, _lib.ptr(s.buf), _lib.stream_ptr()),
                   "esr_split_from_nchw")
        return s

    def to_nchw(self):
        out = torch.empty((self.n_img, self.C, self.H, self.W), dtype=torch.float32, device=self.buf.device)
        _lib.check(_lib.lib().esr_split_to_nchw(_lib.ptr(self.buf), self.n_img, self.C, self.H, self.W, _lib.ptr(out),
                                                _lib.stream_ptr()), "esr_split_to_nchw")
        return out


def pack_weight(w, w2=None):
    """fp32 [Cout,Cin,k,k] CUDA weight(s) -> packed split-bf16 K-blocks (uint8 buffer)."""
    L = _lib.lib()
    w = w.contiguous().float()
    co, ci, k, _ = w.shape
    tot = co * (2 if w2 is not None else 1)
    buf = torch.empty((L.esr_conv_weight_bytes(tot, ci, k),), dtype=torch.uint8, device=w.device)
    w2c = w2.contiguous().float() if w2 is not None else None
    _lib.check(L.esr_pack_conv_weight(_lib.ptr(w), _lib.ptr(w2c), co, ci, k, _lib.ptr(buf), _lib.stream_ptr()),
               "esr_pack_conv_weight")
    return buf


def pad_bias(b, cout):
    npad = (cout + 15) // 16 * 16
    out = torch.zeros((npad,), dtype=torch.float32, device=b.device)
    out[:cout] = b.float()
    return out


def conv_tc(srcs, wpacked, bias, cout, ntaps=9, act=None, act_from=0, src_img=None, n_img=None,
            res=None, res_mode=0, res_img=None, out=None, out_coff=0, out_f32=None,
            epi_mode=0, h_prev=None, z_buf=None, src_chunks=None, chunk_img_step=None):
    """Runs one tensor-core convolution.  srcs: list of Split; returns (out Split or None, out_f32 or None).
    chunk_img_step[i] = k != 0: the 64-channel source i stands for src_chunks[i] chunks, chunk j read from image
    src_img[i][img] + j * k (esr_conv_tc_chunked)."""
    d = _lib.ConvDesc()
    keep = []
    H, W = srcs[0].H, srcs[0].W
    d.n_src = len(srcs)
    for i, s in enumerate(srcs):
        d.src[i] = s.buf.data_ptr()
        d.src_C[i] = s.C
        d.src_n_img[i] = s.n_img
        if src_img is not None and src_img[i] is not None:
            t = src_img[i].to(device=s.buf.device, dtype=torch.int32).contiguous()
            keep.append(t)
            d.src_img[i] = t.data_ptr()
    d.H, d.W = H, W
    d.n_img = n_img if n_img is not None else srcs[0].n_img
    d.ntaps, d.cout = ntaps, cout
    d.wpacked, d.bias = wpacked.data_ptr(), bias.data_ptr()
    d.act, d.act_from, d.res_mode, d.epi_mode = ACT[act], act_from, res_mode, epi_mode
    if res is not None:
        d.res, d.res_C, d.res_n_img = res.buf.data_ptr(), res.C, res.n_img
        if res_img is not None:
            t = res_img.to(device=res.buf.device, dtype=torch.int32).contiguous()
            keep.append(t)
            d.res_img = t.data_ptr()
    if out is not None:
        d.out, d.out_C, d.out_n_img, d.out_coff = out.buf.data_ptr(), out.C, out.n_img, out_coff
    if out_f32 is not None:
        d.out_f32, d.out_f32_C = out_f32.data_ptr(), out_f32.shape[-1]
    if h_prev is not None:
        d.h_prev, d.h_n_img = h_prev.buf.data_ptr(), h_prev.n_img
    if z_buf is not None:
        d.z_buf = z_buf.data_ptr()
    if chunk_img_step is None:
        _lib.check(_lib.lib().esr_conv_tc(ctypes.byref(d), _lib.stream_ptr()), "esr_conv_tc")
    else:
        chunks = (ctypes.c_int * 3)(*(list(src_chunks) + [0] * (3 - len(src_chunks))))
        steps = (ctypes.c_int * 3)(*(list(chunk_img_step) + [0] * (3 - len(chunk_img_step))))
        _lib.check(_lib.lib().esr_conv_tc_chunked(ctypes.byref(d), chunks, steps, _lib.stream_ptr()), "esr_conv_tc_chunked")
    torch.cuda.current_stream().synchronize() if keep else None
    return out, out_f32


# esr_conv_small kinds (include/esr_b200.h) and paths
SMALL_KINDS = {"head_enc0": 0, "enc1": 1, "enc2": 2, "att32": 3, "att16": 4, "recon1": 5, "recon2": 6, "tail": 7,
               "spatial_kernel": 10}
SMALL_PATHS = {"mma": 0, "ffma": 1, "narrow": 2}


def conv_small_supported(kind, path):
    return _lib.lib().esr_conv_small_workspace_bytes(SMALL_KINDS[kind], SMALL_PATHS[path]) > 0


def conv_small(kind, path, x, w, bias, n_img, out=None, out_f32=None, in_img=None, pads=(0, 0, 0, 0), head=None,
               crop=None):
    """One small-channel / narrow-output layer of the network (esr_conv_small) on kernel family `path`.
    x: Split, or fp32 NCHW [*, 2, H, W] for head_enc0 (then head = (w_head, b_head), pads = (top, bottom, left, right));
    out: Split for Cout >= 8, else out_f32 (NHWC, or NCHW [n_img, 2, out_H, out_W] with crop = (top, left) for the tail)."""
    L = _lib.lib()
    k, p = SMALL_KINDS[kind], SMALL_PATHS[path]
    d = _lib.ConvSmallDesc()
    d.kind, d.path, d.n_img = k, p, n_img
    w, bias = w.contiguous().float(), bias.contiguous().float()
    keep = []

    def dev_i32(t):
        t = t.to(device=w.device, dtype=torch.int32).contiguous()
        keep.append(t)
        return t.data_ptr()

    if kind == "head_enc0":
        x = x.contiguous()
        keep.append(x)
        d.in_f32, d.in_n_img, d.H_in, d.W_in = x.data_ptr(), x.shape[0], x.shape[2], x.shape[3]
        d.pad_top, d.pad_bottom, d.pad_left, d.pad_right = pads
        head = [t.contiguous().float() for t in head]
        d.w_head, d.b_head = head[0].data_ptr(), head[1].data_ptr()
    else:
        d.in_, d.in_n_img, d.H_in, d.W_in = x.buf.data_ptr(), x.n_img, x.H, x.W
    if in_img is not None:
        d.in_img = dev_i32(in_img)
    d.w, d.bias = w.data_ptr(), bias.data_ptr()
    if out is not None:
        d.out, d.out_n_img = out.buf.data_ptr(), out.n_img
    if out_f32 is not None:
        d.out_f32 = out_f32.data_ptr()
        if crop is not None:
            d.crop_top, d.crop_left = crop
            d.out_H, d.out_W = out_f32.shape[2], out_f32.shape[3]
    nbytes = L.esr_conv_small_workspace_bytes(k, p)
    ws = torch.empty((max(nbytes, 1),), dtype=torch.uint8, device=w.device)
    d.workspace, d.workspace_bytes = ws.data_ptr(), nbytes
    _lib.check(L.esr_conv_small(ctypes.byref(d), _lib.stream_ptr()), f"esr_conv_small({kind}, {path})")
    torch.cuda.current_stream().synchronize()
    return out if out is not None else out_f32


# esr_glue ops (include/esr_b200.h)
GLUE_OPS = {"ltc_cat": 0, "chan_max": 1, "attn_mlp": 2, "attn_apply": 3, "scale_aggregate": 4, "upsample2x": 5, "copy_split": 6}


def glue(op, n_img, H, W, C, x=None, x2=None, idx=None, N=0, maps=None, sk=None, ck_in=None, att=None, mlp=None, mx=None,
         ck=None, out=None):
    """One launcher of the network's element-wise glue (esr_glue) on n_img images of H x W.
    x, x2, out: Split (their n_img sets the plane stride); idx: int table or None; maps / sk / ck_in / att: fp32 CUDA tensors;
    mlp = (w0, b0, w1, b1); mx: int32 [*, 64] (chan_max writes it, attn_mlp reads it); ck: fp32 [*, 128] (attn_mlp).
    The image count of mx (chan_max) or ck (attn_mlp) is passed as the output's."""
    d = _lib.GlueDesc()
    d.op, d.n_img, d.N, d.H, d.W, d.C = GLUE_OPS[op], n_img, N, H, W, C
    keep = []

    def addr(t):
        if t is None:
            return None
        t = t.contiguous()
        keep.append(t)
        return t.data_ptr()

    if x is not None:
        d.in_, d.in_n_img = x.buf.data_ptr(), x.n_img
    if x2 is not None:
        d.in2, d.in2_n_img = x2.buf.data_ptr(), x2.n_img
    if idx is not None:
        d.idx = addr(idx.to(dtype=torch.int32, device=torch.device("cuda", torch.cuda.current_device())))
    d.maps, d.sk, d.ck_in, d.att = addr(maps), addr(sk), addr(ck_in), addr(att)
    if mlp is not None:
        d.w0, d.b0, d.w1, d.b1 = (addr(t.float()) for t in mlp)
    if mx is not None:
        d.mx = mx.data_ptr()
    if ck is not None:
        d.ck = ck.data_ptr()
    if out is not None:
        d.out, d.out_n_img = out.buf.data_ptr(), out.n_img
    elif op == "chan_max" and mx is not None:
        d.out_n_img = mx.shape[0]
    elif op == "attn_mlp" and ck is not None:
        d.out_n_img = ck.shape[0]
    _lib.check(_lib.lib().esr_glue(ctypes.byref(d), _lib.stream_ptr()), f"esr_glue({op})")
    torch.cuda.current_stream().synchronize()
    return out
