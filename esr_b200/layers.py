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
