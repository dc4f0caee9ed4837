"""Drop-in for the reference's `_ext` pybind module (models/DCNv2/src/vision.cpp:4-8), forward operator.

    import esr_b200.dcn_v2_ext as _ext;  sys.modules['_ext'] = _ext       (see esr_b200.dropin)

dcn_v2_forward keeps the reference's 14-argument signature (models/DCNv2/dcn_v2.py:27-42) and its behaviour:
contiguous fp32 CUDA tensors in the NCHW layout, a freshly allocated output, errors as RuntimeError.
dcn_v2_backward returns the reference's five gradients (fp32 atomics for grad_input, like the reference; int64 fixed point,
bitwise reproducible, in deterministic mode: esr_b200.train.deterministic()).
"""
import torch

from . import _lib


def dcn_v2_forward(input, weight, bias, offset, mask, kernel_h, kernel_w, stride_h, stride_w, pad_h, pad_w,
                   dilation_h, dilation_w, deformable_group):
    if not input.is_cuda:
        raise RuntimeError("Not compiled with CPU support")       # there is no CPU path in esr_b200
    for t in (input, weight, bias, offset, mask):
        if t.dtype != torch.float32:
            raise RuntimeError("dcn_v2_forward: expected float32 tensors")
    B, C, H, W = input.shape
    Co = weight.shape[0]
    if kernel_h != kernel_w or stride_h != stride_w or pad_h != pad_w or dilation_h != dilation_w:
        raise RuntimeError("dcn_v2_forward: only square kernels / strides are implemented")
    if weight.shape[2] != kernel_h or weight.shape[3] != kernel_w:
        raise RuntimeError("Input shape and kernel shape wont match: (%d x %d vs %d x %d)."
                           % (kernel_h, kernel_w, weight.shape[2], weight.shape[3]))
    if C != weight.shape[1]:
        raise RuntimeError("Input shape and kernel channels wont match: (%d vs %d)." % (C, weight.shape[1]))
    L = _lib.lib()
    args = [t.contiguous() for t in (input, weight, bias, offset, mask)]
    Ho = (H + 2 * pad_h - (dilation_h * (kernel_h - 1) + 1)) // stride_h + 1
    Wo = (W + 2 * pad_w - (dilation_w * (kernel_w - 1) + 1)) // stride_w + 1
    out = torch.empty((B, Co, Ho, Wo), dtype=torch.float32, device=input.device)
    with torch.cuda.device(input.device):
        nbytes = L.esr_dcn_v2_workspace_bytes_ex(B, C, H, W, Co, kernel_h, stride_h, pad_h, dilation_h, deformable_group, 0)
        ws = torch.empty((max(nbytes, 256),), dtype=torch.uint8, device=input.device)
        rc = L.esr_dcn_v2_forward(*[_lib.ptr(t) for t in args], B, C, H, W, Co, kernel_h, stride_h, pad_h, dilation_h,
                                  deformable_group, _lib.ptr(out), _lib.ptr(ws), nbytes, _lib.stream_ptr())
    if rc != 0:
        raise RuntimeError("dcn_v2_forward: " + L.esr_last_error().decode())
    return out


def dcn_v2_backward(input, weight, bias, offset, mask, grad_output, kernel_h, kernel_w, stride_h, stride_w, pad_h, pad_w,
                    dilation_h, dilation_w, deformable_group):
    """-> [grad_input, grad_offset, grad_mask, grad_weight, grad_bias]  (models/DCNv2/dcn_v2.py:50-66).
    In deterministic mode (esr_b200.train.deterministic()) the gradients are bitwise reproducible; only the network's own
    configuration (64 -> 64, 3x3, 8 groups) has that mode, any other raises ESRError there."""
    from .train import deterministic
    if not input.is_cuda:
        raise RuntimeError("Not compiled with CPU support")
    for t in (input, weight, bias, offset, mask, grad_output):
        if t.dtype != torch.float32:
            raise RuntimeError("dcn_v2_backward: expected float32 tensors")
    B, C, H, W = input.shape
    Co = weight.shape[0]
    L = _lib.lib()
    args = [t.contiguous() for t in (input, weight, bias, offset, mask, grad_output)]
    outs = [torch.empty_like(args[0]), torch.empty_like(args[3]), torch.empty_like(args[4]), torch.empty_like(args[1]),
            torch.empty_like(args[2])]
    flags = _lib.DETERMINISTIC if deterministic() else 0
    with torch.cuda.device(input.device):
        nbytes = L.esr_dcn_v2_backward_workspace_bytes_ex(B, C, H, W, Co, kernel_h, stride_h, pad_h, dilation_h, deformable_group,
                                                          flags)
        ws = torch.empty((max(nbytes, 256),), dtype=torch.uint8, device=input.device)
        rc = L.esr_dcn_v2_backward_ex(*[_lib.ptr(t) for t in args], B, C, H, W, Co, kernel_h, stride_h, pad_h, dilation_h,
                                      deformable_group, *[_lib.ptr(t) for t in outs], flags, _lib.ptr(ws), nbytes, _lib.stream_ptr())
    if rc != 0:                                                    # ESRError is a RuntimeError, as the reference raises
        raise (_lib.ESRError if flags else RuntimeError)("dcn_v2_backward: " + L.esr_last_error().decode())
    return outs
