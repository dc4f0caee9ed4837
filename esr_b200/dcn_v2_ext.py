"""Drop-in for the reference's `_ext` pybind module (models/DCNv2/src/vision.cpp:4-8), forward operator.

    import esr_b200.dcn_v2_ext as _ext;  sys.modules['_ext'] = _ext       (see esr_b200.dropin)

dcn_v2_forward keeps the reference's 14-argument signature (models/DCNv2/dcn_v2.py:27-42) and its behaviour:
contiguous fp32 CUDA tensors in the NCHW layout, a freshly allocated output, errors as RuntimeError.  Both operators
serve every configuration with equal height / width kernel, stride, padding and dilation; a non-square one, or a tensor
whose shape does not match the geometry, raises RuntimeError before anything is launched.
dcn_v2_backward returns the reference's five gradients (fp32 atomics for grad_input, like the reference; int64 fixed point,
bitwise reproducible, in deterministic mode: esr_b200.train.deterministic()).
"""
import torch

from . import _lib


def _ws(nbytes, device):
    return torch.empty((max(int(nbytes), 256),), dtype=torch.uint8, device=device)


def _check_args(op, input, weight, bias, offset, mask, grad_output, kernel_h, kernel_w, stride_h, stride_w, pad_h, pad_w,
                dilation_h, dilation_w, deformable_group):
    """The checks both operators make before any launch (the CPU-tensor message first, as in the reference).  The kernels
    read offset, mask, bias and grad_output at the sizes the geometry implies, so a tensor of another shape raises here
    instead of being read out of bounds.  -> (B, C, H, W, Co, Ho, Wo)"""
    if not input.is_cuda:
        raise RuntimeError("Not compiled with CPU support")       # there is no CPU path in esr_b200
    tensors = [input, weight, bias, offset, mask] + ([] if grad_output is None else [grad_output])
    if any(t.device != input.device for t in tensors):
        raise RuntimeError("%s: expected all tensors on %s" % (op, input.device))
    for t in tensors:
        if t.dtype != torch.float32:
            raise RuntimeError("%s: expected float32 tensors" % op)
    if input.dim() != 4 or weight.dim() != 4:
        raise RuntimeError("%s: expected 4-d input and weight" % op)
    B, C, H, W = input.shape
    Co = weight.shape[0]
    if kernel_h != kernel_w or stride_h != stride_w or pad_h != pad_w or dilation_h != dilation_w:
        raise RuntimeError("%s: only square kernels / strides are implemented" % op)
    if weight.shape[2] != kernel_h or weight.shape[3] != kernel_w:
        raise RuntimeError("Input shape and kernel shape wont match: (%d x %d vs %d x %d)."
                           % (kernel_h, kernel_w, weight.shape[2], weight.shape[3]))
    if C != weight.shape[1]:
        raise RuntimeError("Input shape and kernel channels wont match: (%d vs %d)." % (C, weight.shape[1]))
    Ho = (H + 2 * pad_h - (dilation_h * (kernel_h - 1) + 1)) // stride_h + 1
    Wo = (W + 2 * pad_w - (dilation_w * (kernel_w - 1) + 1)) // stride_w + 1
    K = kernel_h * kernel_w
    want = [("offset", offset, [B, 2 * deformable_group * K, Ho, Wo]), ("mask", mask, [B, deformable_group * K, Ho, Wo]),
            ("bias", bias, [Co])]
    if grad_output is not None:
        want.append(("grad_output", grad_output, [B, Co, Ho, Wo]))
    for name, t, shape in want:
        if list(t.shape) != shape:
            raise RuntimeError("%s: %s has shape %s, expected %s" % (op, name, list(t.shape), shape))
    return B, C, H, W, Co, Ho, Wo


def dcn_v2_forward(input, weight, bias, offset, mask, kernel_h, kernel_w, stride_h, stride_w, pad_h, pad_w,
                   dilation_h, dilation_w, deformable_group):
    B, C, H, W, Co, Ho, Wo = _check_args("dcn_v2_forward", input, weight, bias, offset, mask, None, kernel_h, kernel_w,
                                         stride_h, stride_w, pad_h, pad_w, dilation_h, dilation_w, deformable_group)
    L = _lib.lib()
    args = [t.contiguous() for t in (input, weight, bias, offset, mask)]
    out = torch.empty((B, Co, Ho, Wo), dtype=torch.float32, device=input.device)
    with torch.cuda.device(input.device):
        nbytes = L.esr_dcn_v2_workspace_bytes_ex(B, C, H, W, Co, kernel_h, stride_h, pad_h, dilation_h, deformable_group, 0)
        ws = _ws(nbytes, input.device)
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
    B, C, H, W, Co, _, _ = _check_args("dcn_v2_backward", input, weight, bias, offset, mask, grad_output, kernel_h, kernel_w,
                                       stride_h, stride_w, pad_h, pad_w, dilation_h, dilation_w, deformable_group)
    L = _lib.lib()
    args = [t.contiguous() for t in (input, weight, bias, offset, mask, grad_output)]
    outs = [torch.empty_like(args[0]), torch.empty_like(args[3]), torch.empty_like(args[4]), torch.empty_like(args[1]),
            torch.empty_like(args[2])]
    flags = _lib.DETERMINISTIC if deterministic() else 0
    with torch.cuda.device(input.device):
        nbytes = L.esr_dcn_v2_backward_workspace_bytes_ex(B, C, H, W, Co, kernel_h, stride_h, pad_h, dilation_h, deformable_group,
                                                          flags)
        ws = _ws(nbytes, input.device)
        rc = L.esr_dcn_v2_backward_ex(*[_lib.ptr(t) for t in args], B, C, H, W, Co, kernel_h, stride_h, pad_h, dilation_h,
                                      deformable_group, *[_lib.ptr(t) for t in outs], flags, _lib.ptr(ws), nbytes, _lib.stream_ptr())
    if rc != 0:                                                    # ESRError is a RuntimeError, as the reference raises
        raise (_lib.ESRError if flags else RuntimeError)("dcn_v2_backward: " + L.esr_last_error().decode())
    return outs
