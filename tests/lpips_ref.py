"""TEST INFRASTRUCTURE ONLY -- torch restatement of LPIPS v0.1 with the AlexNet backbone, any dtype and device.

Follows loss/PerceptualSimilarity/models: PerceptualLoss.forward (__init__.py:32-46, normalize 2x - 1, then
DistModel.forward(target, pred)), PNetLin.forward (networks_basic.py:73-101) with ScalingLayer (:103-110, fp32 buffers),
pretrained_networks.py:57-95 alexnet (torchvision alexnet().features sliced at relu1 .. relu5), normalize_tensor
(__init__.py:48-50) and NetLinLayer's bias-free 1x1 conv; and loss/restore.py:18-39 perceptual_loss.__call__'s channel logic.
seeded_alexnet / seeded_heads build the weights from an explicit torch.Generator, so any machine rebuilds them without the
reference or a download.  tests/golden/make_golden_lpips.py pins this restatement to the reference's own code.
"""
import torch
import torch.nn.functional as F

CHANNELS = (64, 192, 384, 256, 256)
ALEX_SHAPES = (("features.0", (64, 3, 11, 11)), ("features.3", (192, 64, 5, 5)), ("features.6", (384, 192, 3, 3)),
               ("features.8", (256, 384, 3, 3)), ("features.10", (256, 256, 3, 3)))


def seeded_alexnet(seed=0):
    """torchvision alexnet state-dict entries features.{0,3,6,8,10}.{weight,bias} (fp32, CPU): He-scaled normal weights and
    small positive biases, so that every ReLU layer stays alive on count images."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for name, shape in ALEX_SHAPES:
        fan_in = shape[1] * shape[2] * shape[3]
        sd[name + ".weight"] = torch.randn(shape, generator=g) * (2.0 / fan_in) ** 0.5
        sd[name + ".bias"] = torch.rand((shape[0],), generator=g) * 0.1
    return sd


def seeded_heads(seed=1):
    """v0.1 heads lin{l}.model.1.weight [1, C, 1, 1], non-negative like the trained ones."""
    g = torch.Generator().manual_seed(seed)
    return {f"lin{l}.model.1.weight": torch.rand((1, c, 1, 1), generator=g) * 0.1 for l, c in enumerate(CHANNELS)}


def features(x, sd):
    """relu1 .. relu5 of alexnet().features for x [N, 3, H, W] (already scaled)."""
    w = {k: v.to(device=x.device, dtype=x.dtype) for k, v in sd.items()}
    h1 = F.relu(F.conv2d(x, w["features.0.weight"], w["features.0.bias"], stride=4, padding=2))
    h2 = F.relu(F.conv2d(F.max_pool2d(h1, 3, 2), w["features.3.weight"], w["features.3.bias"], padding=2))
    h3 = F.relu(F.conv2d(F.max_pool2d(h2, 3, 2), w["features.6.weight"], w["features.6.bias"], padding=1))
    h4 = F.relu(F.conv2d(h3, w["features.8.weight"], w["features.8.bias"], padding=1))
    h5 = F.relu(F.conv2d(h4, w["features.10.weight"], w["features.10.bias"], padding=1))
    return [h1, h2, h3, h4, h5]


def scaling_layer(x):
    shift = torch.tensor([-.030, -.088, -.188], dtype=torch.float32).to(x)[None, :, None, None]
    scale = torch.tensor([.458, .448, .450], dtype=torch.float32).to(x)[None, :, None, None]
    return (x - shift) / scale


def normalize_tensor(f, eps=1e-10):
    return f / (torch.sqrt(torch.sum(f ** 2, dim=1, keepdim=True)) + eps)


def pnetlin(in0, in1, sd, heads):
    """PNetLin.forward: [N, 1, 1, 1]."""
    o0, o1 = features(scaling_layer(in0), sd), features(scaling_layer(in1), sd)
    val = None
    for l in range(5):
        d = (normalize_tensor(o0[l]) - normalize_tensor(o1[l])) ** 2
        w = heads[f"lin{l}.model.1.weight"].to(device=d.device, dtype=d.dtype)
        r = F.conv2d(d, w).mean([2, 3], keepdim=True)
        val = r if val is None else val + r
    return val


def perceptual_model(pred, target, sd, heads, normalize=False):
    """PerceptualLoss.forward."""
    if normalize:
        target = 2 * target - 1
        pred = 2 * pred - 1
    return pnetlin(target, pred, sd, heads)


def perceptual_loss(pred, target, sd, heads, weight=1.0, normalize=True):
    """loss/restore.py:18-39 perceptual_loss.__call__ (raises where the reference raises)."""
    assert pred.size() == target.size()
    if pred.shape[1] == 1:
        pred = torch.cat([pred, pred, pred], dim=1)
        target = torch.cat([target, target, target], dim=1)
        dist = perceptual_model(pred, target, sd, heads, normalize)
    elif pred.shape[1] == 3:
        dist = perceptual_model(pred, target, sd, heads, normalize)
    else:
        num_ch = pred.shape[1]
        dist = 0
        for idx in range(num_ch):
            dist += perceptual_model(pred[:, idx].repeat(1, 3, 1, 1), target[:, idx].repeat(1, 3, 1, 1), sd, heads, normalize)
        dist /= num_ch
    return weight * dist.mean()


def pair_distance(a, b, sd, heads, normalize=True):
    """LPIPS of one image pair a, b [3, H, W] as the C ABI computes it (perceptual_model on a batch of one), float."""
    return float(perceptual_model(a[None], b[None], sd, heads, normalize).reshape(()))
