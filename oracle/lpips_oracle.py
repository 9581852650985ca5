"""CPU oracle for LPIPS v0.1 (AlexNet trunk, linear calibration) — TEST INFRASTRUCTURE ONLY; prepared for the next row of
SURVEY.md §8f (feature_criterion "LPIPS" of three shipped DASR configs and the validation metric).

Restates <DASR checkout>/codes/PerceptualSimilarity: models/util.py:26-44 (PerceptualLoss.forward with normalize=True),
networks_basic.py:27-107 (PNetLin, ScalingLayer, NetLinLayer in eval mode), pretrained_networks.py:57-96 (AlexNet
slices relu1..relu5), util.normalize_tensor (eps 1e-10) and the spatial average.  Pinned by tests/golden/lpips_alex.pt
(oracle/gen_golden_lpips.py drives the reference's PNetLin with synthetic AlexNet conv weights — the torchvision
checkpoint is not available offline — and the reference's own linear-layer weights weights/v0.1/alex.pth)."""
from collections import OrderedDict

import torch
import torch.nn.functional as F

ALEX_CONVS = [(64, 3, 11, 4, 2), (192, 64, 5, 1, 2), (384, 192, 3, 1, 1), (256, 384, 3, 1, 1), (256, 256, 3, 1, 1)]   # cout, cin, k, s, p
ALEX_FEATURE_IDX = [0, 3, 6, 8, 10]                      # torchvision alexnet.features indices of the convs
SHIFT = (-0.030, -0.088, -0.188)
SCALE = (0.458, 0.448, 0.450)


def alex_shapes():
    """state_dict layout of the reference's PNetLin.net (slice{1..5}.{features index}.weight|bias)."""
    s = OrderedDict()
    for i, ((co, ci, k, _, _), fi) in enumerate(zip(ALEX_CONVS, ALEX_FEATURE_IDX)):
        s['net.slice%d.%d.weight' % (i + 1, fi)] = (co, ci, k, k)
        s['net.slice%d.%d.bias' % (i + 1, fi)] = (co,)
    return s


def alex_features(x, sd):
    outs, t = [], x
    for i, ((_, _, _, s, p), fi) in enumerate(zip(ALEX_CONVS, ALEX_FEATURE_IDX)):
        if i in (1, 2):
            t = F.max_pool2d(t, 3, 2)                    # features[2], features[5]
        t = F.relu(F.conv2d(t, sd['net.slice%d.%d.weight' % (i + 1, fi)], sd['net.slice%d.%d.bias' % (i + 1, fi)], stride=s, padding=p))
        outs.append(t)
    return outs


def lpips(pred, target, sd, lins):
    """pred, target in [0, 1] ([N,3,H,W]); lins: five [1,C,1,1] non-negative weights.  Returns [N,1,1,1]."""
    shift = torch.tensor(SHIFT).view(1, 3, 1, 1)
    scale = torch.tensor(SCALE).view(1, 3, 1, 1)
    prep = lambda t: ((2 * t - 1) - shift) / scale
    f0, f1 = alex_features(prep(target), sd), alex_features(prep(pred), sd)      # model.forward(target, pred)
    val = 0
    for a, b, w in zip(f0, f1, lins):
        na = a / (a.pow(2).sum(1, keepdim=True).sqrt() + 1e-10)
        nb = b / (b.pow(2).sum(1, keepdim=True).sqrt() + 1e-10)
        val = val + F.conv2d((na - nb) ** 2, w).mean([2, 3], keepdim=True)
    return val
