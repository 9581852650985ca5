"""Drop-in for codes/DSN/receptive_cal.py (and codes/SRN/utils/receptive_cal.py): receptive-field
bookkeeping + the domain-distance map (DDM) of create_dataset_modified.py:14-24, with the O(patch x rf^2) numpy
scatter (`weights_matrix`, receptive_cal.py:34-43) replaced by the dasr_ddm gather kernels.

Same names and return values: outFromIn, printLayer, receptive_cal, getWeights, weights_matrix, layerInfos.
`getWeights` returns a float64 numpy array shaped like `img` ([1,1,h,w]) — the array the reference np.save()s as
`ddm_target/<name>.npy` and that LRHR_wavelet_unpairEq_fake_w_dataset.py:64-68 loads.
Quirk preserved: the reference overwrites (jump, rf, start) of the H axis with the W axis' values
(receptive_cal.py:56-57) before calling weights_matrix."""
import math

import numpy as np
import torch

layerInfos = []


def outFromIn(conv, layerIn):
    n_in, j_in, r_in, start_in = layerIn[0], layerIn[1], layerIn[2], layerIn[3]
    k, s, p = conv[0], conv[1], conv[2]
    n_out = math.floor((n_in - k + 2 * p) / s) + 1
    actualP = (n_out - 1) * s - n_in + k
    pL = math.floor(actualP / 2)
    j_out = j_in * s
    r_out = r_in + (k - 1) * j_in
    start_out = start_in + ((k - 1) / 2 - pL) * j_in
    return n_out, j_out, r_out, start_out


def printLayer(layer, layer_name):
    print(layer_name + ":")
    print("\t n features: %s \n \t jump: %s \n \t receptive size: %s \t start: %s " % (layer[0], layer[1], layer[2], layer[3]))


def receptive_cal(imsize, convnet):
    currentLayer = [imsize, 1, 1, 0.5]
    for i in range(len(convnet)):
        currentLayer = outFromIn(convnet[i], currentLayer)
        layerInfos.append(currentLayer)
    return currentLayer


def _windows(n_f, size, jump, rf, start):
    """[lo, hi) of every window (receptive_cal.py:40-41, clipped like numpy slicing) and, per coordinate, the contiguous
    range of windows covering it."""
    lo = [int(max(0, start + i * jump - rf // 2)) for i in range(n_f)]
    hi = [min(size, max(0, int(start + i * jump + rf - rf // 2))) for i in range(n_f)]
    first = np.full(size, 1, dtype=np.int32)       # empty range (first > last) where nothing covers the coordinate
    last = np.full(size, 0, dtype=np.int32)
    seen = np.zeros(size, dtype=bool)
    for i in range(n_f):
        for c in range(lo[i], hi[i]):
            if not seen[c]:
                first[c], seen[c] = i, True
            last[c] = i
    return first, last


def weights_matrix(patch, img, n_f_h, n_f_w, jump, rf, start):
    """Scatter-add of the patch values over their receptive-field windows (receptive_cal.py:34-43) as a CUDA gather.
    Returns the SUM only (like the reference); getWeights divides by the coverage count."""
    s, cnt = _ddm(patch, img, n_f_h, n_f_w, jump, rf, start)
    return s * cnt


def _ddm(patch, img, n_f_h, n_f_w, jump, rf, start):
    from dasr_b200 import _lib, ops
    if not torch.cuda.is_available():
        raise _lib.DasrError('receptive_cal.getWeights runs on CUDA only; no CPU fallback exists')
    shape = tuple(img.shape)
    B, C, H, W = shape
    pt = torch.as_tensor(np.asarray(patch, dtype=np.float32) if not torch.is_tensor(patch) else patch.detach().float().cpu().numpy())
    if pt.shape[0] * pt.shape[1] != B * C:
        pt = pt.expand(B, C, pt.shape[2], pt.shape[3])
    pt = pt.contiguous().cuda()
    ilo, ihi = _windows(n_f_h, H, jump, rf, start)
    jlo, jhi = _windows(n_f_w, W, jump, rf, start)
    out = ops.ddm(pt[:, :, :n_f_h, :n_f_w].contiguous(), H, W, ilo, ihi, jlo, jhi)
    cnt = (np.maximum(ihi - ilo + 1, 0).astype(np.float64)[:, None] * np.maximum(jhi - jlo + 1, 0).astype(np.float64)[None, :])
    return out.cpu().numpy().reshape(shape), cnt.reshape(1, 1, H, W)


def getWeights(patch, img, currentLayer_h, currentLayer_w):
    n_f_h, jump, rf, start = currentLayer_h[0], currentLayer_h[1], currentLayer_h[2], currentLayer_h[3]
    n_f_w, jump, rf, start = currentLayer_w[0], currentLayer_w[1], currentLayer_w[2], currentLayer_w[3]   # sic (reference :56-57)
    avg, _ = _ddm(patch, img, n_f_h, n_f_w, jump, rf, start)
    return avg


def domain_distance_map_handler(fake_img, D_out, convnet, fs_type):
    """create_dataset_modified.py:14-24."""
    if fs_type.lower() == 'gau' or fs_type == 'avg_pool':
        ddm_shape = (fake_img.shape[0], 1, fake_img.shape[2], fake_img.shape[3])
    elif fs_type.lower() == 'wavelet':
        ddm_shape = (fake_img.shape[0], 1, fake_img.shape[2] // 2, fake_img.shape[3] // 2)
    else:
        raise NotImplementedError('Frequency Separation [{:s}] not recognized'.format(fs_type))
    ddm = torch.zeros(ddm_shape)
    currentLayer_h, currentLayer_w = receptive_cal(ddm.shape[2], convnet), receptive_cal(ddm.shape[3], convnet)
    return getWeights(D_out, ddm, currentLayer_h, currentLayer_w)
