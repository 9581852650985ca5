"""CPU oracle of the adaptive-weight RRDB generators (RRDBNet_Residual_conv_concat / RRDBNet_Residual_conv) and of the
synthetic checkpoints of the DASR_Adaptive_Model test path — TEST INFRASTRUCTURE ONLY, in plain PyTorch (CPU, fp32) like
oracle/srn_oracle.py, whose RRDB pieces it reuses.  Pinned against the reference by tests/golden/adaptive_*.pt
(oracle/gen_golden_adaptive.py, tests/test_oracle_golden_adaptive.py).
"""
import math
from collections import OrderedDict

import torch
import torch.nn.functional as F

from oracle.srn_oracle import _conv, rdb_forward, synth, synth_state_dict


# --------------------------------------------------------------------------------------------------
# adaptive-weight RRDB generators (architecture.py:208-297, block.py:462-528)
# --------------------------------------------------------------------------------------------------


def adaptive_rrdb_shapes(nb, nb_ada, concat, in_nc=3, out_nc=3, nf=64, gc=32, upscale=4):
    """state_dict key -> shape of RRDBNet_Residual_conv_concat (concat) / RRDBNet_Residual_conv.  B.sequential returns a
    single block itself, so nb = 1 / nb_ada = 1 drop the block index from the keys."""
    s = OrderedDict()
    s['fea_conv.0.weight'] = (nf, in_nc, 3, 3)
    s['fea_conv.0.bias'] = (nf,)

    def rdbs(prefix):
        for r in (1, 2, 3):
            for c in range(1, 6):
                s['%sRDB%d.conv%d.0.weight' % (prefix, r, c)] = (gc if c < 5 else nf, nf + (c - 1) * gc, 3, 3)
                s['%sRDB%d.conv%d.0.bias' % (prefix, r, c)] = (gc if c < 5 else nf,)
    for b in range(nb):
        rdbs('rb_blocks.' if nb == 1 else 'rb_blocks.%d.' % b)
    for b in range(nb_ada):
        pre = 'rb_blocks_ada.' if nb_ada == 1 else 'rb_blocks_ada.%d.' % b
        rdbs(pre)
        for name in (('adaptive_conv', 'res_conv') if concat else ('res_conv',)):
            s['%s%s.0.weight' % (pre, name)] = (nf, nf + (1 if concat else 0), 3, 3)
            s['%s%s.0.bias' % (pre, name)] = (nf,)
            s['%s%s.2.weight' % (pre, name)] = (nf, nf, 3, 3)
            s['%s%s.2.bias' % (pre, name)] = (nf,)
    s['LR_conv.0.weight'] = (nf, nf, 3, 3)
    s['LR_conv.0.bias'] = (nf,)
    n_up = int(math.log(upscale, 2))
    for i in [1 + 3 * u for u in range(n_up)] + [3 * n_up, 3 * n_up + 2]:
        s['up_conv.%d.weight' % i] = (out_nc if i == 3 * n_up + 2 else nf, nf, 3, 3)
        s['up_conv.%d.bias' % i] = (out_nc if i == 3 * n_up + 2 else nf,)
    return s


def adaptive_rrdb_forward(x, a, sd, nb, nb_ada, concat, upscale=4):
    """RRDBNet_Residual_conv(_concat).forward(x, a): fea -> adaptive blocks -> RRDBs -> LR_conv + fea -> up_conv."""
    fea = _conv(x, sd, 'fea_conv.0')
    t = fea
    for b in range(nb_ada):
        pre = 'rb_blocks_ada.' if nb_ada == 1 else 'rb_blocks_ada.%d.' % b
        two = lambda v, name: _conv(_conv(v, sd, pre + name + '.0', True), sd, pre + name + '.2', True)
        u = t
        if concat:           # block.py:522-528
            for r in (1, 2, 3):
                t = rdb_forward(two(torch.cat((t, a * 0.2), 1), 'adaptive_conv'), sd, pre + 'RDB%d' % r)
            t = t * 0.2 + two(torch.cat((u, a * 1), 1), 'res_conv')
        else:                # block.py:483-488
            for r in (1, 2, 3):
                t = rdb_forward(t, sd, pre + 'RDB%d' % r)
            t = t * (a * 1) + two(u, 'res_conv') * 0.1
    for b in range(nb):
        inp = t
        for r in (1, 2, 3):
            t = rdb_forward(t, sd, ('rb_blocks.' if nb == 1 else 'rb_blocks.%d.' % b) + 'RDB%d' % r)
        t = t * 0.2 + inp
    t = _conv(t, sd, 'LR_conv.0') + fea
    n_up = int(math.log(upscale, 2))
    for u in range(n_up):
        t = _conv(F.interpolate(t, scale_factor=2, mode='nearest'), sd, 'up_conv.%d' % (1 + 3 * u), True)
    t = _conv(t, sd, 'up_conv.%d' % (3 * n_up), True)
    return _conv(t, sd, 'up_conv.%d' % (3 * n_up + 2))


def synth_patchd_state_dict(seed, n_in=3):
    """Synthetic state_dict of the BatchNorm FS patch discriminator (DSN DiscriminatorBasic, norm 'Batch', behind the
    'avg_pool' / 'gau' high-pass filter): the map network of DASR_Adaptive_Model."""
    sd = OrderedDict()
    convs = {0: (64, n_in, 5, 5), 2: (128, 64, 5, 5), 5: (256, 128, 5, 5), 8: (1, 256, 1, 1)}
    for i, (idx, shp) in enumerate(sorted(convs.items())):
        sd['net.net.%d.weight' % idx] = synth(shp, seed * 1000 + 2 * i, math.sqrt(6.0 / (shp[1] * shp[2] * shp[3])))
        sd['net.net.%d.bias' % idx] = synth((shp[0],), seed * 1000 + 2 * i + 1, 0.05)
        if idx in (2, 5):
            c, j = shp[0], idx + 1
            sd['net.net.%d.weight' % j] = synth((c,), seed * 1000 + 100 + idx, 0.1, 1.0)
            sd['net.net.%d.bias' % j] = synth((c,), seed * 1000 + 200 + idx, 0.1)
            sd['net.net.%d.running_mean' % j] = synth((c,), seed * 1000 + 300 + idx, 0.1)
            sd['net.net.%d.running_var' % j] = synth((c,), seed * 1000 + 400 + idx, 0.1, 1.0)
            sd['net.net.%d.num_batches_tracked' % j] = torch.tensor(7)
    return sd


def synth_adaptive_g(nb, nb_ada, concat, seed, gain):
    """Synthetic adaptive generator weights; the map channel of the 65-channel convs is scaled up x40 so that the map term
    changes the output visibly."""
    sd = synth_state_dict(adaptive_rrdb_shapes(nb, nb_ada, concat), seed, gain)
    for k, v in sd.items():
        if v.dim() == 4 and v.shape[1] == 65:
            v[:, 64] *= 40.0
    return sd
