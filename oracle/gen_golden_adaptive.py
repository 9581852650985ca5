"""Generate tests/golden/adaptive_g.pt and tests/golden/adaptive_test.pt by running the UNMODIFIED reference
(<DASR checkout>/codes/SRN) on CPU: the adaptive-weight generators RRDBNet_Residual_conv_concat / RRDBNet_Residual_conv and the
DASR_Adaptive_Model test path.  Test infrastructure only, imported like oracle/gen_golden.py (DASR_REFERENCE = the checkout's
root, oracle/ref_stubs for the third-party modules the reference imports at module level).

    python oracle/gen_golden_adaptive.py

Stand-in: the reference's networks.define_patchD returns an unbound name when gpu_ids is empty (networks.py:242-245: the
net is only assigned inside `if gpu_ids:`).  For the CPU run the script replaces it by the same construction without the
DataParallel wrapper.  All weights and inputs come from oracle.srn_oracle.synth* and oracle.adaptive_oracle (hash based, no RNG).
"""
import json
import os
import sys
import tempfile
from collections import OrderedDict

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF = os.path.join(os.environ.get('DASR_REFERENCE', 'DASR'), 'codes')   # a ShuhangGu/DASR checkout
sys.path.insert(0, os.path.join(HERE, 'ref_stubs'))
sys.path.insert(0, os.path.join(REF, 'SRN'))
sys.path.insert(0, REF)
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import models.modules.architecture as arch  # noqa: E402  (reference)
import models.networks as ref_networks  # noqa: E402
from models import create_model  # noqa: E402
from options.options import dict_to_nonedict  # noqa: E402

from oracle import adaptive_oracle as AO  # noqa: E402
from oracle import srn_oracle as O  # noqa: E402

OUT = os.path.join(ROOT, 'tests', 'golden')
CONFIG = os.path.join(OUT, 'test_DASR_Adaptive.json')
torch.set_num_threads(8)

# generator fixtures: (name, class, concat, nb, nb_ada, weight seed); nb_ada = 1 for the plain variant (define_G's quirk)
GENERATORS = [('concat', arch.RRDBNet_Residual_conv_concat, True, 1, 2, 301),
              ('plain', arch.RRDBNet_Residual_conv, False, 1, 1, 302)]
GAIN = 0.3
# (x shape, x seed, map seed): a ragged batch of two, and one image spanning several 16 x 8 tiles
INPUTS = [((2, 3, 21, 13), 311, 312), ((1, 3, 40, 24), 313, 314)]
# DASR_Adaptive_Model test path: G = concat variant nb 1 / ada_nb 2, map net = BatchNorm FSD behind an 11x11 box filter
TEST = dict(nb=1, ada_nb=2, g_seed=321, d_seed=322, lr_seed=323, hr_seed=324, lr_shape=(2, 3, 20, 12))


def save(name, obj):
    path = os.path.join(OUT, name)
    torch.save(obj, path)
    print('%-22s %8.1f KB' % (name, os.path.getsize(path) / 1024))


def _define_patchD(opt):
    """networks.py:229-245 without the DataParallel branch (whose return value is the only assignment of `netD`)."""
    o = opt['network_patchD']
    net = arch.FS_Discriminator(kernel_size=o['kernel_size'], D_arch='FSD', filter_type=o['FS_type'], norm_layer=o['norm_layer'])
    ref_networks.init_weights(net, init_type='kaiming', scale=1)
    return net


ref_networks.define_patchD = _define_patchD


def test_opt(config, g_path, d_path, gpu_ids=None):
    """The shipped test config with the synthetic checkpoints and a small generator (tests/test_gpu_adaptive.py builds the same)."""
    with open(config) as f:
        opt = json.loads(''.join(line.split('//')[0] + '\n' for line in f), object_pairs_hook=OrderedDict)
    opt['is_train'] = False
    opt['gpu_ids'] = gpu_ids
    opt['val_lpips'] = False          # LPIPS needs the pretrained AlexNet; the metric has its own fixtures
    opt['network_G'].update(nb=TEST['nb'], ada_nb=TEST['ada_nb'], scale=opt['scale'])
    opt['path'].update(pretrain_model_G=g_path, Patch_Discriminator=d_path)
    return opt


def gen_generators():
    rec = OrderedDict(gain=GAIN, inputs=INPUTS)
    for name, cls, concat, nb, nb_ada, seed in GENERATORS:
        net = cls(3, 3, 64, nb, gc=32, upscale=4, norm_type=None, act_type='leakyrelu', mode='CNA', upsample_mode='upconv',
                  nb_ada=nb_ada)
        keys = [(k, tuple(v.shape)) for k, v in net.state_dict().items()]
        shapes = AO.adaptive_rrdb_shapes(nb, nb_ada, concat)
        assert keys == list(shapes.items())
        sd = AO.synth_adaptive_g(nb, nb_ada, concat, seed, GAIN)
        net.load_state_dict(sd, strict=True)
        outs = []
        with torch.no_grad():
            for shape, xs, ms in INPUTS:
                x, a = O.synth_image(shape, xs), O.synth_image((shape[0], 1) + shape[2:], ms)
                out = net(x, a)
                zero = net(x, torch.zeros_like(a))
                effect = float((out - zero).abs().max() / out.abs().max())
                print('  %s %s: map effect rel-Linf %.3f' % (name, shape, effect))
                outs.append(dict(shape=shape, x_seed=xs, map_seed=ms, out=out.clone(), map_effect=effect))
        rec[name] = dict(nb=nb, nb_ada=nb_ada, w_seed=seed, keys=keys, n_params=sum(v.numel() for v in sd.values()), outs=outs)
    save('adaptive_g.pt', rec)


def gen_test_path():
    with tempfile.TemporaryDirectory() as tmp:
        g_path, d_path = os.path.join(tmp, 'G.pth'), os.path.join(tmp, 'D.tar')
        torch.save(AO.synth_adaptive_g(TEST['nb'], TEST['ada_nb'], True, TEST['g_seed'], GAIN), g_path)
        torch.save({'models_d_state_dict': AO.synth_patchd_state_dict(TEST['d_seed'])}, d_path)
        model = create_model(dict_to_nonedict(test_opt(CONFIG, g_path, d_path)))
        n, c, h, w = TEST['lr_shape']
        data = {'LR': O.synth_image(TEST['lr_shape'], TEST['lr_seed']), 'HR': O.synth_image((n, c, 4 * h, 4 * w), TEST['hr_seed'])}
        model.feed_data(data, False)
        model.test()
        vis = model.get_current_visuals()
        stats = OrderedDict((k, v.clone()) for k, v in model.net_patchD.state_dict().items() if 'running' in k or 'batches' in k)
        save('adaptive_test.pt', dict(TEST, SR=vis['SR'].clone(), fake_H=model.fake_H.clone(), map=model.adaptive_weights.clone(),
                                      bn_stats=stats, keys=list(vis.keys())))


if __name__ == '__main__':
    gen_generators()
    gen_test_path()
