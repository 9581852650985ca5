"""CPU checks of the adaptive-weight generators (RRDBNet_Residual_conv_concat / RRDBNet_Residual_conv) and the
DASR_Adaptive_Model test path: the oracle against the fixtures written by the reference (oracle/gen_golden_adaptive.py), and
the host side of the mirrors (keys, define_G, option file, model construction)."""
import os

import pytest
import torch

from oracle import adaptive_oracle as AO
from oracle import srn_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CONFIG = os.path.join(ROOT, 'tests', 'golden', 'test_DASR_Adaptive.json')


def rel_linf(a, b):
    return float((a - b).abs().max() / b.abs().max())


@pytest.mark.parametrize('name', ['concat', 'plain'])
def test_adaptive_generator_oracle_vs_reference(golden, name):
    g = golden('adaptive_g.pt')[name]
    concat = name == 'concat'
    assert list(AO.adaptive_rrdb_shapes(g['nb'], g['nb_ada'], concat).items()) == g['keys']
    sd = AO.synth_adaptive_g(g['nb'], g['nb_ada'], concat, g['w_seed'], golden('adaptive_g.pt')['gain'])
    assert sum(v.numel() for v in sd.values()) == g['n_params']
    for rec in g['outs']:
        shape = rec['shape']
        x, a = O.synth_image(shape, rec['x_seed']), O.synth_image((shape[0], 1) + shape[2:], rec['map_seed'])
        with torch.no_grad():
            out = AO.adaptive_rrdb_forward(x, a, sd, g['nb'], g['nb_ada'], concat)
        assert rel_linf(out, rec['out']) <= 1e-5
        assert rec['map_effect'] > 0.04          # the map term is visible above the bf16 tolerance of the GPU tests


def test_adaptive_test_path_oracle_vs_reference(golden):
    g = golden('adaptive_test.pt')
    sd = AO.synth_adaptive_g(g['nb'], g['ada_nb'], True, g['g_seed'], 0.3)
    x = O.synth_image(g['lr_shape'], g['lr_seed'])
    with torch.no_grad():
        out = AO.adaptive_rrdb_forward(x, g['map'], sd, g['nb'], g['ada_nb'], True)
    assert rel_linf(out, g['fake_H']) <= 1e-5
    assert torch.equal(g['SR'], g['fake_H'][0])


@pytest.mark.parametrize('which,nb_ada,concat', [('RRDB_Residual_conv_concat', 2, True), ('RRDB_Residual_conv', 1, False)])
def test_define_G_keys_match_reference(golden, which, nb_ada, concat):
    from dasr_b200.srn.models import networks
    from dasr_b200.srn.options.options import dict_to_nonedict
    opt = dict_to_nonedict({'is_train': False, 'gpu_ids': None, 'network_G': {
        'which_model_G': which, 'norm_type': None, 'mode': 'CNA', 'nf': 64, 'nb': 1, 'in_nc': 3, 'out_nc': 3, 'gc': 32,
        'scale': 4, 'ada_nb': 2}})
    net = networks.define_G(opt)
    assert [(k, tuple(v.shape)) for k, v in net.state_dict().items()] == golden('adaptive_g.pt')['concat' if concat else 'plain']['keys']
    # RRDB_Residual_conv ignores ada_nb: define_G does not pass it (networks.py:131-134), one adaptive block
    assert net.nb_ada == nb_ada


def test_adaptive_generator_refuses_grad_and_cpu():
    from dasr_b200 import _lib
    from dasr_b200.srn.models.modules.architecture import RRDBNet_Residual_conv_concat
    net = RRDBNet_Residual_conv_concat(3, 3, 64, 1, nb_ada=1)
    x, a = torch.zeros(1, 3, 8, 8), torch.zeros(1, 1, 8, 8)
    with pytest.raises(NotImplementedError, match='training of the adaptive generators is not built'):
        net(x, a)
    with torch.no_grad(), pytest.raises(_lib.DasrError):
        net(x, a)


def _test_opt(g_path=None, d_path=None):
    from dasr_b200.srn.options.options import dict_to_nonedict, parse
    opt = parse(CONFIG, is_train=False)
    opt['gpu_ids'] = None
    opt['val_lpips'] = False
    opt['network_G'].update(nb=1, ada_nb=2)
    opt['path'].update(pretrain_model_G=g_path, Patch_Discriminator=d_path)
    return dict_to_nonedict(opt)


def test_shipped_test_config_parses():
    from dasr_b200.srn.options.options import parse
    opt = parse(CONFIG, is_train=False)
    assert opt['model'] == 'DASR_Adaptive_Model'
    assert opt['network_G']['which_model_G'] == 'RRDB_Residual_conv_concat' and opt['network_G']['ada_nb'] == 4
    assert opt['network_patchD']['norm_layer'] == 'Batch' and opt['network_patchD']['FS_type'] == 'avg_pool'


def test_create_model_builds_test_path_on_cpu_and_refuses_compute(tmp_path):
    from dasr_b200 import _lib
    from dasr_b200.srn.models import create_model
    g_path, d_path = str(tmp_path / 'G.pth'), str(tmp_path / 'D.tar')
    torch.save(AO.synth_adaptive_g(1, 2, True, 1, 0.3), g_path)
    torch.save({'models_d_state_dict': AO.synth_patchd_state_dict(2)}, d_path)
    model = create_model(_test_opt(g_path, d_path))
    assert type(model).__name__ == 'DASR_Adaptive_Model'
    assert torch.equal(model.netG.state_dict()['fea_conv.0.weight'], torch.load(g_path)['fea_conv.0.weight'])
    model.feed_data({'LR': torch.zeros(1, 3, 8, 8)}, False)
    with pytest.raises(_lib.DasrError):
        model.test()


def test_training_is_refused_with_reason():
    from dasr_b200.srn.models import create_model
    opt = _test_opt()
    opt['is_train'] = True
    with pytest.raises(NotImplementedError, match='FS'):
        create_model(opt)
