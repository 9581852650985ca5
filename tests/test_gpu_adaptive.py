"""GPU tests of the adaptive-weight generators: the weight-map epilogue of the wgmma conv (dasr_conv_tc_map /
dasr_conv_tc2_map) against the fp32 conv, both generators against the reference fixtures and the oracle, and the
DASR_Adaptive_Model test path end to end through create_model."""
import os

import pytest
import torch

from oracle import adaptive_oracle as AO
from oracle import srn_oracle as O

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CONFIG = os.path.join(ROOT, 'tests', 'golden', 'test_DASR_Adaptive.json')


def rel_linf(a, b):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def _nhwc(shape, seed, dt, scale=1.0):
    return (O.synth(shape, seed, scale)).to(dt).cuda()


def _conv_f32(u16, w, b, **kw):
    from dasr_b200 import ops
    u = u16.float().contiguous()
    out = torch.empty(u.shape[:3] + (w.shape[0],), device='cuda')
    ops.conv2d_f32(u, ops.pack_filter_f32(w), b, out, 3, 1, 1, **kw)
    return out


@pytest.mark.parametrize('pair', [False, True])
@pytest.mark.parametrize('dt', [torch.bfloat16, torch.float16])
@pytest.mark.parametrize('hw', [(16, 8), (21, 13), (40, 24)])
def test_map_channel_epilogue_vs_fp32_concat(hw, dt, pair):
    """conv(cat(u, s * map)) + LeakyReLU: 64 channels on the MMAs, the map channel in the epilogue."""
    from dasr_b200 import ops
    H, W = hw
    N, s = 2, 0.2
    u = _nhwc((N, H, W, 64), 1, dt)
    amap = O.synth_image((N, 1, H, W), 2).cuda()
    w = O.synth((64, 65, 3, 3), 3, 0.05).cuda()
    w[:, 64] *= 20
    b = O.synth((64,), 4, 0.05).cuda()
    out = torch.empty((N, H, W, 64), dtype=dt, device='cuda')
    ops.conv_tc(u, ops.pack_filter_tc(w[:, :64].contiguous(), ops.TC_FPROP, dt), b, out, act=ops.ACT_LRELU, slope=0.2, pair=pair,
                amap=amap, map_mode=ops.MAP_CHANNEL, map_scale=s, map_w=ops.map_channel_taps(w, 64))
    cat = torch.cat((u.float(), (amap * s).permute(0, 2, 3, 1)), 3).contiguous()
    ref = _conv_f32(cat, w, b, act=ops.ACT_LRELU, slope=0.2)
    assert rel_linf(out, ref) < 1e-2        # bf16 / f16 operand rounding against fp32 (as test_rrdbnet_bf16_tcgen05_vs_oracle)


@pytest.mark.parametrize('pair', [False, True])
@pytest.mark.parametrize('dt', [torch.bfloat16, torch.float16])
@pytest.mark.parametrize('hw', [(16, 8), (21, 13), (40, 24)])
@pytest.mark.parametrize('with_pre', [False, True])
def test_map_scale_epilogue_vs_fp32_composition(hw, dt, pair, with_pre):
    """v = map * (alpha * act(conv(u) + bias + pre) + beta1 * res1) + beta2 * res2."""
    from dasr_b200 import ops
    H, W = hw
    N = 2
    u = _nhwc((N, H, W, 64), 11, dt)
    pre = _nhwc((N, H, W, 64), 12, dt, 0.5) if with_pre else None
    r1, r2 = _nhwc((N, H, W, 64), 13, dt), _nhwc((N, H, W, 64), 14, dt)
    amap = O.synth_image((N, 1, H, W), 15).cuda()
    w, b = O.synth((64, 64, 3, 3), 16, 0.05).cuda(), O.synth((64,), 17, 0.05).cuda()
    out = torch.empty((N, H, W, 64), dtype=dt, device='cuda')
    ops.conv_tc(u, ops.pack_filter_tc(w, ops.TC_FPROP, dt), b, out, act=ops.ACT_LRELU, slope=0.2, alpha=0.2, pre=pre,
                res1=r1, beta1=1.0, res2=r2, beta2=0.1, pair=pair, amap=amap, map_mode=ops.MAP_SCALE)
    z = _conv_f32(u, w, b)
    if with_pre:
        z = z + pre.float()
    m = amap.permute(0, 2, 3, 1)
    ref = m * (0.2 * torch.nn.functional.leaky_relu(z, 0.2) + r1.float()) + 0.1 * r2.float()
    assert rel_linf(out, ref) < 1e-2


def _generator(name, g):
    from dasr_b200.srn.models.modules import architecture as A
    cls = A.RRDBNet_Residual_conv_concat if name == 'concat' else A.RRDBNet_Residual_conv
    net = cls(3, 3, 64, g['nb'], nb_ada=g['nb_ada'])
    sd = AO.synth_adaptive_g(g['nb'], g['nb_ada'], name == 'concat', g['w_seed'], 0.3)
    net.load_state_dict(sd, strict=True)
    return net.cuda().eval(), sd


@pytest.mark.parametrize('name', ['concat', 'plain'])
def test_adaptive_generators_fp32_vs_reference_and_bf16_fp16_vs_oracle(golden, name):
    fx = golden('adaptive_g.pt')
    g = fx[name]
    net, sd = _generator(name, g)
    for rec in g['outs']:
        shape = rec['shape']
        x, a = O.synth_image(shape, rec['x_seed']), O.synth_image((shape[0], 1) + shape[2:], rec['map_seed'])
        with torch.no_grad():
            net.precision = 'fp32'
            assert rel_linf(net(x.cuda(), a.cuda()), rec['out']) < 1e-3
            ref = AO.adaptive_rrdb_forward(x, a, sd, g['nb'], g['nb_ada'], name == 'concat')
            for prec in ('bf16', 'fp16'):
                net.precision = prec
                for _ in range(3):          # eager, eager (graph key seen), captured graph replay
                    assert rel_linf(net(x.cuda(), a.cuda()), ref) < 1e-2, prec


@pytest.mark.parametrize('name', ['concat', 'plain'])
def test_adaptive_generators_batch_equals_per_image(golden, name):
    """The map is indexed per image: a batched bf16 forward equals the per-image forwards bit for bit."""
    net, _ = _generator(name, golden('adaptive_g.pt')[name])
    net.precision = 'bf16'
    x, a = O.synth_image((3, 3, 40, 72), 331).cuda(), O.synth_image((3, 1, 40, 72), 332).cuda()
    with torch.no_grad():
        full = net(x, a)
        parts = torch.cat([net(x[i:i + 1], a[i:i + 1]) for i in range(3)], 0)
    assert torch.equal(full, parts)


@pytest.mark.parametrize('prec,tol', [('fp32', 1e-3), ('bf16', 2e-2)])
def test_dasr_adaptive_model_test_path_end_to_end(golden, tmp_path, monkeypatch, prec, tol):
    """options/test/test_DASR_Adaptive.json through create_model -> feed_data -> test -> get_current_visuals, with a synthetic
    G checkpoint and a DSN checkpoint ({'models_d_state_dict': ...}) of the map network."""
    from dasr_b200.srn.models import create_model
    from dasr_b200.srn.options.options import dict_to_nonedict, parse
    g = golden('adaptive_test.pt')
    monkeypatch.setenv('DASR_B200_PRECISION', prec)
    g_path, d_path = str(tmp_path / 'G.pth'), str(tmp_path / 'D.tar')
    torch.save(AO.synth_adaptive_g(g['nb'], g['ada_nb'], True, g['g_seed'], 0.3), g_path)
    torch.save({'models_d_state_dict': AO.synth_patchd_state_dict(g['d_seed'])}, d_path)
    opt = parse(CONFIG, is_train=False)
    opt['val_lpips'] = False
    opt['network_G'].update(nb=g['nb'], ada_nb=g['ada_nb'])
    opt['path'].update(pretrain_model_G=g_path, Patch_Discriminator=d_path)
    model = create_model(dict_to_nonedict(opt))
    n, c, h, w = g['lr_shape']
    model.feed_data({'LR': O.synth_image(g['lr_shape'], g['lr_seed']), 'HR': O.synth_image((n, c, 4 * h, 4 * w), g['hr_seed'])}, False)
    model.test()
    vis = model.get_current_visuals()
    assert list(vis.keys()) == g['keys']
    assert rel_linf(model.adaptive_weights, g['map']) < 1e-3
    assert rel_linf(vis['SR'], g['SR']) < tol
    stats = model.net_patchD.state_dict()
    for k, v in g['bn_stats'].items():
        if v.dtype == torch.int64:
            assert int(stats[k]) == int(v), k
        else:
            assert rel_linf(stats[k], v) < 1e-3, k
