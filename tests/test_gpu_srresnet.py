"""SRResNet on the wgmma kernels, on the GPU.

  * The pixel-shuffle conv (ops.conv_tc_ps) is bit-identical to torch's pixel shuffle of the plain launch with the same
    filter: each output element is the same fp32 sum, only its store goes elsewhere.
  * The unshuffle-and-mask kernel is bit-identical to torch's pixel_unshuffle of the masked gradient.
  * The TC_PS pack (single-filter kernel and the training step's batch jobs) holds the float64 encoding, rounded.
  * Under the shadow fixture every launch of SRResNet inference and of one training step agrees with its float64 contract.
  * Module level: the reference's f1 fixture and SRResNet-16 against the fp32 layer list, within derived bounds; the
    mixed-precision SRModel steps against the fp32 ones; the CUDA-graph step against the eager one; precision 'fp32' and
    the default against the layer list, bit for bit.

Bounds.  A 16-bit mode rounds every stored activation (and gradient) and every filter once, each with relative error at
most u = 2^-8 (bf16: 8 significant bits) or 2^-11 (fp16: 11), the bound conv_tc_ref uses for one rounding; the fp32
accumulation adds nothing at this scale (K <= 2304 products, 2^-24 each).  To first order the relative errors of the
roundings an output depends on add up, so with R such roundings on its path rel-Linf <= R u.  The forward of SRResNet-nb
at x4 has R = 2 (3 + 2 nb + 2) + 1: one filter rounding and one output rounding per conv (the last layer writes fp32,
counted anyway) and the input's.  Measured on an H100 80GB HBM3 (700 W power limit): the f1 fixture 1.16e-2 (bf16) and
1.31e-3 (fp16) against bounds 7.4e-2 / 9.3e-3; SRResNet-16 2.15e-2 / 2.74e-3 against 1.8e-1 / 2.3e-2; the SRModel
gradients 1.57e-2 rel-L2 against 2.2e-1."""
import inspect

import pytest
import torch
import torch.nn.functional as F

from oracle import srn_oracle as O
from tests.test_gpu_conv_tc_exact import shadow  # noqa: F401  (the pytest fixture)

pytestmark = pytest.mark.gpu

U = {'bf16': 2.0 ** -8, 'fp16': 2.0 ** -11}
DT = {'bf16': torch.bfloat16, 'fp16': torch.float16}


def rel_linf(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def rel_l2(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def fwd_roundings(nb):
    return 2 * (3 + 2 * nb + 2) + 1


def _srresnet(nb, nf=64, upscale=4, res_scale=1, seed=81):
    from dasr_b200.srn.models.modules.sr_nets import SRResNet
    net = SRResNet(3, 3, nf, nb, upscale=upscale, norm_type=None, act_type='relu', mode='CNA', res_scale=res_scale,
                   upsample_mode='pixelshuffle')
    sd = net.state_dict()
    for i, (k, v) in enumerate(sd.items()):
        fan_in = v[0].numel()
        sd[k] = O.synth(tuple(v.shape), seed * 1000 + i, (6.0 / fan_in) ** 0.5 if v.dim() == 4 else 0.05)
    net.load_state_dict(sd)
    return net


def _bits(t):
    return t.view(torch.int16) if t.element_size() == 2 else t.view(torch.int32)


# ------------------------------------------------------------------------------------------------------------------------
# kernels
# ------------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('hw', [(13, 29), (16, 32)], ids=['ragged', 'tiles'])
@pytest.mark.parametrize('act', ['none', 'relu'])
@pytest.mark.parametrize('nf', [32, 64])
@pytest.mark.parametrize('prec', ['bf16', 'fp16'])
def test_ps_launch_is_pixel_shuffle_of_the_plain_launch(prec, nf, act, hw):
    from dasr_b200 import ops
    dt = DT[prec]
    H, W = hw
    N = 2
    a = ops.ACT_RELU if act == 'relu' else ops.ACT_NONE
    x = O.synth((N, H, W, nf), 11 + nf).to(dt).cuda()
    w = O.synth((4 * nf, nf, 3, 3), 12 + nf, (6.0 / (9 * nf)) ** 0.5).cuda()
    b = O.synth((4 * nf,), 13 + nf, 0.1).cuda()
    nt = 64 if nf % 64 == 0 else 32
    plain = torch.empty((N, H, W, 4 * nf), dtype=dt, device='cuda')
    ops.conv_tc(x, ops.pack_filter_tc(w, ops.TC_FPROP, dt), b, plain, nt=nt, act=a)
    want = F.pixel_shuffle(plain.permute(0, 3, 1, 2), 2).permute(0, 2, 3, 1).contiguous()
    # into a channel slice of a wider tensor: the channels around it must keep their bits
    wide = O.synth((N, 2 * H, 2 * W, nf + 64), 14).to(dt).cuda()
    before = wide.clone()
    ops.conv_tc_ps(x, ops.pack_filter_tc(w, ops.TC_PS, dt), b, ops.View(wide, nf, 32), act=a)
    torch.cuda.synchronize()
    got = wide[..., 32:32 + nf].contiguous()
    assert torch.equal(_bits(got), _bits(want)), '%d of %d elements differ' % (int((got != want).sum()), got.numel())
    assert torch.equal(_bits(wide[..., :32]), _bits(before[..., :32]))
    assert torch.equal(_bits(wide[..., 32 + nf:]), _bits(before[..., 32 + nf:]))
    if a == ops.ACT_RELU:
        assert bool((got == 0).any()) and bool((got > 0).any())


@pytest.mark.parametrize('masked', [True, False])
@pytest.mark.parametrize('shape', [(2, 7, 13, 64), (1, 16, 8, 32)])
def test_unshuffle_mask_kernel_is_bit_identical(shape, masked):
    from dasr_b200 import ops
    N, H, W, C = shape
    g = O.synth((N, 2 * H, 2 * W, C), 21).to(torch.bfloat16).cuda()
    y = O.synth((N, 2 * H, 2 * W, C), 22).to(torch.bfloat16).cuda() if masked else None
    out = torch.full((N, H, W, 4 * C), float('nan'), dtype=torch.bfloat16, device='cuda')
    ops.pixel_unshuffle_mask(g, y, out)
    gm = g * (y > 0) if masked else g
    want = F.pixel_unshuffle(gm.permute(0, 3, 1, 2), 2).permute(0, 2, 3, 1).contiguous()
    torch.cuda.synchronize()
    assert torch.equal(_bits(out), _bits(want))


def test_ps_packs_hold_the_float64_encoding():
    from dasr_b200 import engine, ops
    from tests.test_srresnet_float64 import encode_ps
    w = O.synth((256, 64, 3, 3), 31, 0.2)
    for dt in (torch.bfloat16, torch.float16):
        got = ops.pack_filter_tc(w.cuda(), ops.TC_PS, dt).cpu()
        assert torch.equal(_bits(got), _bits(encode_ps(w).to(dt))), dt
    # the training step's batch jobs: the same bf16 pack, and the dgrad / plain packs of the single-filter kernel
    net = _srresnet(1).cuda()
    params = [p.detach() for p in net.parameters()]
    L = engine.SRResNetLayout(1, 4)
    bp = engine._SRResNetPacker(params, L)
    bp.launch()
    torch.cuda.synchronize()
    for u in range(L.n_up):
        i = L.i_up0 + u
        assert torch.equal(_bits(bp.cache.d[('w', i, ops.TC_PS)][1]), _bits(ops.pack_filter_tc(params[2 * i], ops.TC_PS))), i
        assert torch.equal(_bits(bp.cache.d[('wd', i)][1]), _bits(ops.pack_filter_tc(params[2 * i], ops.TC_DGRAD))), i
    assert torch.equal(_bits(bp.cache.d[('w', 1, ops.TC_FPROP)][1]), _bits(ops.pack_filter_tc(params[2], ops.TC_FPROP)))


# ------------------------------------------------------------------------------------------------------------------------
# every launch against its float64 contract (the shadow fixture of test_gpu_conv_tc_exact.py, extended to conv_tc_ps)
# ------------------------------------------------------------------------------------------------------------------------

@pytest.fixture
def shadow_ps(shadow, monkeypatch):
    """shadow + ops.conv_tc_ps: the plain conv model on the parity-major filter rows (conv_tc_ref with its bound), its
    value and bound pixel-shuffled"""
    from dasr_b200 import ops
    from tests.test_gpu_conv_tc_exact import conv_tc_ref
    real = ops.conv_tc_ps

    def conv_tc_ps(inp, w_packed, bias, out, nt=None, act=ops.ACT_NONE, slope=0.2, alpha=1.0):
        o = ops.as_view(out)
        inp_v = ops.as_view(inp)
        torch.cuda.synchronize()
        snap_in = inp_v.t[..., inp_v.coff:inp_v.coff + inp_v.c].clone()
        real(inp, w_packed, bias, out, nt=nt, act=act, slope=slope, alpha=alpha)
        torch.cuda.synchronize()
        C = o.c
        N, H, W, _ = snap_in.shape
        bias_pm = None if bias is None else bias.reshape(C, 4).t().reshape(-1).contiguous()    # parity-major columns
        tmp = torch.empty((N, H, W, 4 * C), dtype=snap_in.dtype, device='cuda')
        ref, tol = conv_tc_ref(snap_in, w_packed, bias_pm, tmp, act=act, slope=slope, alpha=alpha, bound=True)
        shuf = lambda v: v.reshape(N, H, W, 2, 2, C).permute(0, 1, 3, 2, 4, 5).reshape(N, 2 * H, 2 * W, C)
        got = o.t[..., o.coff:o.coff + C].double()
        bad = ~((got - shuf(ref)).abs() <= shuf(tol))
        desc = 'launch %d: conv_tc_ps cin %d -> 4 x %d' % (len(shadow['calls']), inp_v.c, C)
        shadow['calls'].append(desc)
        assert not bool(bad.any()), '%s: %d elements outside the bound' % (desc, int(bad.sum()))
    monkeypatch.setattr(ops, 'conv_tc_ps', conv_tc_ps)
    return shadow


@pytest.mark.parametrize('prec', ['bf16', 'fp16'])
@pytest.mark.parametrize('nf', [32, 64, 128])
def test_shadow_srresnet_inference(shadow_ps, prec, nf):
    """nf 128: two Cout tiles per output parity of the pixel-shuffle conv"""
    net = _srresnet(2, nf=nf).cuda().eval()
    net.precision = prec
    with torch.no_grad():
        net(O.synth_image((2, 3, 37, 26), 91).cuda())
    assert sum('conv_tc_ps' in c for c in shadow_ps['calls']) == 2


@pytest.mark.parametrize('nf', [32, 64, 128])
def test_shadow_srresnet_mixed_precision_training(shadow_ps, nf):
    net = _srresnet(2, nf=nf, res_scale=0.5).cuda()
    net.train_precision = 'bf16'
    out = net(O.synth_image((2, 3, 21, 18), 92).cuda())
    (out * O.synth(tuple(out.shape), 93).cuda()).sum().backward()
    assert any('mask=True' in c for c in shadow_ps['calls'])


# ------------------------------------------------------------------------------------------------------------------------
# module level
# ------------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('prec', ['bf16', 'fp16'])
def test_f1_srresnet_fixture_16bit(golden, prec):
    """the reference's SRResNet (nb 2, nf 64, x4, pixel shuffle) output in eval mode, bound R u with R = 19"""
    from dasr_b200.srn.models.modules.architecture import SRResNet
    from tests.test_gpu_f1 import synth_sd
    g = golden('f1_modules.pt')['srresnet']
    net = SRResNet(3, 3, 64, 2, upscale=4, norm_type=None, act_type='relu', mode='CNA', upsample_mode='pixelshuffle')
    net.load_state_dict(synth_sd(net, g['w_seed']), strict=False)
    net.cuda().eval()
    net.precision = prec
    x = O.synth_image(g['x_shape'], g['x_seed']).cuda()
    with torch.no_grad():
        out = net(x)
        out2 = net(x)               # the CUDA-graph replay of the same shape
    e = rel_linf(out, g['out'])
    bound = fwd_roundings(2) * U[prec]
    print('f1 srresnet %s: rel-Linf %.3e vs the reference fixture (bound %.3e)' % (prec, e, bound))
    assert e <= bound
    assert torch.equal(out, out2)


@pytest.mark.parametrize('prec', ['bf16', 'fp16'])
def test_srresnet16_against_the_fp32_layer_list(prec):
    """SRResNet-16 (nf 64, x4) on 4 x 3 x 64 x 64, bound R u with R = 47"""
    net = _srresnet(16, seed=83).cuda().eval()
    x = O.synth_image((4, 3, 64, 64), 84).cuda()
    with torch.no_grad():
        net.precision = 'fp32'
        ref = net(x)
        net.precision = prec
        out = net(x)
    e = rel_linf(out, ref)
    bound = fwd_roundings(16) * U[prec]
    print('SRResNet-16 %s vs fp32: rel-Linf %.3e, rel-L2 %.3e (bound %.3e)' % (prec, e, rel_l2(out, ref), bound))
    assert e <= bound


def test_environment_leaves_uncovered_nf_on_the_layer_list(monkeypatch):
    """nf 96 has no wgmma plan: chosen by the environment, 16-bit modes keep the fp32 layer list (bit for bit)"""
    from dasr_b200.srn.models.modules.sr_nets import _Compiled
    monkeypatch.setenv('DASR_B200_PRECISION', 'bf16')
    monkeypatch.setenv('DASR_B200_TRAIN_PRECISION', 'bf16')
    net = _srresnet(1, nf=96).cuda()
    x = O.synth_image((1, 3, 11, 13), 86).cuda()
    with torch.no_grad():
        want = _Compiled.forward(net.eval(), x)
        got = net(x)
    assert torch.equal(_bits(got), _bits(want))
    net.train()(x).sum().backward()              # the fp32 layer list's training node, not the bf16 one
    assert all(p.grad is not None for p in net.parameters())


def test_fp32_and_default_are_the_layer_list(monkeypatch):
    """precision 'fp32', and no precision anywhere, run the fp32 layer list unchanged (bit for bit)"""
    from dasr_b200.srn.models.modules.sr_nets import _Compiled
    monkeypatch.delenv('DASR_B200_PRECISION', raising=False)
    net = _srresnet(2).cuda().eval()
    x = O.synth_image((2, 3, 19, 23), 85).cuda()
    with torch.no_grad():
        want = _Compiled.forward(net, x)
        default = net(x)
        net.precision = 'fp32'
        fp32 = net(x)
    assert torch.equal(_bits(default), _bits(want)) and torch.equal(_bits(fp32), _bits(want))


def _sr_model(nb, train_precision, sd):
    from helpers import make_opt, unwrap
    from dasr_b200.srn.models import create_model
    opt = make_opt(True, 'sr', nb=nb)
    opt['network_G']['which_model_G'] = 'sr_resnet'
    m = create_model(opt)
    unwrap(m.netG).load_state_dict(sd)
    unwrap(m.netG).train_precision = train_precision
    return m


def test_sr_model_mixed_precision_steps_against_fp32(monkeypatch):
    """two SRModel steps (sr_resnet nb 2, L1 loss, Adam) in bf16 and in fp32 from the same weights.
    l_pix: |dl| <= R u max|out| (the forward bound, R = 19).  Filter / bias gradients of the first step: rel-L2 <= R' u
    with R' = 3 R (each conv adds its filter, output-gradient and saved-activation roundings on the backward path)."""
    monkeypatch.delenv('DASR_B200_TRAIN_PRECISION', raising=False)
    nb = 2
    sd = _srresnet(nb, seed=86).state_dict()
    data = {'LR': O.synth_image((4, 3, 16, 16), 87), 'HR': O.synth_image((4, 3, 64, 64), 88)}
    runs = {}
    for tp in ('fp32', 'bf16'):
        m = _sr_model(nb, tp, sd)
        losses, grads = [], None
        for step in range(2):
            m.feed_data(data)
            m.optimize_parameters(step)
            losses.append(m.log_dict['l_pix'])
            if step == 0:
                grads = [(k, p.grad.detach().clone()) for k, p in m.netG.named_parameters()]
                out_max = float(m.fake_H.detach().abs().max())
        runs[tp] = (losses, grads, out_max)
        del m
    (l32, g32, omax), (l16, g16, _) = runs['fp32'], runs['bf16']
    R = fwd_roundings(nb)
    worst = max(rel_l2(a, b) for (_, a), (_, b) in zip(g16, g32))
    print('SRModel steps: l_pix fp32 %s bf16 %s, worst gradient rel-L2 %.3e (bound %.3e)' % (l32, l16, worst, 3 * R * U['bf16']))
    for a, b in zip(l16, l32):
        assert abs(a - b) <= R * U['bf16'] * omax
    assert worst <= 3 * R * U['bf16']


def _module_step(sd, nb, x, pattern, graph, monkeypatch):
    from dasr_b200.srn.models.modules.sr_nets import SRResNet
    monkeypatch.setenv('DASR_B200_GRAPH', '1' if graph else '0')
    net = SRResNet(3, 3, 64, nb, upscale=4, norm_type=None, act_type='relu', mode='CNA', res_scale=0.5,
                   upsample_mode='pixelshuffle')
    net.load_state_dict(sd)
    net.cuda()
    net.train_precision = 'bf16'
    res = None
    for _ in range(3):                  # graphs: captured at the second sighting, replayed at the third
        net.zero_grad()
        out = net(x)
        (out * pattern).sum().backward()
        torch.cuda.synchronize()
        res = [('out', out.detach().clone())] + [(n, p.grad.detach().clone()) for n, p in net.named_parameters()]
    if graph:
        assert net._train_graphs, 'the CUDA-graph training path was not taken'
    return res


def test_graph_training_step_is_bit_identical_to_eager(monkeypatch):
    from tests.test_engine_float64 import _bit_diff
    nb = 2
    sd = _srresnet(nb, res_scale=0.5, seed=89).state_dict()
    x = O.synth_image((2, 3, 19, 14), 90).cuda()
    pattern = O.synth((2, 3, 76, 56), 94).cuda()
    eager = _module_step(sd, nb, x, pattern, False, monkeypatch)
    graph = _module_step(sd, nb, x, pattern, True, monkeypatch)
    assert _bit_diff(eager, graph) is None, 'eager vs CUDA graph: ' + str(_bit_diff(eager, graph))


def test_bf16_training_refuses_the_input_gradient():
    from dasr_b200 import _lib
    net = _srresnet(1).cuda()
    net.train_precision = 'bf16'
    with pytest.raises(_lib.DasrError):
        net(O.synth_image((1, 3, 8, 8), 95).cuda().requires_grad_(True))


def test_gpu_training_plan_equals_the_float64_plan(monkeypatch):
    """the ops calls of a real eager mixed-precision step are the ones the float64 check ran"""
    from dasr_b200 import engine, ops
    from tests import test_engine_float64 as E
    from tests import test_srresnet_float64 as S
    for name in S.NEW:
        monkeypatch.setitem(E.BACKEND, name, S.NEW[name][0])
        monkeypatch.setitem(E.SIGS, name, inspect.signature(getattr(ops, name)))
        monkeypatch.setitem(E.WRITES, name, S.NEW[name][1])
    monkeypatch.setitem(E.BACKEND, 'pack_filter_tc', S.pack_filter_tc)
    be = E.Backend()
    with pytest.MonkeyPatch.context() as mp:
        E.install(mp, be)
        for name in S.NEW:
            mp.setattr(ops, name, lambda *a, _n=name, **kw: be.launch(_n, a, kw))
        S.run_train(2, 64, 4, 0.5)
    net = S._srresnet(2, 64, 4, 71 + 2, 0.5).cuda()
    ps = [p.detach().clone().requires_grad_(True) for p in net.parameters()]
    x = E._x(72, (S.N, 3, S.H, S.W)).cuda()
    pattern = O.synth((S.N, 3, 4 * S.H, 4 * S.W), 73).cuda()

    def step():
        out = engine.SRResNetFunctionBF16.apply(x, 2, 4, 0.5, engine._PackCache(), None, *ps)
        (out * pattern).sum().backward()
    gpu = E.record_gpu_plan(step)
    for i, (a, b) in enumerate(zip(gpu, be.plan)):
        assert a == b, 'call %d differs:\n  gpu %s\n  f64 %s' % (i, a, b)
    assert len(gpu) == len(be.plan), (len(gpu), len(be.plan))
