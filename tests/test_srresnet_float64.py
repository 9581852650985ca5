"""SRResNet on the wgmma kernels, checked in float64 against autograd of the reference network.

The float64 backend of test_engine_float64.py (every ops launch wrapper replaced by the float64 value of its contract) is
extended with the models of the two wrappers SRResNet adds:
  * conv_tc_ps: the 3x3 conv model (the packed filter decoded back to the conv's channel order) followed by a pixel
    shuffle, then the bias, activation and alpha the launch asks for, elementwise;
  * pixel_unshuffle_mask: a select of the gradient where the layer's output is positive, then a pixel unshuffle;
  * pack_filter_tc of kind TC_PS: kind 0's encoding of the filter with its rows in parity-major order.
The inference forward (bf16 and fp16 plans) and the mixed-precision training step (through SRResNetFunctionBF16) must
equal float64 autograd of helpers.native_forward (the module tree evaluated with torch's own operators) to 1e-9 of the
largest value of each tensor: the output, every filter gradient and every bias gradient.  Deliberately wrong wirings
(a dropped res_scale, a LeakyReLU mask slope in a ReLU network) must fail that bound."""
import copy
import inspect
import os
import sys
import time

import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from dasr_b200 import engine, ops  # noqa: E402
from oracle import srn_oracle as O  # noqa: E402
from tests import test_engine_float64 as E  # noqa: E402
from tests.helpers import native_forward  # noqa: E402
from tests.test_engine_float64 import TOL, backend  # noqa: E402,F401  (backend: the pytest fixture)
from tests.test_gpu_conv_tc_exact import _contract, _geometry, decode_filter  # noqa: E402

N, H, W = 2, 7, 9


def to_conv_order(rows, c):
    """parity-major rows (b * c + cc) -> the conv's channel order (4 cc + b), along dim 0"""
    return rows.reshape(4, c, *rows.shape[1:]).transpose(0, 1).reshape(4 * c, *rows.shape[1:])


def to_parity_major(rows, c):
    """the conv's channel order (4 cc + b) -> parity-major rows (b * c + cc), along dim 0"""
    return rows.reshape(c, 4, *rows.shape[1:]).transpose(0, 1).reshape(4 * c, *rows.shape[1:])


def encode_ps(w):
    """float64 pack of kind TC_PS: kind 0's layout of the filter with its rows in parity-major order"""
    return E.encode_filter_tc(to_parity_major(w.detach().double(), w.shape[0] // 4), ops.TC_FPROP)


def decode_ps(w_packed, k, c):
    """[9 taps][4c conv output channels][k]: the packed TC_PS filter in the conv's channel order"""
    return to_conv_order(decode_filter(w_packed, ops.TC_FPROP, k, 4 * c)[0].transpose(0, 1), c).transpose(0, 1)


def pack_filter_tc(w, kind, dtype=None):
    return encode_ps(w) if kind == ops.TC_PS else E.encode_filter_tc(w, kind)


def conv_tc_ps(inp, w_packed, bias, out, nt=None, act=ops.ACT_NONE, slope=0.2, alpha=1.0):
    o = ops.as_view(out)
    x = E._get(inp)
    acc = _contract(x, decode_ps(w_packed, x.shape[-1], o.c)[None], *_geometry(ops.TC_FPROP))   # [N, H, W, 4c]
    if bias is not None:
        acc = acc + bias.double()
    v = F.pixel_shuffle(acc.permute(0, 3, 1, 2), 2).permute(0, 2, 3, 1)
    if act == ops.ACT_RELU:
        v = torch.where(v < 0, torch.zeros_like(v), v)
    elif act == ops.ACT_LRELU:
        v = torch.where(v < 0, v * slope, v)
    E._put(o, v * alpha)


def pixel_unshuffle_mask(g_hr, y_hr, g_lr):
    g = g_hr.double()
    if y_hr is not None:
        g = torch.where(y_hr > 0, g, torch.zeros_like(g))
    g_lr.copy_(F.pixel_unshuffle(g.permute(0, 3, 1, 2), 2).permute(0, 2, 3, 1))


NEW = {'conv_tc_ps': (conv_tc_ps, ('out',)), 'pixel_unshuffle_mask': (pixel_unshuffle_mask, ('g_lr',))}


@pytest.fixture
def be(backend, monkeypatch):
    """the float64 backend with the SRResNet wrappers"""
    for name, (fn, writes) in NEW.items():
        monkeypatch.setitem(E.BACKEND, name, fn)
        monkeypatch.setitem(E.SIGS, name, inspect.signature(getattr(ops, name)))
        monkeypatch.setitem(E.WRITES, name, writes)
        monkeypatch.setattr(ops, name, lambda *a, _n=name, **kw: backend.launch(_n, a, kw))
    monkeypatch.setitem(E.BACKEND, 'pack_filter_tc', pack_filter_tc)
    return backend


def test_models_take_the_wrappers_arguments():
    for name, (fn, _) in NEW.items():
        assert list(inspect.signature(fn).parameters) == list(inspect.signature(getattr(ops, name)).parameters), name


def test_ps_pack_round_trip():
    """encode -> decode of the TC_PS layout gives the filter back; packed row b * c + cc holds conv channel 4 cc + b"""
    c, cin = 16, 64
    w = O.synth((4 * c, cin, 3, 3), 5).double()
    packed = encode_ps(w)
    assert packed.numel() == E._real_lib().dasr_pack_filter_tc_bytes(4 * c, cin, ops.TC_PS) // 2
    back = decode_ps(packed, cin, c)                                   # [tap][4c][cin]
    assert torch.equal(back.permute(1, 2, 0).reshape(4 * c, cin, 3, 3), w)
    rows = decode_filter(packed, ops.TC_FPROP, cin, 4 * c)[0]          # [tap][packed row][cin]
    assert torch.equal(rows[:, 1 * c + 3], w[4 * 3 + 1].reshape(cin, 9).t())


def _srresnet(nb, nf, upscale, seed, res_scale):
    from dasr_b200.srn.models.modules.sr_nets import SRResNet
    net = SRResNet(3, 3, nf, nb, upscale=upscale, norm_type=None, act_type='relu', mode='CNA', res_scale=res_scale,
                   upsample_mode='pixelshuffle')
    sd = net.state_dict()
    for i, (k, v) in enumerate(sd.items()):
        fan_in = v[0].numel()
        sd[k] = O.synth(tuple(v.shape), seed * 1000 + i, (6.0 / fan_in) ** 0.5 if v.dim() == 4 else 0.1)
    net.load_state_dict(sd)
    return net


def _truth(net, x, pattern=None):
    n64 = copy.deepcopy(net).double()
    out = native_forward(n64, x.double())
    if pattern is None:
        return out.detach(), None
    (out * pattern.double()).sum().backward()
    return out.detach(), [(k, p.grad) for k, p in n64.named_parameters()]


def run_inference(nb, nf, upscale, half, res_scale):
    net = _srresnet(nb, nf, upscale, 61 + nb, res_scale)
    params = [p.detach() for p in net.parameters()]
    x = E._x(62, (N, 3, H, W))
    with torch.no_grad():
        out = engine.srresnet_forward_bf16(x, params, nb, upscale, None, half=half, res_scale=res_scale)
    ref, _ = _truth(net, x)
    return [('out', out, ref)]


def run_train(nb, nf, upscale, res_scale):
    """one mixed-precision step through SRResNetFunctionBF16 (eager); float64 parameters with fp32 values, so the node's
    fp32 casts are exact and its gradients are not rounded on the way out"""
    net = _srresnet(nb, nf, upscale, 71 + nb, res_scale)
    names = [k for k, _ in net.named_parameters()]
    ps = [p.detach().double().requires_grad_(True) for p in net.parameters()]
    x = E._x(72, (N, 3, H, W))
    pattern = O.synth((N, 3, upscale * H, upscale * W), 73)
    out = engine.SRResNetFunctionBF16.apply(x, nb, upscale, res_scale, engine._PackCache(), None, *ps)
    (out * pattern.to(out.dtype)).sum().backward()
    ref, grads = _truth(net, x, pattern)
    return [('out', out.detach(), ref)] + [(k, p.grad, g) for (k, g), p in zip(grads, ps)]


@pytest.mark.parametrize('upscale', [2, 4])
@pytest.mark.parametrize('prec', ['bf16', 'fp16'])
def test_srresnet_inference_float64(be, prec, upscale):
    t0 = time.time()
    E._report('srresnet %s x%d' % (prec, upscale), be, run_inference(2, 64, upscale, prec == 'fp16', 0.5), t0)


@pytest.mark.parametrize('upscale,nf,res_scale', [(4, 64, 1.0), (2, 32, 0.5)])
def test_srresnet_train_float64(be, upscale, nf, res_scale):
    t0 = time.time()
    E._report('srresnet train x%d nf %d' % (upscale, nf), be, run_train(2, nf, upscale, res_scale), t0)
    ops_used = {p[0] for p in be.plan}
    assert {'conv_tc_ps', 'pixel_unshuffle_mask', 'conv3x3_wgrad_tc', 'bias_grad'} <= ops_used, ops_used


def _drop_res_scale(i, name, a):
    if name == 'conv_tc' and a.get('res1') is not None and a.get('alpha', 1.0) != 1.0:
        a['alpha'] = 1.0
        return True
    return False


def _lrelu_mask(i, name, a):
    if name == 'conv_tc' and a.get('mask') is not None:
        a['mask_slope'] = 0.2
        return True
    return False


@pytest.mark.parametrize('mutation', ['dropped_res_scale', 'lrelu_mask_slope'])
def test_wrong_wiring_is_caught(be, mutation):
    be.mutate = {'dropped_res_scale': _drop_res_scale, 'lrelu_mask_slope': _lrelu_mask}[mutation]
    pairs = run_train(1, 32, 2, 0.5)
    assert be.mutated > 0, 'the mutation found no launch to change'
    worst, where = E.compare(pairs)
    assert worst > 1e3 * TOL, '%s went unnoticed (worst %.3g at %s)' % (mutation, worst, where)
