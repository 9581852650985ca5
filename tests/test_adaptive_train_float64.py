"""Training of the adaptive-weight RRDB generators, checked in float64 against autograd of the oracle.

The float64 backend of test_engine_float64.py (every ops launch wrapper replaced by the float64 value of its contract) is
extended with the models of the three wrappers the adaptive backward adds (csrc/map_bwd.cu):
  * map_channel_dgrad: the gradient of a MAP_CHANNEL conv's map input channel, s * sum over taps and output channels of
    the map taps times the output gradient at the pixel the tap reaches (torch's padded shifts);
  * map_channel_wgrad: the filter gradient of that channel, s * sum over pixels of the output gradient times the shifted map;
  * map_scale_bwd: gt = map * g and the per-pixel sum of g * t.
map_axpby's bf16 form (the plain variant's a * t3 + 0.1 R in the mixed-precision forward) is the existing fp32 model: the
backend does not round.  The fp32 node (AdaptiveRRDBFunction) and the bf16 node (AdaptiveRRDBFunctionBF16) must equal
float64 autograd of oracle.adaptive_oracle.adaptive_rrdb_forward to 1e-9 of the largest value of each tensor (the concat
variant: 2^-20, fp32(0.2) != 0.2 in the MAP_CHANNEL epilogue): the output, every parameter gradient, the map gradient and,
for fp32, the input-image gradient.  The side-stream reductions are checked for ordering as in test_engine_float64.py.
Deliberately wrong wirings must fail that bound."""
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
from dasr_b200.ops import View  # noqa: E402
from oracle import adaptive_oracle as AO  # noqa: E402
from oracle import srn_oracle as O  # noqa: E402
from tests import test_engine_float64 as E  # noqa: E402
from tests.test_engine_float64 import TOL, TOL_MAP_CHANNEL, backend  # noqa: E402,F401  (backend: the pytest fixture)

F64 = torch.float64
N, H, W = 2, 13, 11


def _shifted(t, dy, dx):
    """t [N, C, H, W] read at (y + dy, x + dx), zero outside the image"""
    h, w = t.shape[-2:]
    return F.pad(t, (1, 1, 1, 1))[..., 1 + dy:1 + dy + h, 1 + dx:1 + dx + w]


def _store(ga, v, accumulate):
    d = ga.view(v.shape)
    d.copy_(v + d.double() if accumulate else v)


def map_channel_dgrad(g, w_map, s, ga, accumulate=False):
    G = E._get(g).permute(0, 3, 1, 2)                        # [N, C, H, W]
    wm = w_map.double()
    v = sum((_shifted(G, 1 - t // 3, 1 - t % 3) * wm[t].view(1, -1, 1, 1)).sum(1) for t in range(9))
    _store(ga, s * v, accumulate)


def map_channel_wgrad(g, amap, s, dw, ch, accumulate=False):
    G = E._get(g).permute(0, 3, 1, 2)
    A = amap.double().reshape(G.shape[0], 1, G.shape[2], G.shape[3])
    v = torch.stack([(G * _shifted(A, t // 3 - 1, t % 3 - 1)).sum((0, 2, 3)) for t in range(9)], 1)     # [C][9]
    d = dw[:, ch].view(G.shape[1], 9)
    d.copy_(s * v + d if accumulate else s * v)


def map_scale_bwd(g, t, amap, gt, ga, accumulate=False):
    G = E._get(g)
    if gt is not None:
        E._put(gt, amap.double().reshape(G.shape[:-1] + (1,)) * G)
    if ga is not None:
        _store(ga, (G * E._get(t, G.shape[-1])).sum(-1), accumulate)


NEW = {'map_channel_dgrad': (map_channel_dgrad, ('ga',)), 'map_channel_wgrad': (map_channel_wgrad, ('dw',)),
       'map_scale_bwd': (map_scale_bwd, ('gt', 'ga'))}


@pytest.fixture
def be(backend, monkeypatch):
    """the float64 backend with the adaptive backward's wrappers"""
    for name, (fn, writes) in NEW.items():
        monkeypatch.setitem(E.BACKEND, name, fn)
        monkeypatch.setitem(E.SIGS, name, inspect.signature(getattr(ops, name)))
        monkeypatch.setitem(E.WRITES, name, writes)
        monkeypatch.setattr(ops, name, lambda *a, _n=name, **kw: backend.launch(_n, a, kw))
    return backend


def test_models_take_the_wrappers_arguments():
    for name, (fn, _) in NEW.items():
        assert list(inspect.signature(fn).parameters) == list(inspect.signature(getattr(ops, name)).parameters), name


def _conv65(inp, a, s, w):
    """float64 3x3 conv of [inp | s * a] (NCHW) with the 65-channel filter w, no bias"""
    return F.conv2d(torch.cat([inp, s * a], 1), w, padding=1)


def test_models_are_autograd_of_their_formulas():
    """each model equals float64 autograd of the formula it restates: the map channel of a 65-channel conv, and the map
    product out = a * t"""
    g = torch.Generator().manual_seed(3)
    rnd = lambda *s: torch.rand(s, generator=g, dtype=F64) * 2 - 1
    C, s = 40, 0.2
    x, a, w, go = rnd(2, 64, 7, 5), rnd(2, 1, 7, 5).requires_grad_(True), rnd(C, 65, 3, 3).float().double().requires_grad_(True), rnd(2, C, 7, 5)
    ga, gw = torch.autograd.grad((_conv65(x, a, s, w) * go).sum(), [a, w])
    gbuf = torch.zeros(2, 7, 5, C + 8, dtype=F64)
    gbuf[..., 8:] = go.permute(0, 2, 3, 1)
    got = torch.full((2, 1, 7, 5), 0.5, dtype=F64)
    map_channel_dgrad(View(gbuf, C, 8), ops.map_channel_taps(w, 64).double(), s, got, accumulate=True)
    assert torch.allclose(got - 0.5, ga, rtol=0, atol=1e-13)
    dw = torch.ones(C, 65, 3, 3, dtype=F64)
    map_channel_wgrad(View(gbuf, C, 8), a.detach(), s, dw, 64)
    assert torch.allclose(dw[:, 64], gw[:, 64], rtol=0, atol=1e-13) and bool((dw[:, :64] == 1).all())
    t = rnd(2, 7, 5, C).requires_grad_(True)
    am = rnd(2, 1, 7, 5).requires_grad_(True)
    out = am.permute(0, 2, 3, 1) * t
    gt_ref, ga_ref = torch.autograd.grad((out * gbuf[..., 8:]).sum(), [t, am])
    gt, gam = torch.zeros(2, 7, 5, C, dtype=F64), torch.zeros(2, 1, 7, 5, dtype=F64)
    map_scale_bwd(View(gbuf, C, 8), t.detach(), am.detach(), gt, gam)
    assert torch.allclose(gt, gt_ref, rtol=0, atol=1e-13) and torch.allclose(gam, ga_ref, rtol=0, atol=1e-13)


def _generator(concat, nb, nb_ada, seed):
    from dasr_b200.srn.models.modules import architecture as A
    sd = AO.synth_adaptive_g(nb, nb_ada, concat, seed, 0.5)
    cls = A.RRDBNet_Residual_conv_concat if concat else A.RRDBNet_Residual_conv
    net = cls(3, 3, 64, nb, gc=32, upscale=4, nb_ada=nb_ada)
    net.load_state_dict(sd)
    return sd, [p.detach() for p in net._engine_params()], E._names(net, net._engine_params())


def run(prec, concat, nb, nb_ada, need_map=True, shape=(N, 3, H, W)):
    """one training step of the fp32 or bf16 node on float64 parameters / map with fp32 values (the node's casts are exact),
    against float64 autograd of the oracle"""
    seed = 81 + 2 * nb + nb_ada + (10 if concat else 0)
    sd, params, names = _generator(concat, nb, nb_ada, seed)
    ps = [p.double().requires_grad_(True) for p in params]
    x = E._x(seed + 1, shape)
    amap = E._x(seed + 2, (shape[0], 1) + shape[2:]).double().requires_grad_(need_map)
    pattern = O.synth((shape[0], 3, 4 * shape[2], 4 * shape[3]), seed + 3)
    if prec == 'fp32':
        xg = x.double().requires_grad_(True)
        out = engine.AdaptiveRRDBFunction.apply(xg, amap, nb, nb_ada, concat, 4, *ps)
    else:
        out = engine.AdaptiveRRDBFunctionBF16.apply(x, amap, nb, nb_ada, concat, 4, engine._PackCache(), *ps)
    (out * pattern.to(out.dtype)).sum().backward()
    s64 = E._sd64(sd)
    x64, a64 = x.double().requires_grad_(True), amap.detach().clone().requires_grad_(True)
    ref = AO.adaptive_rrdb_forward(x64, a64, s64, nb, nb_ada, concat)
    grads = torch.autograd.grad((ref * pattern.double()).sum(), [s64[n] for n in names] + [a64, x64])
    pairs = [('out', out.detach(), ref.detach())] + [(n, p.grad, gr) for n, p, gr in zip(names, ps, grads)]
    if need_map:
        assert amap.grad.shape == amap.shape and amap.grad.dtype == amap.dtype
        pairs.append(('map', amap.grad, grads[-2]))
    else:
        assert amap.grad is None
    if prec == 'fp32':
        pairs.append(('dx', xg.grad, grads[-1]))
    return pairs


CASES = [('concat', 2, 2), ('plain', 1, 1), ('plain', 2, 1)]


@pytest.mark.parametrize('need_map', [True, False], ids=['map-grad', 'no-map-grad'])
@pytest.mark.parametrize('variant,nb,nb_ada', CASES, ids=['%s-nb%d-ada%d' % c for c in CASES])
@pytest.mark.parametrize('prec', ['fp32', 'bf16'])
def test_adaptive_training_float64(be, monkeypatch, prec, variant, nb, nb_ada, need_map):
    monkeypatch.setenv('DASR_B200_BWD_OVERLAP', '1')
    monkeypatch.setenv('DASR_B200_FUSE_MASK', '0')
    t0 = time.time()
    concat = variant == 'concat'
    pairs = run(prec, concat, nb, nb_ada, need_map)
    E._report('adaptive %s %s nb=%d ada=%d' % (prec, variant, nb, nb_ada), be, pairs, t0, TOL_MAP_CHANNEL if concat else TOL)
    used = {p[0] for p in be.plan}
    if prec == 'bf16':
        assert len(be.streams.all) > 1, 'the dense-block reductions did not run on the side stream'
        want = ({'map_channel_dgrad', 'map_channel_wgrad'} if concat else {'map_scale_bwd', 'map_axpby'}) if need_map else set()
        assert want <= used, used
        if not need_map:
            assert 'map_channel_dgrad' not in used
            assert not any(e[0] == 'map_scale_bwd' and e[2].get('ga') is not None for e in be.plan)


# ------------------------------------------------------------------------------------------------------------------------
# the reference's gradients (tests/golden/adaptive_grads.pt)
# ------------------------------------------------------------------------------------------------------------------------

def sample_idx(n, samples):
    """the flat indices at which the fixture keeps a filter gradient of n values (oracle/gen_golden_adaptive_grads.py)"""
    return torch.linspace(0, n - 1, min(n, samples), dtype=F64).round().long()


def fixture_pairs(g, out, named_grads, gmap, dx, samples=512):
    """[(label, got, ref)] of one generator's results against its fixture record g: filter gradients at the fixture's
    sampled indices, as L2 norms and, for the 65-channel filters, their map-channel slices; everything else whole"""
    pairs = [('out', out, g['out']), ('map', gmap, g['map_grad']), ('dx', dx, g['x_grad'])]
    for k, gr in named_grads:
        ref = g['grads'][k]
        if 'full' in ref:
            pairs.append((k, gr, ref['full']))
            continue
        pairs.append((k + '[samples]', gr.reshape(-1)[sample_idx(gr.numel(), samples).to(gr.device)], ref['values']))
        pairs.append((k + '[norm]', gr.double().norm().reshape(1), torch.tensor([ref['norm']], dtype=F64)))
        if 'map_channel' in ref:
            pairs.append((k + '[map channel]', gr[:, 64], ref['map_channel']))
    return pairs


@pytest.mark.parametrize('variant', ['concat', 'plain'])
def test_oracle_gradients_match_the_reference(golden, variant):
    """autograd of oracle.adaptive_oracle.adaptive_rrdb_forward (CPU, fp32) gives the reference's output and gradients to
    1e-5 relative (max|got - ref| / max|ref| per tensor)"""
    rec = golden('adaptive_grads.pt')
    g = rec[variant]
    concat = variant == 'concat'
    n, c, h, w = rec['shape']
    sd = {k: v.clone().requires_grad_(True) for k, v in AO.synth_adaptive_g(g['nb'], g['nb_ada'], concat, g['w_seed'],
                                                                            rec['gain']).items()}
    x = O.synth_image(rec['shape'], rec['x_seed']).requires_grad_(True)
    a = O.synth_image((n, 1, h, w), rec['map_seed']).requires_grad_(True)
    out = AO.adaptive_rrdb_forward(x, a, sd, g['nb'], g['nb_ada'], concat)
    (out * O.synth(tuple(out.shape), rec['pattern_seed'])).sum().backward()
    assert list(sd) == list(g['grads'])
    pairs = fixture_pairs(g, out.detach(), [(k, v.grad) for k, v in sd.items()], a.grad, x.grad, rec['samples'])
    worst = max((float((p.double() - r.double()).abs().max() / r.double().abs().max()), k) for k, p, r in pairs)
    print('%s: worst %.3g (%s)' % (variant, *worst))
    assert worst[0] <= 1e-5, worst


# ------------------------------------------------------------------------------------------------------------------------
# the check can fail
# ------------------------------------------------------------------------------------------------------------------------

def _map_term_dropped(i, name, a):
    if name == 'map_channel_dgrad':
        a['s'] = 0.0
        return True
    if name == 'map_scale_bwd' and a.get('ga') is not None:
        a['ga'] = None
        return True
    return False


def _r_map_scale_02(i, name, a):
    """every use of R's map channel (scale 1) gets A's scale 0.2"""
    if name == 'conv_tc' and a.get('amap') is not None and a.get('map_scale') == 1.0:
        a['map_scale'] = 0.2
        return True
    if name in ('map_channel_dgrad', 'map_channel_wgrad') and a['s'] == 1.0:
        a['s'] = 0.2
        return True
    return False


def _a_not_accumulated(i, name, a):
    if name in ('conv3x3_wgrad_tc', 'map_channel_wgrad', 'bias_grad') and a.get('accumulate'):
        a['accumulate'] = False
        return True
    return False


def _identity_skip(monkeypatch):
    """the backward of an adaptive block treated as if the block had RRDB's identity skip: its input gradient gets the
    block's output gradient added"""
    enter, leave = engine._AdaptiveBackward.enter, engine._AdaptiveBackward.leave

    def enter2(self, r, g, grads):
        if r % 3 == 2:
            v = ops.as_view(g)
            self.skip = View(v.t.clone(), v.c, v.coff)
        return enter(self, r, g, grads)

    def leave2(self, r, g, grads):
        g = leave(self, r, g, grads)
        if r % 3 == 0:
            out = self._new()
            ops.axpby(g, 1.0, self.skip, 1.0, out)
            return out
        return g
    monkeypatch.setattr(engine._AdaptiveBackward, 'enter', enter2)
    monkeypatch.setattr(engine._AdaptiveBackward, 'leave', leave2)


MUTATIONS = {'map_term_dropped': _map_term_dropped, 'r_map_scale_02': _r_map_scale_02,
             'a_grad_not_accumulated': _a_not_accumulated, 'identity_skip': None}


@pytest.mark.parametrize('variant', ['concat', 'plain'])
@pytest.mark.parametrize('mutation', sorted(MUTATIONS))
def test_wrong_wiring_is_caught(be, monkeypatch, mutation, variant):
    if variant == 'plain' and mutation in ('r_map_scale_02', 'a_grad_not_accumulated'):
        pytest.skip('the plain variant has no A and no map channel')
    if MUTATIONS[mutation] is None:
        _identity_skip(monkeypatch)
    else:
        be.mutate = MUTATIONS[mutation]
    concat = variant == 'concat'
    pairs = run('bf16', concat, 1, 1)
    assert MUTATIONS[mutation] is None or be.mutated > 0, 'the mutation found no launch to change'
    worst, where = E.compare(pairs)
    print('%s %s: worst error / max|ref| %.3g (%s)' % (mutation, variant, worst, where))
    assert worst > 1e3 * (TOL_MAP_CHANNEL if concat else TOL), '%s went unnoticed (worst %.3g at %s)' % (mutation, worst, where)


# ------------------------------------------------------------------------------------------------------------------------
# the module's dispatch
# ------------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('tp,env,node', [(None, None, 'AdaptiveRRDBFunction'), (None, 'bf16', 'AdaptiveRRDBFunctionBF16'),
                                         ('fp32', 'bf16', 'AdaptiveRRDBFunction'), ('bf16', None, 'AdaptiveRRDBFunctionBF16')])
def test_module_dispatches_on_train_precision(monkeypatch, tp, env, node):
    """grad-enabled CUDA calls go to the node train_precision (None: DASR_B200_TRAIN_PRECISION, else fp32) names; the
    node is stubbed, the tensors pose as CUDA tensors"""
    from dasr_b200.srn.models.modules import architecture as A
    if env is None:
        monkeypatch.delenv('DASR_B200_TRAIN_PRECISION', raising=False)
    else:
        monkeypatch.setenv('DASR_B200_TRAIN_PRECISION', env)
    seen = []
    for name in ('AdaptiveRRDBFunction', 'AdaptiveRRDBFunctionBF16'):
        monkeypatch.setattr(engine, name, type(name, (), {'apply': staticmethod(lambda *a, _n=name: seen.append((_n, a)))}))
    monkeypatch.setattr(torch.Tensor, 'is_cuda', property(lambda self: True))
    net = A.RRDBNet_Residual_conv(3, 3, 64, 1, nb_ada=1)
    net.train_precision = tp
    x, a = torch.zeros(1, 3, 8, 8), torch.zeros(1, 1, 8, 8)
    net(x, a)
    assert [s[0] for s in seen] == [node]
    assert seen[0][1][7 if node.endswith('BF16') else 6] is net._engine_params()[0]
