"""The state the generator modules keep between calls: the inference CUDA graphs (_GraphedForward), the training graphs
(_TrainGraphs and the raw parameter addresses of their batch packer), the kernel-layout filter caches (_PackCache) and
the gradient arena of RRDBNet.set_grad_arena.

GPU: every case runs twice on fresh modules built from the same weights, once with CUDA graphs and once eagerly
(DASR_B200_GRAPH=0).  A replay issues the launch sequence of the eager run, so outputs, every .grad and the parameters
after the updates must agree bit for bit; each graph case also counts CUDAGraph.replay calls, so a path that quietly fell
back to eager would fail.  Training cases: RRDBNet nb 1 (graphs captured on the first call of a shape) and SRResNet nb 2
(on the second), 2x3x13x11 inputs, pattern-weighted sums as losses.

CPU: the float64 backend of test_engine_float64.py runs RRDBNetFunctionBF16 eagerly with a gradient arena; .grad, which
the optimizer reads, is compared with float64 autograd of the reference network."""
import pytest
import torch
import torch.nn as nn

from dasr_b200 import _lib, dp, engine
from dasr_b200.srn.models.modules import architecture as A
from oracle import adaptive_oracle as AO
from oracle import srn_oracle as O
from tests import test_engine_float64 as E

F64 = torch.float64
DasrError = _lib.DasrError
SHAPE = (2, 3, 13, 11)


# ------------------------------------------------------------------------------------------------------------------------
# CPU: the gradient arena, float64 backend
# ------------------------------------------------------------------------------------------------------------------------

@pytest.fixture
def backend(monkeypatch):
    be = E.Backend()
    E.install(monkeypatch, be)
    return be


def _arena_setup(seed):
    sd, params, names = E._rrdbnet(1, 64, seed, 0.5)
    ps = [p.detach().double().requires_grad_(True) for p in params]      # float64 .grad: no cast after the backward
    arena = torch.zeros(sum(p.numel() for p in ps), dtype=F64)
    return sd, ps, names, arena


def _node(x, ps, arena, cache):
    return engine.RRDBNetFunctionBF16.apply(x, 1, 4, cache, None, arena, *ps)


def _ref_grads(sd, names, terms):
    """float64 autograd of sum over (x, pattern, weight) of weight * (RRDBNet(x) * pattern).sum()"""
    s64 = E._sd64(sd)
    loss = sum(w * (O.rrdbnet_forward(x.double(), s64, 1) * p.double()).sum() for x, p, w in terms)
    return torch.autograd.grad(loss, [s64[n] for n in names])


def _check(label, ps, names, ref):
    worst, where = E.compare([(n, p.grad, r) for n, p, r in zip(names, ps, ref)])
    print('%s: worst .grad error / max|ref| %.3g (%s)' % (label, worst, where))
    assert worst <= E.TOL, '%s: .grad of %s differs from float64 autograd by %.3g of max|ref|' % (label, where, worst)


def _in_arena(t, arena):
    lo = arena.data_ptr()
    return lo <= t.data_ptr() and t.data_ptr() + t.numel() * t.element_size() <= lo + arena.numel() * arena.element_size()


def _pattern(seed):
    return O.synth((SHAPE[0], 3, 4 * SHAPE[2], 4 * SHAPE[3]), seed)


def test_arena_two_nodes_in_one_backward(backend):
    """two generator calls in one loss: each node's backward returns views of the same arena; the one that runs first
    must not hand autograd views that the second overwrites (that gives 2 g_a instead of g_a + g_b)"""
    sd, ps, names, arena = _arena_setup(401)
    x1, x2, p1, p2 = E._x(402), E._x(403), _pattern(404), _pattern(405)
    cache = engine._PackCache()
    o1, o2 = _node(x1, ps, arena, cache), _node(x2, ps, arena, cache)
    ((o1 * p1).sum() + (o2 * p2).sum()).backward()
    _check('two nodes, one backward', ps, names, _ref_grads(sd, names, [(x1, p1, 1), (x2, p2, 1)]))


def test_arena_two_accumulating_backwards(backend):
    """two backwards without zero_grad: the second must not overwrite the .grad views the first left in the arena"""
    sd, ps, names, arena = _arena_setup(411)
    x1, x2, p1, p2 = E._x(412), E._x(413), _pattern(414), _pattern(415)
    cache = engine._PackCache()
    (_node(x1, ps, arena, cache) * p1).sum().backward()
    assert all(_in_arena(p.grad, arena) for p in ps)
    (_node(x2, ps, arena, cache) * p2).sum().backward()
    _check('two accumulating backwards', ps, names, _ref_grads(sd, names, [(x1, p1, 1), (x2, p2, 1)]))


def test_arena_single_call_grads_are_arena_views(backend):
    """the data-parallel step: one call, every .grad equals float64 autograd and is a view inside the arena (zero-copy)"""
    sd, ps, names, arena = _arena_setup(421)
    x, p = E._x(422), _pattern(423)
    (_node(x, ps, arena, engine._PackCache()) * p).sum().backward()
    _check('single call', ps, names, _ref_grads(sd, names, [(x, p, 1)]))
    outside = [n for n, q in zip(names, ps) if not _in_arena(q.grad, arena)]
    assert not outside, '.grad not in the arena: %s' % outside[:4]


@pytest.mark.parametrize('with_arena', [False, True], ids=['fresh', 'arena'])
def test_retain_graph_backward_twice_float64(backend, with_arena):
    """backward twice through one eager node (retain_graph=True): its activations are kept for the second backward, and
    .grad is twice the gradient; a third backward, after the graph was freed, is refused"""
    sd, ps, names, arena = _arena_setup(431)
    x, p = E._x(432), _pattern(433)
    loss = (_node(x, ps, arena if with_arena else None, engine._PackCache()) * p).sum()
    loss.backward(retain_graph=True)
    loss.backward()
    _check('retain_graph x2', ps, names, _ref_grads(sd, names, [(x, p, 2)]))
    with pytest.raises(RuntimeError):
        loss.backward()


def test_broadcast_module_moves_versions(tmp_path):
    """dp.broadcast_module writes the parameters and floating buffers in place so that their version counters move and a
    cached kernel-layout filter is rebuilt (gloo, world_size 1, in process)"""
    import torch.distributed as dist
    net = nn.Sequential(nn.Conv2d(3, 8, 3), nn.BatchNorm2d(8), nn.Conv2d(8, 4, 3))
    cache, made = engine._PackCache(), []
    w = net[2].weight
    cache.get('w', w, lambda: made.append(1))
    dist.init_process_group('gloo', init_method='file://' + str(tmp_path / 'store'), rank=0, world_size=1)
    try:
        before = {n: t._version for n, t in list(net.named_parameters()) + list(net.named_buffers()) if t.is_floating_point()}
        values = {n: t.detach().clone() for n, t in net.state_dict().items()}
        dp.broadcast_module(net)
        after = {n: t._version for n, t in list(net.named_parameters()) + list(net.named_buffers()) if t.is_floating_point()}
    finally:
        dist.destroy_process_group()
    assert set(before) == set(after) and len(before) == 8
    stuck = [n for n in before if after[n] == before[n]]
    assert not stuck, 'version counter did not move: %s' % stuck
    for n, t in net.state_dict().items():
        assert torch.equal(t, values[n]), n
    cache.get('w', w, lambda: made.append(1))
    assert len(made) == 2, 'the packed filter was not rebuilt after the broadcast'


def _generators():
    from dasr_b200.srn.models.modules.sr_nets import SRResNet
    rrdb = A.RRDBNet(3, 3, 64, 1, gc=32, upscale=4)
    ada = A.RRDBNet_Residual_conv(3, 3, 64, 1, gc=32, upscale=4, nb_ada=1)
    srr = SRResNet(3, 3, 64, 2, upscale=4, norm_type=None, act_type='relu', mode='CNA', upsample_mode='pixelshuffle')
    return [('RRDBNet', rrdb, lambda: list(rrdb.parameters())), ('RRDBNet_Residual_conv', ada, ada._engine_params),
            ('SRResNet', srr, lambda: list(srr.parameters()))]


def _replacement(p, scale=1.0):
    """a new nn.Parameter holding p * scale, with p's version counter"""
    q = nn.Parameter(p.detach() * scale)
    with torch.no_grad():
        while q._version < p._version:
            q.mul_(1)
    assert q._version == p._version
    return q


def _owner(net, name):
    """(module, attribute) of the parameter called `name`"""
    mod, attr = net, name
    while '.' in attr:
        head, attr = attr.split('.', 1)
        mod = getattr(mod, head)
    return mod, attr


@pytest.mark.parametrize('versions', [False, True], ids=['train', 'inference'])
def test_graph_key_sees_every_parameter(versions):
    """replacing any single parameter by a new nn.Parameter (same values, same version counter) changes the graph key of
    each generator class, and putting the original back restores it; with versions, so does an in-place update of any
    single parameter"""
    x = torch.zeros(SHAPE)
    for cls, net, plist in _generators():
        k0 = A.graph_key(x, plist(), versions=versions)
        named = list(net.named_parameters())
        assert len(named) == len(plist())
        for name, p in named:
            mod, attr = _owner(net, name)
            setattr(mod, attr, _replacement(p))
            assert A.graph_key(x, plist(), versions=versions) != k0, '%s: replacing %s left the key unchanged' % (cls, name)
            setattr(mod, attr, p)
            assert A.graph_key(x, plist(), versions=versions) == k0
            if versions:
                with torch.no_grad():
                    p.add_(0)
                assert A.graph_key(x, plist(), versions=versions) != k0, '%s: updating %s left the key unchanged' % (cls, name)
                k0 = A.graph_key(x, plist(), versions=versions)


# ------------------------------------------------------------------------------------------------------------------------
# GPU: graph replays against eager runs, bit for bit
# ------------------------------------------------------------------------------------------------------------------------

def _bits(t):
    t = t.detach().contiguous()
    return t.view({4: torch.int32, 2: torch.int16, 8: torch.int64}[t.element_size()])


def _first_diff(a, b):
    assert [n for n, _ in a] == [n for n, _ in b], 'the two runs recorded different things'
    for (n, u), (_, v) in zip(a, b):
        if u.dtype != v.dtype or u.shape != v.shape:
            return '%s: %s %s vs %s %s' % (n, u.dtype, tuple(u.shape), v.dtype, tuple(v.shape))
        if not torch.equal(_bits(u), _bits(v)):
            return '%s: %d elements differ, max |diff| %.3g' % (n, int((u != v).sum()), float((u.float() - v.float()).abs().max()))
    return None


@pytest.fixture
def replays(monkeypatch):
    """number of CUDAGraph.replay calls so far"""
    n = [0]
    real = torch.cuda.CUDAGraph.replay

    def replay(self):
        n[0] += 1
        return real(self)
    monkeypatch.setattr(torch.cuda.CUDAGraph, 'replay', replay)
    return n


def _rrdbnet(seed=501):
    net = A.RRDBNet(3, 3, 64, 1, gc=32, upscale=4)
    net.load_state_dict(O.synth_state_dict(O.rrdbnet_shapes(nb=1), seed, 0.5))
    net.cuda()
    net.precision, net.train_precision = 'bf16', 'bf16'
    return net


def _srresnet(seed=511):
    from dasr_b200.srn.models.modules.sr_nets import SRResNet
    net = SRResNet(3, 3, 64, 2, upscale=4, norm_type=None, act_type='relu', mode='CNA', upsample_mode='pixelshuffle')
    net.load_state_dict({k: O.synth(tuple(v.shape), seed * 1000 + i, (6.0 / v[0].numel()) ** 0.5 if v.dim() == 4 else 0.05)
                         for i, (k, v) in enumerate(net.state_dict().items())})
    net.cuda()
    net.precision, net.train_precision = 'bf16', 'bf16'
    return net


def _adaptive(seed=521):
    net = A.RRDBNet_Residual_conv(3, 3, 64, 1, gc=32, upscale=4, nb_ada=1)
    net.load_state_dict(AO.synth_adaptive_g(1, 1, False, seed, 0.5))
    net.precision = 'bf16'
    return net.cuda()


NETS = {'rrdbnet': _rrdbnet, 'srresnet': _srresnet}


def _x(seed, shape=SHAPE):
    return O.synth_image(shape, seed).cuda()


def _pat(seed, shape=SHAPE):
    return O.synth((shape[0], 3, 4 * shape[2], 4 * shape[3]), seed).cuda()


def _grads(tag, net):
    return [('%s grad %s' % (tag, n), p.grad.detach().clone()) for n, p in net.named_parameters() if p.grad is not None]


def _params(net):
    return [('param %s' % n, p.detach().clone()) for n, p in net.named_parameters()]


def _sgd(net, lr=1e-3):
    """an in-place update of every parameter (versions move, addresses stay), then .grad = None"""
    with torch.no_grad():
        for p in net.parameters():
            if p.grad is not None:
                p.sub_(lr * p.grad)
                p.grad = None


def _both(monkeypatch, replays, make, scenario):
    """(eager record, graph record, replays of the graph run); scenario(net) -> list of (label, tensor)"""
    out = []
    for graph in (False, True):
        monkeypatch.setenv('DASR_B200_GRAPH', '1' if graph else '0')
        net = make()
        n0 = replays[0]
        rec = scenario(net)
        torch.cuda.synchronize()
        out.append((rec, replays[0] - n0))
        del net
    (eager, r_eager), (graph, r_graph) = out
    assert r_eager == 0
    return eager, graph, r_graph


def _assert_same(eager, graph):
    d = _first_diff(eager, graph)
    assert d is None, 'eager vs CUDA graph: ' + d


STEPS = 4


def _two_forwards(variant):
    def scenario(net):
        opt = torch.optim.Adam(net.parameters(), lr=1e-3)
        rec = []
        for s in range(STEPS):
            opt.zero_grad()
            x1, x2, p1, p2 = _x(530 + 4 * s), _x(531 + 4 * s), _pat(532 + 4 * s), _pat(533 + 4 * s)
            if variant == 'sum':                                  # no reference kept to either output
                ((net(x1) * p1).sum() + (net(x2) * p2).sum()).backward()
            elif variant == 'keep':
                o1, o2 = net(x1), net(x2)
                ((o1 * p1).sum() + (o2 * p2).sum()).backward()
                rec += [('step %d out1' % s, o1.detach().clone()), ('step %d out2' % s, o2.detach().clone())]
            else:                                                  # two backwards, in forward order or reversed
                l1, l2 = (net(x1) * p1).sum(), (net(x2) * p2).sum()
                for loss in ((l1, l2) if variant == 'in_order' else (l2, l1)):
                    loss.backward()
            rec += _grads('step %d' % s, net)
            opt.step()
        return rec + _params(net)
    return scenario


@pytest.mark.gpu
@pytest.mark.parametrize('variant', ['sum', 'keep', 'in_order', 'reversed'])
@pytest.mark.parametrize('arch', sorted(NETS))
def test_two_forwards_one_step(monkeypatch, replays, arch, variant):
    """two generator calls before their backward: the first replays the graphs, the second finds them busy and runs
    eagerly; the graph node's backward must read its own activations, not the second call's"""
    eager, graph, n = _both(monkeypatch, replays, NETS[arch], _two_forwards(variant))
    _assert_same(eager, graph)
    assert n == 2 * STEPS, 'expected one forward and one backward replay per step, got %d replays' % n


def _retain(forward_between):
    def scenario(net):
        rec = []
        for s in range(STEPS):
            x, p = _x(550 + 3 * s), _pat(551 + 3 * s)
            loss = (net(x) * p).sum()
            loss.backward(retain_graph=True)
            if forward_between:
                (net(_x(552 + 3 * s)) * p).sum()
            loss.backward()
            rec += _grads('step %d' % s, net)
            _sgd(net)
        return rec + _params(net)
    return scenario


@pytest.mark.gpu
@pytest.mark.parametrize('arch', sorted(NETS))
def test_retain_graph_backward_twice(monkeypatch, replays, arch):
    eager, graph, n = _both(monkeypatch, replays, NETS[arch], _retain(False))
    _assert_same(eager, graph)
    assert n == 3 * STEPS - (3 if arch == 'srresnet' else 0), n


@pytest.mark.gpu
@pytest.mark.parametrize('arch', sorted(NETS))
def test_forward_between_retained_backwards_is_refused(monkeypatch, replays, arch):
    """backward, a replayed forward, then a second backward through the first node: the graphs' activations are the
    second forward's by then, so the graph path refuses (DasrError) where the eager path keeps its own activations"""
    monkeypatch.setenv('DASR_B200_GRAPH', '0')
    _retain(True)(NETS[arch]())
    monkeypatch.setenv('DASR_B200_GRAPH', '1')
    net = NETS[arch]()
    for s in range(2):                                     # SRResNet captures on the second sighting of a shape
        (net(_x(560)) * _pat(561)).sum().backward()
    net.zero_grad()
    n0 = replays[0]
    loss = (net(_x(562)) * _pat(563)).sum()
    loss.backward(retain_graph=True)
    (net(_x(564)) * _pat(563)).sum()
    assert replays[0] - n0 == 3, 'the graphs did not replay'
    with pytest.raises(DasrError):
        loss.backward()


def _dropped(net):
    opt = torch.optim.Adam(net.parameters(), lr=1e-3)
    rec = []
    for s in range(STEPS):
        opt.zero_grad()
        (net(_x(570 + 3 * s)) * _pat(571)).sum()          # a forward whose loss is dropped without backward
        out = net(_x(571 + 3 * s))
        (out * _pat(572 + 3 * s)).sum().backward()
        rec += [('step %d out' % s, out.detach().clone())] + _grads('step %d' % s, net)
        opt.step()
    return rec + _params(net)


@pytest.mark.gpu
@pytest.mark.parametrize('arch', sorted(NETS))
def test_dropped_forward_does_not_block_replay(monkeypatch, replays, arch):
    eager, graph, n = _both(monkeypatch, replays, NETS[arch], _dropped)
    _assert_same(eager, graph)
    assert n == 3 * STEPS - (1 if arch == 'srresnet' else 0), n


def _replace(net, index, scale):
    """replace the index-th parameter by a new nn.Parameter with other values and the same version counter"""
    name, p = list(net.named_parameters())[index]
    mod, attr = _owner(net, name)
    setattr(mod, attr, _replacement(p, scale))


def _replace_index(net):
    n = len(list(net.parameters()))
    i = 3
    assert i not in (0, n // 2, n - 1)
    return i


def _replace_train(net):
    rec = []
    for s in range(STEPS + 2):
        x, p = _x(580), _pat(581 + s)
        out = net(x)
        (out * p).sum().backward()
        rec += [('step %d out' % s, out.detach().clone())] + _grads('step %d' % s, net)
        _sgd(net)
        if s in (1, 3):
            _replace(net, _replace_index(net), 0.75 if s == 1 else 1.25)
    return rec + _params(net)


@pytest.mark.gpu
@pytest.mark.parametrize('arch', sorted(NETS))
def test_parameter_replaced_between_training_steps(monkeypatch, replays, arch):
    eager, graph, n = _both(monkeypatch, replays, NETS[arch], _replace_train)
    _assert_same(eager, graph)
    # RRDBNet captures on every new key; SRResNet on the second sighting (steps 0, 2, 4 are first sightings)
    assert n == 2 * (STEPS + 2) - (6 if arch == 'srresnet' else 0), n


def _replace_infer(net, make):
    rec = []
    x = _x(590)
    with torch.no_grad():
        for s in range(9):
            if s == 3:
                _replace(net, _replace_index(net), 0.5)
            if s == 6:
                net.load_state_dict(make(seed=597).state_dict())
            rec.append(('call %d' % s, net(x).clone()))
    return rec


@pytest.mark.gpu
@pytest.mark.parametrize('arch', sorted(NETS))
def test_parameter_replaced_or_reloaded_between_inference_replays(monkeypatch, replays, arch):
    """calls 0-2, a replaced parameter, calls 3-5, load_state_dict of other weights, calls 6-8: each block is seen,
    captured and replayed"""
    eager, graph, n = _both(monkeypatch, replays, NETS[arch], lambda net: _replace_infer(net, NETS[arch]))
    _assert_same(eager, graph)
    assert n == 6, n
    assert _first_diff(eager[2:3], [('call 2', eager[5][1])]) is not None, 'the replacement did not change the output'


def _infer_after_steps(net):
    opt = torch.optim.Adam(net.parameters(), lr=1e-3)
    rec, xv = [], _x(600, (1, 3, 9, 14))
    for s in range(STEPS):
        opt.zero_grad()
        (net(_x(601)) * _pat(602 + s)).sum().backward()
        opt.step()
        with torch.no_grad():
            rec += [('step %d val a' % s, net(xv).clone()), ('step %d val b' % s, net(xv).clone())]
    return rec + _params(net)


@pytest.mark.gpu
@pytest.mark.parametrize('arch', sorted(NETS))
def test_inference_after_optimizer_steps(monkeypatch, replays, arch):
    """validation after each step: the inference graph of the previous step's weights must not be replayed"""
    eager, graph, n = _both(monkeypatch, replays, NETS[arch], _infer_after_steps)
    _assert_same(eager, graph)
    train = 2 * STEPS - (2 if arch == 'srresnet' else 0)
    assert n == train + STEPS, n


A_, B_, C_ = (2, 3, 13, 11), (1, 3, 10, 17), (3, 3, 8, 8)


def _shapes_infer(seq):
    def scenario(net):
        with torch.no_grad():
            return [('call %d' % i, net(_x(610 + i, s)).clone()) for i, s in enumerate(seq)]
    return scenario


# seen / captured on the second sighting / at most two graphs: A A A B B A C C A B B -> replays at calls 1 2 4 5 7 10
SEQ_INFER = [A_, A_, A_, B_, B_, A_, C_, C_, A_, B_, B_]


@pytest.mark.gpu
@pytest.mark.parametrize('arch', sorted(NETS))
def test_shape_alternation_inference(monkeypatch, replays, arch):
    eager, graph, n = _both(monkeypatch, replays, NETS[arch], _shapes_infer(SEQ_INFER))
    _assert_same(eager, graph)
    assert n == 6, n


def _shapes_train(seq):
    def scenario(net):
        rec = []
        for i, s in enumerate(seq):
            out = net(_x(620 + i, s))
            (out * _pat(640 + i, s)).sum().backward()
            rec += [('step %d out' % i, out.detach().clone())] + _grads('step %d' % i, net)
            _sgd(net)
        return rec + _params(net)
    return scenario


@pytest.mark.gpu
@pytest.mark.parametrize('arch', sorted(NETS))
def test_shape_alternation_training(monkeypatch, replays, arch):
    """A B A C A B: every change of shape re-captures (RRDBNet: on the first call of a shape, so every step replays;
    SRResNet: on the second call in a row, A A B B A C C)"""
    seq = [A_, B_, A_, C_, A_, B_] if arch == 'rrdbnet' else [A_, A_, B_, B_, A_, C_, C_]
    eager, graph, n = _both(monkeypatch, replays, NETS[arch], _shapes_train(seq))
    _assert_same(eager, graph)
    assert n == (12 if arch == 'rrdbnet' else 6), n


@pytest.mark.gpu
def test_adaptive_shapes_and_weight_maps(monkeypatch, replays):
    """the adaptive generator over A A A B B A C C A B B with a different weight map on every call"""
    def scenario(net):
        with torch.no_grad():
            return [('call %d' % i, net(_x(650 + i, s), _x(670 + i, (s[0], 1, s[2], s[3]))).clone())
                    for i, s in enumerate(SEQ_INFER)]
    eager, graph, n = _both(monkeypatch, replays, _adaptive, scenario)
    _assert_same(eager, graph)
    assert n == 6, n


@pytest.mark.gpu
@pytest.mark.parametrize('arch', sorted(NETS))
def test_precision_alternation(monkeypatch, replays, arch):
    """bf16 bf16 fp16 fp16 bf16 bf16 fp16, as bench.py alternates them: replays at calls 1 3 4 5 6"""
    def scenario(net):
        rec, x = [], _x(690)
        with torch.no_grad():
            for i, prec in enumerate(['bf16', 'bf16', 'fp16', 'fp16', 'bf16', 'bf16', 'fp16']):
                net.precision = prec
                rec.append(('call %d %s' % (i, prec), net(x).clone()))
        return rec
    eager, graph, n = _both(monkeypatch, replays, NETS[arch], scenario)
    _assert_same(eager, graph)
    assert n == 5, n
    assert _first_diff(eager[:1], [('call 0 bf16', eager[2][1])]) is not None, 'fp16 gave the bf16 result'


def _forms():
    base = _x(700, (2, 3, 15, 14))
    return {'slice': base[:, :, 1:14, 2:13], 'channels_last': _x(701).contiguous(memory_format=torch.channels_last),
            'fp16': _x(702).half(), 'float64': _x(703).double()}


def _outcome(fn):
    try:
        return fn()
    except (DasrError, NotImplementedError, RuntimeError, TypeError) as e:
        return [('refused %s' % type(e).__name__, torch.zeros(1))]


@pytest.mark.gpu
@pytest.mark.parametrize('form', ['slice', 'channels_last', 'fp16', 'float64'])
@pytest.mark.parametrize('arch', sorted(NETS))
def test_input_forms(monkeypatch, replays, arch, form):
    """a non-contiguous slice, a channels_last tensor, an fp16 and a float64 input, alternating with the plain fp32
    input of the same shape: graph and eager agree (or both refuse), in inference and in training"""
    def scenario(net):
        xs = _forms()
        plain, odd = _x(704), xs[form]
        assert tuple(odd.shape) == SHAPE
        rec = []
        with torch.no_grad():
            for i, x in enumerate([plain, odd, odd, odd, plain, odd]):
                rec += _outcome(lambda: [('infer %d' % i, net(x).clone())])
        for i, x in enumerate([odd, odd, plain, odd, odd]):
            def step():
                out = net(x)
                (out * _pat(705 + i)).sum().backward()
                r = [('step %d out' % i, out.detach().clone())] + _grads('step %d' % i, net)
                _sgd(net)
                return r
            rec += _outcome(step)
        return rec + _params(net)
    eager, graph, n = _both(monkeypatch, replays, NETS[arch], scenario)
    _assert_same(eager, graph)
    assert n > 0


# ---------------------------------------------------------------------------------------------------- the arena on one GPU

def _with_arena(make):
    def build():
        net = make()
        net.set_grad_arena(torch.zeros(sum(p.numel() for p in net.parameters()), device='cuda'))
        return net
    return build


ARENA_CASES = {'two_forwards': _two_forwards('sum'), 'two_forwards_reversed': _two_forwards('reversed'),
               'retain_graph': _retain(False)}


def _accumulate(net):
    opt = torch.optim.Adam(net.parameters(), lr=1e-3)
    rec = []
    for s in range(STEPS):
        opt.zero_grad()
        for k in range(2):                                   # two backwards into the same .grad, no zero_grad between
            (net(_x(720 + 2 * s + k)) * _pat(730 + 2 * s + k)).sum().backward()
        rec += _grads('step %d' % s, net)
        opt.step()
    return rec + _params(net)


ARENA_CASES['accumulate'] = _accumulate


@pytest.mark.gpu
@pytest.mark.parametrize('case', sorted(ARENA_CASES))
def test_arena_matches_fresh_gradients(monkeypatch, replays, case):
    """RRDBNet with a gradient arena (set_grad_arena, as dp.GradBucket does) against the same runs without one, each in
    graph and eager mode: the sums autograd forms are of two fp32 terms, exact in either order"""
    scenario = ARENA_CASES[case]
    plain_e, plain_g, n_plain = _both(monkeypatch, replays, _rrdbnet, scenario)
    arena_e, arena_g, n_arena = _both(monkeypatch, replays, _with_arena(_rrdbnet), scenario)
    _assert_same(plain_e, plain_g)
    for a, b, what in ((plain_e, arena_e, 'eager'), (plain_g, arena_g, 'CUDA graph')):
        d = _first_diff(a, b)
        assert d is None, '%s, with vs without the arena: %s' % (what, d)
    assert n_arena == n_plain and n_arena >= 2 * STEPS, (n_plain, n_arena)


@pytest.mark.gpu
@pytest.mark.parametrize('graph', ['0', '1'])
def test_arena_single_call_steps_are_zero_copy(monkeypatch, replays, graph):
    """the data-parallel step: one generator call per step, every .grad a view inside the arena"""
    monkeypatch.setenv('DASR_B200_GRAPH', graph)
    net = _with_arena(_rrdbnet)()
    arena = net._grad_arena
    opt = torch.optim.Adam(net.parameters(), lr=1e-3)
    n0 = replays[0]
    for s in range(STEPS):
        opt.zero_grad()
        (net(_x(740)) * _pat(741 + s)).sum().backward()
        outside = [n for n, p in net.named_parameters() if not _in_arena(p.grad, arena)]
        assert not outside, 'step %d: .grad not in the arena: %s' % (s, outside[:4])
        opt.step()
    assert replays[0] - n0 == (2 * STEPS if graph == '1' else 0)


# ---------------------------------------------------------------------------------------------------- DASR_Model

def _dasr_steps(graph, monkeypatch, replays):
    from helpers import make_opt, unwrap
    from dasr_b200.srn.models import create_model
    monkeypatch.setenv('DASR_B200_GRAPH', '1' if graph else '0')
    model = create_model(make_opt(True, 'DASR', 1, 'wavelet'))
    G, D = unwrap(model.netG), unwrap(model.netD_target)
    G.load_state_dict(O.synth_state_dict(O.rrdbnet_shapes(nb=1), 801, 0.5))
    G.train_precision = 'bf16'
    D.load_state_dict(O.synth_state_dict(O.nlayer_d_shapes(9, 64, 2), 802, 1.0))
    unwrap(model.netF).load_state_dict(O.synth_state_dict(O.vgg19_shapes(34), 803, 1.0), strict=False)
    B, h, w = 2, 16, 16
    rec, n0 = [], replays[0]
    for step in range(1, 5):
        seed = 810 + 10 * step
        model.feed_data({'LR_real': O.synth_image((B, 3, h, w), seed), 'LR_fake': O.synth_image((B, 3, h, w), seed + 1),
                         'HR': O.synth_image((B, 3, 4 * h, 4 * w), seed + 2),
                         'HR_unpair': O.synth_image((B, 3, 4 * h, 4 * w), seed + 3),
                         'fake_w': O.synth_image((B, 1, h, w), seed + 4)}, True)
        model.optimize_parameters(step)
        torch.cuda.synchronize()
        rec.append(('step %d fake_H' % step, model.fake_H.detach().clone()))
        rec += [('step %d log %s' % (step, k), torch.tensor(float(v), dtype=F64)) for k, v in model.get_current_log().items()]
        rec += _grads('step %d G' % step, G) + _grads('step %d D' % step, D)
        if step % 2:                 # validation after steps 1 and 3; steps 2 -> 3 keep the training fake_H alive
            model.feed_data({'LR': O.synth_image((1, 3, 12, 20), seed + 5)}, False)
            model.test()
            rec.append(('step %d val' % step, model.fake_H.detach().clone()))
    rec += _params(G) + _params(D)
    n = replays[0] - n0
    del model
    return rec, n


@pytest.mark.gpu
def test_dasr_model_steps_graph_equals_eager(monkeypatch, replays):
    """four DASR_Model steps (nb 1, wavelet) with test() on a validation image of another size after steps 1 and 3:
    fake_H, the logged values, every G and D gradient and the parameters agree bit for bit, and every step replays G's
    graphs, also the one after a step whose fake_H (and so its autograd node) is still held"""
    eager, n_eager = _dasr_steps(False, monkeypatch, replays)
    graph, n_graph = _dasr_steps(True, monkeypatch, replays)
    assert n_eager == 0
    _assert_same(eager, graph)
    assert n_graph == 2 * 4, 'expected a forward and a backward replay per step, got %d' % n_graph
