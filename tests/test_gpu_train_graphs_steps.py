"""Mixed-precision training on CUDA graphs across optimizer steps: the graphs must re-pack every filter from the live
parameters on each replay.  Several steps with graph replay and the same steps run eagerly (DASR_B200_GRAPH=0) from the
same weights must give bit-identical outputs, gradients and parameters once the optimizer has changed the parameters, for
SRResNet (SRModel, sr_resnet) and RRDBNet (Adam on the generator alone)."""
import pytest
import torch

from oracle import srn_oracle as O

pytestmark = pytest.mark.gpu


def _bits(t):
    return t.detach().contiguous().view(torch.int32)


def _first_diff(a, b):
    for (n, u), (_, v) in zip(a, b):
        if not torch.equal(_bits(u), _bits(v)):
            return '%s: %d elements differ, max |diff| %.3g' % (n, int((u != v).sum()), float((u - v).abs().max()))
    return None


def _srmodel_steps(sd, nb, data, graph, monkeypatch, steps=4):
    from helpers import make_opt, unwrap
    from dasr_b200.srn.models import create_model
    monkeypatch.setenv('DASR_B200_GRAPH', '1' if graph else '0')
    opt = make_opt(True, 'sr', nb=nb)
    opt['network_G']['which_model_G'] = 'sr_resnet'
    m = create_model(opt)
    g = unwrap(m.netG)
    g.load_state_dict(sd)
    g.train_precision = 'bf16'
    rec = []
    for step in range(steps):
        m.feed_data(data)
        m.optimize_parameters(step)
        torch.cuda.synchronize()
        rec.append([('step %d out' % step, m.fake_H.detach().float().clone())] +
                   [('step %d grad %s' % (step, n), p.grad.detach().clone()) for n, p in g.named_parameters()])
    rec.append([('param %s' % n, p.detach().clone()) for n, p in g.named_parameters()])
    if graph:
        assert g._train_graphs, 'the CUDA-graph training path was not taken'
    del m
    return rec


def test_srmodel_graph_steps_equal_eager_steps(monkeypatch):
    """four SRModel steps (sr_resnet nb 2, L1, Adam): capture at the second step, replays at the third and fourth"""
    from dasr_b200.srn.models.modules.sr_nets import SRResNet
    nb = 2
    net = SRResNet(3, 3, 64, nb, upscale=4, norm_type=None, act_type='relu', mode='CNA', upsample_mode='pixelshuffle')
    sd = {k: O.synth(tuple(v.shape), 301000 + i, (6.0 / v[0].numel()) ** 0.5 if v.dim() == 4 else 0.05)
          for i, (k, v) in enumerate(net.state_dict().items())}
    data = {'LR': O.synth_image((4, 3, 16, 16), 302), 'HR': O.synth_image((4, 3, 64, 64), 303)}
    eager = _srmodel_steps(sd, nb, data, False, monkeypatch)
    graph = _srmodel_steps(sd, nb, data, True, monkeypatch)
    assert not torch.equal(eager[-1][-1][1], sd['model.10.bias'].cuda()), 'the optimizer did not change the last layer'
    for e, g in zip(eager, graph):
        d = _first_diff(e, g)
        assert d is None, 'eager vs CUDA graph: ' + d


def _rrdb_steps(sd, nb, x, pattern, graph, monkeypatch, steps=4):
    from dasr_b200.srn.models.modules.architecture import RRDBNet
    monkeypatch.setenv('DASR_B200_GRAPH', '1' if graph else '0')
    net = RRDBNet(3, 3, 64, nb, gc=32, upscale=4)
    net.load_state_dict(sd)
    net.cuda()
    net.train_precision = 'bf16'
    opt = torch.optim.Adam(net.parameters(), lr=1e-3)
    rec = []
    for step in range(steps):
        opt.zero_grad()
        out = net(x)
        (out * pattern).sum().backward()
        opt.step()
        torch.cuda.synchronize()
        rec.append([('step %d out' % step, out.detach().clone())] +
                   [('step %d grad %s' % (step, n), p.grad.detach().clone()) for n, p in net.named_parameters()])
    if graph:
        assert net._train_graphs, 'the CUDA-graph training path was not taken'
    return rec


def test_rrdbnet_graph_steps_equal_eager_steps(monkeypatch):
    """four Adam steps of RRDBNet nb 1: capture at the first step, replays after every parameter update"""
    nb = 1
    sd = O.synth_state_dict(O.rrdbnet_shapes(nb=nb), 311, 0.5)
    x = O.synth_image((2, 3, 13, 11), 312).cuda()
    pattern = O.synth((2, 3, 52, 44), 313).cuda()
    eager = _rrdb_steps(sd, nb, x, pattern, False, monkeypatch)
    graph = _rrdb_steps(sd, nb, x, pattern, True, monkeypatch)
    for e, g in zip(eager, graph):
        d = _first_diff(e, g)
        assert d is None, 'eager vs CUDA graph: ' + d
