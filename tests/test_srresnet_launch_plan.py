"""The launch plan of SRResNet on the wgmma kernels, checked without a GPU, with the recorder of test_engine_launch_plan.py:
the bf16 / fp16 inference forwards at x4 and x2 (one of them on a ragged input), the mixed-precision training forward and
the training step's filter-pack job table.  The recorded plans must equal tests/golden/srresnet_launch_plans.json.

`python tests/test_srresnet_launch_plan.py` rewrites the fixture from the current tree."""
import hashlib
import json
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tests.test_engine_launch_plan import _fields, _install, _real_lib, plan  # noqa: E402,F401  (plan: the pytest fixture)

FIXTURE = os.path.join(ROOT, 'tests', 'golden', 'srresnet_launch_plans.json')


def _net(nb, upscale):
    from dasr_b200.srn.models.modules.sr_nets import SRResNet
    torch.manual_seed(0)
    return SRResNet(3, 3, 64, nb, upscale=upscale, norm_type=None, act_type='relu', mode='CNA', res_scale=1,
                    upsample_mode='pixelshuffle')


def _inference(nb, upscale, prec, shape):
    net = _net(nb, upscale).eval()
    net.precision = prec
    net(torch.rand(*shape))


def _train(nb, upscale):
    from dasr_b200 import engine
    params = [q.detach() for q in _net(nb, upscale).parameters()]
    engine.srresnet_forward_bf16_train(torch.rand(2, 3, 12, 16), params, nb, upscale, engine._PackCache())


def _packer(rec, tok, nb):
    """the job table of one SRResNet training-step packer (decoded, pointers as tokens), its cache keys, and its launch"""
    from dasr_b200 import engine
    from dasr_b200._lib import PackJob
    params = [q.detach() for q in _net(nb, 4).parameters()]
    bp = engine._SRResNetPacker(params, engine.SRResNetLayout(nb, 4))
    for t in params + bp.keep:
        tok.tensor(t)
    jobs = (PackJob * bp.njobs).from_buffer_copy(bytes(bp.table.numpy()))
    for j in jobs:
        f = _fields(j)
        f['src'], f['dst'] = tok.raw(j.src), tok.raw(j.dst)
        rec.calls.append(['job', f])
    for key in sorted(bp.cache.d, key=repr):
        t = bp.cache.d[key][1]
        rec.calls.append(['cache', repr(key), list(t.shape), str(t.dtype), tok.tensor(t)])
    bp.launch()


CONFIGS = {}
for _up in (4, 2):
    for _prec in ('bf16', 'fp16'):
        CONFIGS['srresnet_nb2_x%d_%s' % (_up, _prec)] = \
            (lambda rec, tok, up=_up, prec=_prec: _inference(2, up, prec, (2, 3, 12, 16)))
CONFIGS['srresnet_nb2_x4_bf16_ragged'] = lambda rec, tok: _inference(2, 4, 'bf16', (1, 3, 23, 37))
CONFIGS['srresnet_train_nb2_x4'] = lambda rec, tok: _train(2, 4)
CONFIGS['srresnet_train_nb2_x2'] = lambda rec, tok: _train(2, 2)
CONFIGS['srresnet_packer_nb2'] = lambda rec, tok: _packer(rec, tok, 2)


def _record(rec, tok, name):
    with torch.no_grad():
        CONFIGS[name](rec, tok)
    calls = json.loads(json.dumps(rec.calls))
    return dict(n=len(calls), sha256=hashlib.sha256(json.dumps(calls).encode()).hexdigest(), calls=calls)


@pytest.mark.parametrize('name', sorted(CONFIGS))
def test_srresnet_launch_plan_matches_fixture(plan, name):
    rec, tok = plan
    got = _record(rec, tok, name)
    with open(FIXTURE) as f:
        want = json.load(f)[name]
    assert got['n'] == want['n'], (got['n'], want['n'])
    for i, (a, b) in enumerate(zip(got['calls'], want['calls'])):
        assert a == b, 'call %d of %s differs:\n got %s\nwant %s' % (i, name, a, b)
    assert got['sha256'] == want['sha256']


def test_ps_launch_parameters(plan):
    """every pixel-shuffle launch: setup kind 4 geometry, Cout 4 nf in tiles of nf, the HR tensor's channel stride, the
    staged epilogue (fields that are zero are not recorded)"""
    rec, tok = plan
    calls = _record(rec, tok, 'srresnet_nb2_x4_bf16')['calls']
    ps = [c[-2] for c in calls if c[0] == 'dasr_conv_tc' and c[-2].get('out_mul') == 2]
    assert len(ps) == 2
    for p in ps:
        assert (p['nvar'], p['ntaps'], p['cout'], p['nt'], p['out_cs'], p.get('epi_mode', 0)) == (1, 9, 256, 64, 64, 0)
        assert p['out_py'] == [0, 0, 1, 1] and p['out_px'] == [0, 1, 0, 1] and p['act'] == 2


@pytest.mark.parametrize('nf', [96, 192])
def test_uncovered_nf_set_on_the_module_raises(nf):
    """nf without a wgmma plan (a dgrad without a Cout tile that fits one SM): a 16-bit mode set on the module is refused
    with the reason before any launch"""
    from dasr_b200 import _lib, engine
    from dasr_b200.srn.models.modules.sr_nets import SRResNet
    assert engine.srresnet_tc_reason(nf) and all(engine.srresnet_tc_reason(n) is None for n in (32, 64, 128))
    net = SRResNet(3, 3, nf, 1, upscale=4, norm_type=None, act_type='relu', mode='CNA', upsample_mode='pixelshuffle').eval()
    net.precision = 'bf16'
    with pytest.raises(_lib.DasrError, match='nf %d' % nf):
        with torch.no_grad():
            net(torch.rand(1, 3, 8, 8))


if __name__ == '__main__':
    class _MP:
        """pytest's monkeypatch, enough of it for the fixture (patches are not undone: the process ends)."""
        setattr = staticmethod(setattr)

        @staticmethod
        def setenv(k, v):
            os.environ[k] = v
    out, lib = {}, _real_lib()
    for name in sorted(CONFIGS):
        rec, tok = _install(_MP(), lib)
        out[name] = _record(rec, tok, name)
        print(name, out[name]['n'], out[name]['sha256'][:16])
    with open(FIXTURE, 'w') as f:
        f.write('{\n' + ',\n'.join('%s: {"n": %d, "sha256": %s, "calls": [\n%s]}' % (
            json.dumps(k), v['n'], json.dumps(v['sha256']), ',\n'.join(json.dumps(c) for c in v['calls']))
            for k, v in out.items()) + '\n}\n')
