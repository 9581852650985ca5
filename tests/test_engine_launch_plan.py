"""The launch plan of the wgmma generator forwards, checked without a GPU.

engine.py decides every kernel launch of the generators.  Here its forwards run on CPU tensors against a recording stand-in
for the C-ABI library: host-only queries (conv setup, pair-kernel support, packed-filter sizes, workspace sizes) go to the
real library, every other entry point is recorded and returns success.  Device pointers become tokens (ordinal of the
storage by first use, byte offset), parameter structs are recorded field by field.  The recorded plans must equal
tests/golden/engine_launch_plans.json, so a change of engine.py that alters any launch, its order or its parameters fails
here.  The backward is not covered: it needs CUDA streams and events.

`python tests/test_engine_launch_plan.py` rewrites the fixture from the current tree."""
import ctypes as C
import hashlib
import json
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
FIXTURE = os.path.join(ROOT, 'tests', 'golden', 'engine_launch_plans.json')
HOST_ONLY = {'dasr_conv_tc_setup', 'dasr_conv_tc2_supported', 'dasr_pack_filter_tc_bytes', 'dasr_last_error'}


def _value(v):
    return [_value(e) for e in v] if isinstance(v, C.Array) else v


def _nonzero(v):
    return any(_nonzero(e) for e in v) if isinstance(v, list) else v != 0


def _fields(s):
    """The fields of a ctypes struct that are not zero (the structs have no padding, so this is their byte image)."""
    out = {}
    for name, _ in s._fields_:
        v = _value(getattr(s, name))
        if _nonzero(v):
            out[name] = v
    return out


class _Recorder:
    """Stands in for the loaded library: records the calls of a forward instead of launching kernels."""

    def __init__(self, lib, tok):
        self.lib, self.tok, self.calls = lib, tok, []

    def __getattr__(self, name):
        fn = getattr(self.lib, name)
        if name in HOST_ONLY or name.endswith('_workspace'):
            return fn

        def record(*args):
            self.calls.append([name] + [self.arg(a) for a in args])
            return 0
        return record

    def arg(self, a):
        if type(a).__name__ == 'CArgObject':          # C.byref(struct)
            return _fields(a._obj)
        return a


class _Tokens:
    """Pointer -> [storage ordinal by first use, byte offset].  Every storage seen stays referenced, so a freed CPU buffer
    cannot hand its address to a later one."""

    def __init__(self):
        self.ords, self.keep = {}, []

    def tensor(self, t):
        st = t.untyped_storage()
        base = st.data_ptr()
        if base not in self.ords:
            self.ords[base] = (len(self.ords), st.nbytes())
            self.keep.append(st)
        return ['ptr', self.ords[base][0], t.data_ptr() - base]

    def raw(self, p):
        if p is None:
            return None
        for base, (o, n) in self.ords.items():
            if base <= p < base + n:
                return ['ptr', o, p - base]
        raise AssertionError('pointer outside every storage the forward used')


def _install(mp, lib):
    """Route the forwards of dasr_b200 into a fresh recorder over the real library `lib`; mp: pytest's monkeypatch."""
    from dasr_b200 import _lib, engine, ops
    tok = _Tokens()
    rec = _Recorder(lib, tok)

    def p(t):
        if t is None:
            return None
        if not t.is_contiguous():
            raise _lib.DasrError('dasr_b200 kernels need contiguous tensors')
        return tok.tensor(t)
    mp.setattr(_lib, '_lib', rec)
    mp.setattr(_lib, 'LAUNCHES', _lib.LAUNCHES)
    mp.setattr(ops, '_p', p)
    mp.setattr(ops, '_stream', lambda: None)
    mp.setattr(engine, '_need_cuda', lambda x, what: None)
    mp.setenv('DASR_B200_GRAPH', '0')
    return rec, tok


def _real_lib():
    from dasr_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__ as g
        g.build()
    return _lib.load()


@pytest.fixture
def plan(monkeypatch):
    return _install(monkeypatch, _real_lib())


def _rrdbnet(nb, prec):
    from dasr_b200.srn.models.modules.architecture import RRDBNet
    torch.manual_seed(0)
    net = RRDBNet(3, 3, 64, nb, gc=32, upscale=4).eval()
    net.precision = prec
    net(torch.rand(2, 3, 12, 16))


def _adaptive(concat, prec):
    from dasr_b200.srn.models.modules import architecture as A
    torch.manual_seed(0)
    cls = A.RRDBNet_Residual_conv_concat if concat else A.RRDBNet_Residual_conv
    net = cls(3, 3, 64, 1, gc=32, upscale=4, nb_ada=1).eval()
    net.precision = prec
    net(torch.rand(2, 3, 12, 16), torch.rand(2, 1, 12, 16))


def _train(nb):
    from dasr_b200 import engine
    from dasr_b200.srn.models.modules.architecture import RRDBNet
    torch.manual_seed(0)
    params = [q.detach() for q in RRDBNet(3, 3, 64, nb, gc=32, upscale=4).parameters()]
    engine.rrdb_forward_bf16_train(torch.rand(2, 3, 12, 16), params, nb, 4, engine._PackCache())


def _batch_packer(rec, tok, nb):
    """The job table of one _BatchPacker (decoded, pointers as tokens), its cache keys, and its launch."""
    from dasr_b200 import engine
    from dasr_b200._lib import PackJob
    from dasr_b200.srn.models.modules.architecture import RRDBNet
    torch.manual_seed(0)
    params = [q.detach() for q in RRDBNet(3, 3, 64, nb, gc=32, upscale=4).parameters()]
    L = engine.RRDBLayout(nb, 64, 4)
    bp = engine._BatchPacker(params, L, L.nf)
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
for _nb in (1, 2):
    for _prec in ('bf16', 'fp16', 'bf16_layer', 'fp16_layer'):
        CONFIGS['rrdbnet_nb%d_%s' % (_nb, _prec)] = (lambda rec, tok, nb=_nb, prec=_prec: _rrdbnet(nb, prec))
for _concat in (True, False):
    for _prec in ('bf16', 'fp16'):
        CONFIGS['adaptive_%s_%s' % ('concat' if _concat else 'plain', _prec)] = \
            (lambda rec, tok, concat=_concat, prec=_prec: _adaptive(concat, prec))
CONFIGS['train_nb2'] = lambda rec, tok: _train(2)
CONFIGS['batch_packer_nb1'] = lambda rec, tok: _batch_packer(rec, tok, 1)


def _record(rec, tok, name):
    with torch.no_grad():
        CONFIGS[name](rec, tok)
    calls = json.loads(json.dumps(rec.calls))
    return dict(n=len(calls), sha256=hashlib.sha256(json.dumps(calls).encode()).hexdigest(), calls=calls)


@pytest.mark.parametrize('name', sorted(CONFIGS))
def test_launch_plan_matches_fixture(plan, name):
    rec, tok = plan
    got = _record(rec, tok, name)
    with open(FIXTURE) as f:
        want = json.load(f)[name]
    assert got['n'] == want['n'], (got['n'], want['n'])
    for i, (a, b) in enumerate(zip(got['calls'], want['calls'])):
        assert a == b, 'call %d of %s differs:\n got %s\nwant %s' % (i, name, a, b)
    assert got['sha256'] == want['sha256']


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
