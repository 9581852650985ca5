"""Generate tests/golden/adaptive_grads.pt by running the UNMODIFIED reference generators (<DASR checkout>/codes/SRN,
models/modules/architecture.py RRDBNet_Residual_conv_concat / RRDBNet_Residual_conv) forward and backward on CPU in fp32:
the output, every parameter gradient, the map gradient and the input-image gradient of sum(out * pattern).  A gradient of more
than SAMPLES values (the filters) is kept as its L2 norm and its values at SAMPLES evenly spaced flat indices (sample_idx), so
the fixture stays small; biases, the map-channel slices of the 65-channel filters, the output and the map / input gradients
are kept whole.  Imported like oracle/gen_golden_adaptive.py (DASR_REFERENCE = the checkout's root, oracle/ref_stubs for
the third-party modules the reference imports at module level).  Weights, inputs, maps and loss patterns come from oracle.srn_oracle.synth* and
oracle.adaptive_oracle (hash based, no RNG).

    python oracle/gen_golden_adaptive_grads.py
"""
import os
import sys
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

from oracle import adaptive_oracle as AO  # noqa: E402
from oracle import srn_oracle as O  # noqa: E402

OUT = os.path.join(ROOT, 'tests', 'golden', 'adaptive_grads.pt')
torch.set_num_threads(8)

# (name, class, concat, nb, nb_ada, weight seed)
GENERATORS = [('concat', arch.RRDBNet_Residual_conv_concat, True, 2, 2, 401),
              ('plain', arch.RRDBNet_Residual_conv, False, 2, 1, 402)]
GAIN = 0.3
SHAPE = (2, 3, 21, 13)              # a ragged batch of two
X_SEED, MAP_SEED, PATTERN_SEED = 411, 412, 413
SAMPLES = 512


def sample_idx(n):
    """the flat indices at which a gradient of n values is kept"""
    return torch.linspace(0, n - 1, min(n, SAMPLES), dtype=torch.float64).round().long()


def pack(g):
    if g.numel() <= SAMPLES:
        return dict(full=g.clone())
    d = dict(norm=float(g.double().norm()), values=g.reshape(-1)[sample_idx(g.numel())].clone())
    if g.dim() == 4 and g.shape[1] == 65:
        d['map_channel'] = g[:, 64].clone()
    return d


def main():
    rec = OrderedDict(samples=SAMPLES, gain=GAIN, shape=SHAPE, x_seed=X_SEED, map_seed=MAP_SEED, pattern_seed=PATTERN_SEED)
    n, c, h, w = SHAPE
    for name, cls, concat, nb, nb_ada, seed in GENERATORS:
        net = cls(3, 3, 64, nb, gc=32, upscale=4, norm_type=None, act_type='leakyrelu', mode='CNA', upsample_mode='upconv',
                  nb_ada=nb_ada)
        sd = AO.synth_adaptive_g(nb, nb_ada, concat, seed, GAIN)
        net.load_state_dict(sd, strict=True)
        x = O.synth_image(SHAPE, X_SEED).requires_grad_(True)
        a = O.synth_image((n, 1, h, w), MAP_SEED).requires_grad_(True)
        out = net(x, a)
        pattern = O.synth(tuple(out.shape), PATTERN_SEED)
        (out * pattern).sum().backward()
        grads = OrderedDict((k, pack(p.grad)) for k, p in net.named_parameters())
        print('  %s: out max %.3g, map grad max %.3g, %d parameter gradients' % (
            name, float(out.detach().abs().max()), float(a.grad.abs().max()), len(grads)))
        rec[name] = dict(nb=nb, nb_ada=nb_ada, w_seed=seed, out=out.detach().clone(), grads=grads, map_grad=a.grad.clone(),
                         x_grad=x.grad.clone())
    torch.save(rec, OUT)
    print('%s %.1f KB' % (OUT, os.path.getsize(OUT) / 1024))


if __name__ == '__main__':
    main()
