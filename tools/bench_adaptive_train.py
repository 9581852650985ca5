"""Forward + backward time of the adaptive-weight RRDB generators' training nodes, bf16 (mixed precision) and fp32, next to
RRDBNet-23 at the same shape (eager; RRDBNet's bf16 step also eager, DASR_B200_GRAPH=0, so the three run the same way):
  * RRDBNet_Residual_conv nb 19: the generator of train_DASR_Adaptive.json (define_G gives it one adaptive block);
  * RRDBNet_Residual_conv_concat nb 19, nb_ada 4;
  * RRDBNet nb 23.
Batches 4 x 3 x 48 x 48 (that config's batch) and 16 x 3 x 48 x 48.  Each configuration: `--warmup` untimed steps, then
`--steps` steps between CUDA events (loss = sum(out * pattern), gradients of every parameter and, for the adaptive
generators, of the map).  Prints one JSON object with the card's name and power limit.

    python tools/bench_adaptive_train.py [--steps 5] [--warmup 2] [--out result.json]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ['DASR_B200_GRAPH'] = '0'

import torch  # noqa: E402

from oracle import adaptive_oracle as AO  # noqa: E402
from oracle import srn_oracle as O  # noqa: E402

NETS = [('adaptive_plain_nb19', False, 19, 1), ('adaptive_concat_nb19_ada4', True, 19, 4), ('rrdbnet_nb23', None, 23, 0)]
BATCHES = [4, 16]
HW = 48


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True)
    name, power = [s.strip() for s in q.stdout.strip().splitlines()[0].split(',')]
    return name, power


def build(kind, nb, nb_ada):
    from dasr_b200.srn.models.modules import architecture as A
    if kind is None:
        net = A.RRDBNet(3, 3, 64, nb, gc=32, upscale=4)
        net.load_state_dict(O.synth_state_dict(O.rrdbnet_shapes(nb=nb), 7, 0.3))
    else:
        cls = A.RRDBNet_Residual_conv_concat if kind else A.RRDBNet_Residual_conv
        net = cls(3, 3, 64, nb, gc=32, upscale=4, nb_ada=nb_ada)
        net.load_state_dict(AO.synth_adaptive_g(nb, nb_ada, kind, 7, 0.3))
    return net.cuda()


def time_steps(net, adaptive, n, prec, steps, warmup):
    net.train_precision = prec
    x = O.synth_image((n, 3, HW, HW), 11).cuda()
    amap = O.synth_image((n, 1, HW, HW), 12).cuda()
    pattern = O.synth((n, 3, 4 * HW, 4 * HW), 13).cuda()

    def step():
        net.zero_grad(set_to_none=True)
        a = amap.clone().requires_grad_(True)
        out = net(x, a) if adaptive else net(x)
        (out * pattern).sum().backward()
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(steps):
        step()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_adaptive_train: no CUDA device; nothing is measured without one')
    name, power = card()
    res = dict(card=name, power_limit=power, hw=HW, steps=args.steps, warmup=args.warmup, ms_per_step={})
    for label, kind, nb, nb_ada in NETS:
        net = build(kind, nb, nb_ada)
        for n in BATCHES:
            for prec in ('bf16', 'fp32'):
                ms = time_steps(net, kind is not None, n, prec, args.steps, args.warmup)
                res['ms_per_step']['%s/N%d/%s' % (label, n, prec)] = round(ms, 2)
                print('%-28s N %2d %s: %9.2f ms / forward + backward' % (label, n, prec, ms), file=sys.stderr, flush=True)
        del net
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
