"""Time RRDBNet_Residual_conv_concat (nb 19, ada_nb 4: options/test/test_DASR_Adaptive.json) against RRDBNet-23 on the wgmma
bf16 path, CUDA-graph replay, CUDA events; the two generators alternate in one run.  Prints one JSON line.

    python tools/bench_adaptive.py [--steps 10] [--warmup 3]

Workloads: 16x3x256x256 (the RRDBNet benchmark shape) and one AIM-validation-sized image, 1x3x339x510.  FLOPs are counted
from shapes (2 per MAC, LR-pixel convs plus the x2 / x4 layers); the map stencil of the 65-channel convs is not counted.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from oracle import adaptive_oracle as AO  # noqa: E402
from oracle import srn_oracle as O  # noqa: E402

NF, GC = 64, 32


def flops_per_lr_pixel(nb, nb_ada):
    """2 x MACs per LR pixel of the generator (x4, 3 -> 3 channels)."""
    mac = lambda cin, cout: 9 * cin * cout
    rdb = sum(mac(NF + k * GC, GC) for k in range(4)) + mac(NF + 4 * GC, NF)
    lr_side = mac(3, NF) + 3 * (nb + nb_ada) * rdb + mac(NF, NF)
    ada = 4 * (mac(NF + 1, NF) + mac(NF, NF))       # per adaptive block: A (3x) and R (1x), each 65 -> 64 -> 64
    hr_side = 4 * mac(NF, NF) + 16 * (mac(NF, NF) + mac(NF, NF) + mac(NF, 3))
    return 2 * (lr_side + nb_ada * ada + hr_side)


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in q.split(',')]
        return name, power
    except Exception as e:  # pragma: no cover
        return torch.cuda.get_device_name(0), 'unknown (%s)' % type(e).__name__


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--rounds', type=int, default=3, help='alternations of the two generators per shape')
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_adaptive needs a GPU'
    from dasr_b200.srn.models.modules.architecture import RRDBNet, RRDBNet_Residual_conv_concat
    ada = RRDBNet_Residual_conv_concat(3, 3, NF, 19, nb_ada=4)
    ada.load_state_dict(AO.synth_adaptive_g(19, 4, True, 401, 0.3))
    base = RRDBNet(3, 3, NF, 23)
    base.load_state_dict(O.synth_state_dict(O.rrdbnet_shapes(nb=23), 402, 0.3))
    ada, base = ada.cuda().eval(), base.cuda().eval()
    ada.precision = base.precision = 'bf16'
    name, power = card()
    res = {'metric': 'adaptive_vs_rrdbnet23_forward', 'card': name, 'power_limit': power, 'precision': 'bf16', 'shapes': []}
    f_ada, f_base = flops_per_lr_pixel(19, 4), flops_per_lr_pixel(23, 0)
    res['flop_per_lr_pixel'] = {'adaptive_nb19_ada4': f_ada, 'rrdbnet23': f_base, 'ratio': f_ada / f_base}
    for shape in ((16, 3, 256, 256), (1, 3, 339, 510)):
        x = O.synth_image(shape, 403).cuda()
        a = O.synth_image((shape[0], 1) + shape[2:], 404).cuda()
        runs = {'adaptive': (lambda: ada(x, a)), 'rrdbnet23': (lambda: base(x))}
        times = {k: [] for k in runs}
        with torch.no_grad():
            for k, fn in runs.items():
                for _ in range(max(args.warmup, 2) + 1):      # eager, eager (graph key seen), captured graph + replays
                    fn()
            torch.cuda.synchronize()
            for _ in range(args.rounds):
                for k, fn in runs.items():
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(args.steps):
                        fn()
                    e1.record()
                    e1.synchronize()
                    times[k].append(e0.elapsed_time(e1) / args.steps)
        npx = shape[0] * shape[2] * shape[3]
        row = {'shape': list(shape)}
        for k, f in (('adaptive', f_ada), ('rrdbnet23', f_base)):
            t = times[k]
            row[k] = {'ms': min(t), 'ms_runs': t, 'tflops': f * npx / (min(t) * 1e-3) / 1e12}
        row['time_per_flop_ratio'] = (row['adaptive']['ms'] / f_ada) / (row['rrdbnet23']['ms'] / f_base)
        row['rrdbnet23_spread'] = max(times['rrdbnet23']) / min(times['rrdbnet23']) - 1
        res['shapes'].append(row)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
