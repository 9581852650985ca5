"""Time SRResNet-16 (nf 64, x4, pixel shuffle: options/test/test_SRResNet.json) inference in fp32 / bf16 / fp16 and the
train_SRResNet.json step (SRModel, batch 16, HR 128, L1 + Adam) in fp32 and bf16.  Prints one JSON line.

    python tools/bench_srresnet.py [--steps 10] [--warmup 3] [--train-steps 20]

Weights: deterministic, with the magnitudes of the reference's init (kaiming, scale 0.1).
Inference: 16x3x256x256, CUDA-graph replay for the 16-bit modes (the module's own capture on the second sighting of a
shape), CUDA events around `steps` forwards after `warmup` untimed ones, the fp32 / bf16 / fp16 runs alternated `rounds`
times; the best round is reported with all rounds.  Algorithmic FLOPs are counted from shapes (2 per MAC):
5,145,984 per LR pixel (stem 3,456; 33 trunk convs 2,433,024; pixel-shuffle conv 1 294,912; pixel-shuffle conv 2 at 2x
1,179,648; HR_conv0 at 4x 1,179,648; HR_conv1 55,296).  The card name and power limit are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from oracle import srn_oracle as O  # noqa: E402

NF, NB = 64, 16


def flops_per_lr_pixel(nb=NB, nf=NF, in_nc=3, out_nc=3):
    """2 x MACs per LR pixel of SRResNet x4 with pixel-shuffle upsampling"""
    mac = lambda cin, cout: 9 * cin * cout
    return 2 * (mac(in_nc, nf) + (2 * nb + 1) * mac(nf, nf) + mac(nf, 4 * nf) + 4 * mac(nf, 4 * nf) + 16 * mac(nf, nf)
                + 16 * mac(nf, out_nc))


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in q.split(',')]
        return name, power
    except Exception as e:  # pragma: no cover
        return torch.cuda.get_device_name(0), 'unknown (%s)' % type(e).__name__


def _net(gain=0.1):
    """deterministic weights with the magnitudes of the reference's init (define_G: kaiming, scale 0.1)"""
    from dasr_b200.srn.models.modules.sr_nets import SRResNet
    net = SRResNet(3, 3, NF, NB, upscale=4, norm_type=None, act_type='relu', mode='CNA', upsample_mode='pixelshuffle')
    sd = net.state_dict()
    for i, (k, v) in enumerate(sd.items()):
        sd[k] = O.synth(tuple(v.shape), 501000 + i, gain * (6.0 / v[0].numel()) ** 0.5 if v.dim() == 4 else 0.01)
    net.load_state_dict(sd)
    return net


def bench_inference(args):
    net = _net().cuda().eval()
    x = O.synth_image((16, 3, 256, 256), 502).cuda()
    precs = ('fp32', 'bf16', 'fp16')
    times = {p: [] for p in precs}
    steps = {p: (max(1, args.steps // 5) if p == 'fp32' else args.steps) for p in precs}
    with torch.no_grad():
        for p in precs:
            net.precision = p
            for _ in range(max(args.warmup, 3)):          # eager, eager (shape seen), captured graph + replays
                net(x)
        torch.cuda.synchronize()
        for _ in range(args.rounds):
            for p in precs:
                net.precision = p
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(steps[p]):
                    net(x)
                e1.record()
                e1.synchronize()
                times[p].append(e0.elapsed_time(e1) / steps[p])
        net.precision = 'fp32'
        ref = net(x)
        errs = {}
        for p in ('bf16', 'fp16'):
            net.precision = p
            errs[p] = float((net(x) - ref).abs().max() / ref.abs().max())
    f = flops_per_lr_pixel()
    npx = 16 * 256 * 256
    out = {}
    for p in precs:
        ms = min(times[p])
        out[p] = {'ms': ms, 'ms_runs': times[p], 'steps': steps[p], 'output_mpix_per_s': 16 * npx / (ms * 1e-3) / 1e6,
                  'algorithmic_tflops': f * npx / (ms * 1e-3) / 1e12}
        if p in errs:
            out[p]['rel_linf_vs_fp32'] = errs[p]
    return out


def _sr_model(train_precision):
    from dasr_b200.srn.models import create_model
    from dasr_b200.srn.options.options import dict_to_nonedict
    opt = dict_to_nonedict({
        'name': 'bench_srresnet', 'model': 'sr', 'scale': 4, 'gpu_ids': [0], 'is_train': True, 'chop': False,
        'val_lpips': False, 'path': {'pretrain_model_G': None, 'models': '/tmp', 'training_state': '/tmp'},
        'network_G': {'which_model_G': 'sr_resnet', 'norm_type': None, 'mode': 'CNA', 'nf': NF, 'nb': NB, 'in_nc': 3,
                      'out_nc': 3, 'gc': 32, 'group': 1, 'scale': 4},
        'train': {'lr_G': 2e-4, 'weight_decay_G': 0, 'beta1_G': 0.9, 'lr_scheme': 'MultiStepLR',
                  'lr_steps': [200000, 400000], 'lr_gamma': 0.5, 'pixel_criterion': 'l1', 'pixel_weight': 1.0,
                  'manual_seed': 0, 'niter': 1000000}})
    m = create_model(opt)
    g = m.netG.module if isinstance(m.netG, torch.nn.DataParallel) else m.netG
    g.load_state_dict(_net().state_dict())
    g.train_precision = train_precision
    return m


def bench_train(args):
    data = {'LR': O.synth_image((16, 3, 32, 32), 503).pin_memory(), 'HR': O.synth_image((16, 3, 128, 128), 504).pin_memory()}
    out = {}
    for tp in ('fp32', 'bf16'):
        m = _sr_model(tp)
        for step in range(max(args.warmup, 3)):          # eager, graph capture, replays
            m.feed_data(data)
            m.optimize_parameters(step)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for step in range(args.train_steps):
            m.feed_data(data)
            m.optimize_parameters(step)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        out[tp] = {'it_per_s': args.train_steps / dt, 'ms_per_step': 1e3 * dt / args.train_steps,
                   'l_pix_last': m.log_dict['l_pix']}
        del m
        torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--rounds', type=int, default=3, help='alternations of the inference precisions')
    ap.add_argument('--train-steps', type=int, default=20)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_srresnet needs a GPU'
    name, power = card()
    res = {'metric': 'srresnet16_x4', 'card': name, 'power_limit': power, 'flop_per_lr_pixel': flops_per_lr_pixel(),
           'inference_16x3x256x256': bench_inference(args), 'train_SRResNet_step_b16_hr128': bench_train(args)}
    print(json.dumps(res))


if __name__ == '__main__':
    main()
