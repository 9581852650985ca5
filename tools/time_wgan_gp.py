"""What the WGAN-GP gradient penalty costs per training step: CUDA-event times of
  * the DSN iteration (De_resnet 8 blocks x4, FSD Instance wavelet D, VGG perceptual loss), batch 8, 256x256 crops,
    with --wgan and without, G in fp32 and in mixed precision;
  * the SRGAN step (RRDB_net nb 1, Discriminator_VGG_128 with BatchNorm), batch 16, HR 128, gan_type wgan-gp and vanilla.
Warm-up first; the card name and power limit are read in the same run.  One JSON line.  Random-init weights.

  python tools/time_wgan_gp.py [--iters 20] [--warmup 5]"""
import argparse
import contextlib
import io
import json
import os
import subprocess
import sys
import warnings

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
os.environ.setdefault('DASR_B200_ALLOW_RANDOM_VGG', '1')

import torch  # noqa: E402


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:      # noqa: BLE001
        q = 'unknown (%s)' % e
    return q


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def dsn(wgan, prec, iters, warmup):
    from dasr_b200.dsn.loss import GeneratorLoss
    from dasr_b200.dsn.model import De_resnet, Discriminator
    from dasr_b200.dsn.train import train_iteration
    from oracle import srn_oracle as O
    dev = torch.device('cuda', 0)
    with warnings.catch_warnings(), contextlib.redirect_stdout(io.StringIO()):
        warnings.simplefilter('ignore')
        mg = De_resnet(8, 4).to(dev)
        mg.precision = prec
        md = Discriminator(kernel_size=5, D_arch='FSD', norm_layer='Instance', filter_type='wavelet', cs='cat', wgan=wgan).to(dev)
        gl = GeneratorLoss(per_type='VGG', filter='wavelet', kernel_size=5, w_col=1, w_tex=0.005, w_per=0.01, wgan=wgan).to(dev)
    og = torch.optim.Adam(mg.parameters(), lr=1e-4, betas=[0.5, 0.999])
    od = torch.optim.Adam(md.parameters(), lr=1e-4, betas=[0.5, 0.999])
    inp, bic, dis = (O.synth_image(s, i).to(dev) for s, i in (((8, 3, 256, 256), 700), ((8, 3, 64, 64), 800), ((8, 3, 64, 64), 900)))
    return timed(lambda: train_iteration(mg, md, gl, og, od, inp, bic, dis, log=False), iters, warmup)


def srgan(gan_type, iters, warmup):
    from dasr_b200.srn.models import create_model
    from dasr_b200.srn.options.options import dict_to_nonedict
    from helpers import make_opt
    from oracle import srn_oracle as O
    opt = dict(make_opt(True, 'srgan', 1, gpu=True))
    opt['network_D'] = dict(opt['network_D'], which_model_D='discriminator_vgg_128', norm_type='batch', nf=64, in_nc=3)
    opt['train'] = dict(opt['train'], gan_type=gan_type, gp_weigth=10, gan_weight=5e-3, feature_weight=0, pixel_weight=1e-2)
    with contextlib.redirect_stdout(io.StringIO()):
        model = create_model(dict_to_nonedict(opt))
    data = {'LR': O.synth_image((16, 3, 32, 32), 901).cuda(), 'HR': O.synth_image((16, 3, 128, 128), 902).cuda()}

    def step():
        model.feed_data(data, True)
        model.optimize_parameters(1)
    return timed(step, iters, warmup)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('time_wgan_gp.py measures on the GPU; no CUDA device found')
    out = {'card': card()}
    for prec in ('fp32', 'bf16'):
        for wgan in (False, True):
            out['dsn_b8_crop256_%s_%s_ms' % (prec, 'wgan' if wgan else 'gan')] = round(dsn(wgan, prec, a.iters, a.warmup), 2)
    for gt in ('vanilla', 'wgan-gp'):
        out['srgan_vgg128_b16_hr128_%s_ms' % gt] = round(srgan(gt, a.iters, a.warmup), 2)
    out['card_after'] = card()
    print(json.dumps(out))


if __name__ == '__main__':
    main()
