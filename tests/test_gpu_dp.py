"""Data-parallel equivalence on real GPUs (SURVEY §4 iv, §8e): a 2-rank DASR_Model step with B_local crops per rank
(torchrun, NCCL) must produce the gradients and post-Adam weights of a single-GPU step on the concatenated batch.
Needs 2 GPUs; skipped on a single-GPU machine."""
import os
import subprocess
import sys

import pytest
import torch

from oracle import srn_oracle as O

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

WORKER = r'''
import os, sys, torch, torch.distributed as dist
sys.path.insert(0, %(root)r); sys.path.insert(0, os.path.join(%(root)r, 'tests'))
os.environ['DASR_B200_ALLOW_RANDOM_VGG'] = '1'
from oracle import srn_oracle as O
from helpers import make_opt, unwrap
rank = int(os.environ['RANK']); world = int(os.environ['WORLD_SIZE'])
torch.cuda.set_device(int(os.environ['LOCAL_RANK']))
dist.init_process_group('nccl', device_id=torch.device('cuda', int(os.environ['LOCAL_RANK'])))
from dasr_b200.srn.models import create_model
prec, out, BL = sys.argv[1], sys.argv[2], int(sys.argv[3])
os.environ['DASR_B200_TRAIN_PRECISION'] = prec
torch.manual_seed(1000 + rank)                      # every rank draws its own init; rank 0's weights are broadcast
model = create_model(make_opt(True, 'DASR', 1, 'wavelet'))
if rank == 0:                                       # the weights the single-GPU run will use
    unwrap(model.netG).load_state_dict(O.synth_state_dict(O.rrdbnet_shapes(nb=1), 11, 0.3))
    unwrap(model.netD_target).load_state_dict(O.synth_state_dict(O.nlayer_d_shapes(9, 64, 2), 12, 1.0))
    unwrap(model.netF).load_state_dict(O.synth_state_dict(O.vgg19_shapes(34), 13, 1.0), strict=False)
from dasr_b200 import dp
for net in (model.netG, model.netD_target, model.netF):
    dp.broadcast_module(net)                        # (GradBucket broadcast G and D at construction; do it again after the load)
B, h = BL * world, 8
full = {'LR_real': O.synth_image((B, 3, h, h), 21), 'LR_fake': O.synth_image((B, 3, h, h), 22), 'HR': O.synth_image((B, 3, 4 * h, 4 * h), 23),
        'HR_unpair': O.synth_image((B, 3, 4 * h, 4 * h), 24), 'fake_w': O.synth_image((B, 1, h, h), 25)}
mine = {k: v[rank * BL:(rank + 1) * BL].contiguous() for k, v in full.items()}
for step in (1, 2):
    model.feed_data(mine, True)
    model.optimize_parameters(step)
assert model.grad_sync.active
if prec == 'bf16':                                  # G's gradients are written straight into the bucket: only D's 6 tensors are copied
    assert model.grad_sync.last_copies <= 8, model.grad_sync.last_copies
torch.cuda.synchronize()
if rank == 0:
    torch.save({'G': {k: v.cpu() for k, v in unwrap(model.netG).state_dict().items()},
                'D': {k: v.cpu() for k, v in unwrap(model.netD_target).state_dict().items()},
                'gG': {k: p.grad.cpu().clone() for k, p in unwrap(model.netG).named_parameters()},
                'copies': model.grad_sync.last_copies}, out)
dist.barrier()
dist.destroy_process_group()
'''


@pytest.mark.parametrize('prec', ['fp32', 'bf16'])
def test_dp2_step_equals_single_gpu_step_on_the_concatenated_batch(tmp_path, prec, monkeypatch):
    if torch.cuda.device_count() < 2:
        pytest.skip('needs 2 GPUs')
    from dasr_b200.srn.models import create_model
    from helpers import make_opt, unwrap
    BL = 2
    script = tmp_path / 'w.py'
    script.write_text(WORKER % {'root': ROOT})
    out = tmp_path / 'dp.pt'
    port = str(29600 + os.getpid() % 300)
    r = subprocess.run([sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node', '2', '--master-addr', '127.0.0.1',
                        '--master-port', port, str(script), prec, str(out), str(BL)], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, (r.stdout[-2000:], r.stderr[-4000:])
    got = torch.load(str(out))
    # single GPU, batch = 2 * BL
    monkeypatch.setenv('DASR_B200_TRAIN_PRECISION', prec)
    model = create_model(make_opt(True, 'DASR', 1, 'wavelet'))
    unwrap(model.netG).load_state_dict(O.synth_state_dict(O.rrdbnet_shapes(nb=1), 11, 0.3))
    unwrap(model.netD_target).load_state_dict(O.synth_state_dict(O.nlayer_d_shapes(9, 64, 2), 12, 1.0))
    unwrap(model.netF).load_state_dict(O.synth_state_dict(O.vgg19_shapes(34), 13, 1.0), strict=False)
    B, h = 2 * BL, 8
    # the reference pairing: sample i of LR_fake goes with sample i of HR / fake_w; each rank held a contiguous slice
    full = {'LR_real': O.synth_image((B, 3, h, h), 21), 'LR_fake': O.synth_image((B, 3, h, h), 22), 'HR': O.synth_image((B, 3, 4 * h, 4 * h), 23),
            'HR_unpair': O.synth_image((B, 3, 4 * h, 4 * h), 24), 'fake_w': O.synth_image((B, 1, h, h), 25)}
    for step in (1, 2):
        model.feed_data(full, True)
        model.optimize_parameters(step)
    tol = 2e-4 if prec == 'fp32' else 2e-2
    worst = 0.0
    for k, p in unwrap(model.netG).named_parameters():
        a, b = got['gG'][k], p.grad.cpu()
        err = float((a - b).abs().max() / b.abs().max().clamp_min(1e-20))
        worst = max(worst, err)
        assert err < tol, (k, err)
    # post-Adam weights: the first Adam steps move every weight by ~lr * sign(gradient), so the UPDATES are compared
    # (fraction of elements whose update has the same sign; differences only where the gradient is ~0)
    init = {'G': O.synth_state_dict(O.rrdbnet_shapes(nb=1), 11, 0.3), 'D': O.synth_state_dict(O.nlayer_d_shapes(9, 64, 2), 12, 1.0)}
    agree_min = 1.0
    for name, net in (('G', model.netG), ('D', model.netD_target)):
        for k, v in unwrap(net).state_dict().items():
            a, b = got[name][k] - init[name][k], v.cpu() - init[name][k]
            m = (a != 0) & (b != 0)
            if int(m.sum()) < 16:
                continue
            agree_min = min(agree_min, float((torch.sign(a[m]) == torch.sign(b[m])).float().mean()))
    assert agree_min > (0.99 if prec == 'fp32' else 0.9), agree_min
    print('dp2 vs single (%s): worst relative gradient difference %.2e, update sign agreement >= %.4f, gather copies per step %d' % (prec, worst, agree_min, got['copies']))
