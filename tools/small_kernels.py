"""Workload for the per-kernel ncu pass over everything that is NOT the wgmma conv (VERDICT r1 weak #8): one DASR train step
in the fp32 parity mode and one in the mixed-precision mode (configs[2], no CUDA graphs), one DSN iteration in each mode
(configs[4]), an LPIPS loss forward / backward, a BatchNorm discriminator forward / backward, a domain-distance map.

  DASR_B200_GRAPH=0 ncu --metrics gpu__time_duration.sum,dram__bytes_read.sum,dram__bytes_write.sum \\
      --clock-control none --csv --log-file profiling/small_kernels.csv python tools/small_kernels.py
  python tools/summarize_small_kernels.py profiling/small_kernels.csv
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ['DASR_B200_GRAPH'] = '0'
os.environ.setdefault('DASR_B200_ALLOW_RANDOM_VGG', '1')
import torch
import bench


class A:
    train_steps = 1


dev = torch.device('cuda', 0)
torch.cuda.set_device(0)
sync = torch.cuda.synchronize
ident = lambda ms: ms
for prec in ('fp32', 'bf16'):
    bench.bench_train(A, dev, 0, 1, sync, ident, prec)
    bench.bench_dsn(A, dev, 0, 1, sync, ident, prec)

# LPIPS (AlexNet net-lin) loss forward + backward on 16 x 3 x 128 x 128 crops
from dasr_b200.lpips import PerceptualLoss
cri = PerceptualLoss(model='net-lin', net='alex', use_gpu=True).cuda()
a = torch.rand(16, 3, 128, 128, device=dev, requires_grad=True)
b = torch.rand(16, 3, 128, 128, device=dev)
cri(a, b).mean().backward()

# BatchNorm discriminator (SRGAN / ESRGAN configs): forward + backward, batch 16 x 3 x 128 x 128
from dasr_b200.srn.models.modules.architecture import Discriminator_VGG_128
d = Discriminator_VGG_128(3, 64).cuda().train()
x = torch.rand(16, 3, 128, 128, device=dev, requires_grad=True)
d(x).sum().backward()

# domain-distance map of a 1024 x 1024 image (23 x 23 receptive field, jump 4 — the DSN FS discriminator on a 2x DWT band)
import numpy as np
from dasr_b200.dsn import receptive_cal as rc
convnet = [[5, 1, 2], [5, 1, 2], [5, 1, 2], [1, 1, 0]]
img = torch.zeros(1, 3, 2048, 2048)
D_out = torch.rand(1, 1, 1024, 1024)
rc.domain_distance_map_handler(img, D_out, convnet, 'wavelet')
sync()
print('done')
