"""Generate tests/golden/dsn_autorepro.pt from the UNMODIFIED reference DSN modules for the option set the Auto-Reproduce
launchers use (codes/DSN/auto_reproduce_launcher_{aim2019,realsr}.sh: --filter avg_pool, default --per_type LPIPS,
--discriminator FSD, default --norm_layer Instance) plus the BatchNorm FS discriminator of the shipped checkpoint
(codes/DSN/last_iteration.tar).  Test infrastructure only.

    python oracle/gen_golden_dsn2.py

AlexNet / VGG16 are built without downloading weights; the LPIPS trunk gets synthetic weights (seed 81, as in
gen_golden_lpips.py), its linear layers are the reference's own weights/v0.1/alex.pth.
"""
import os
import sys
from collections import OrderedDict

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF = os.path.join(os.environ.get('DASR_REFERENCE', 'DASR'), 'codes')   # a ShuhangGu/DASR checkout
sys.path.insert(0, os.path.join(HERE, 'ref_stubs'))
sys.path.insert(0, REF)
sys.path.insert(0, os.path.join(REF, 'DSN'))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
import torchvision  # noqa: E402
import torchvision.models.vgg as tv_vgg  # noqa: E402

_orig_vgg16 = tv_vgg.vgg16
tv_vgg.vgg16 = lambda pretrained=True, **k: _orig_vgg16(weights=None)
_orig_alex = torchvision.models.alexnet
torchvision.models.alexnet = lambda pretrained=True, **k: _orig_alex(weights=None)

import model as ref_model  # noqa: E402  (reference DSN/model.py)
import loss as ref_loss  # noqa: E402   (reference DSN/loss.py)

from oracle import dsn_oracle as D  # noqa: E402
from oracle import lpips_oracle as LP  # noqa: E402
from oracle import srn_oracle as O  # noqa: E402

torch.set_num_threads(8)
ref_loss.FilterLow.cuda = lambda self, *a, **k: self      # harness patch: DSN/loss.py:64 moves the colour filter to CUDA unconditionally
out = {}

# ---- GeneratorLoss as the launchers build it: un-padded 5x5 box colour filter + LPIPS perceptual loss ----------------
for ft in ('avg_pool', 'gau'):
    g = ref_loss.GeneratorLoss(per_type='LPIPS', filter=ft, kernel_size=5, w_col=1, w_tex=0.006, w_per=0.01, wgan=False)
    pnet = g.perceptual_loss.loss.loss_network.model.net          # PNetLin inside DistModel
    sdA = O.synth_state_dict(LP.alex_shapes(), seed=81, gain=1.0)
    pnet.load_state_dict(sdA, strict=False)
    pnet.eval()
    tex = O.synth_image((2, 1, 16, 16), 162).requires_grad_(True)
    img = O.synth_image((2, 3, 48, 40), 163).requires_grad_(True)
    tgt = O.synth_image((2, 3, 48, 40), 164)
    total = g(tex, img, tgt)
    total.backward()
    out['gloss_' + ft] = dict(total=total.detach(), tex_loss=g.last_tex_loss.detach(), per_loss=g.last_per_loss.detach(),
                              col_loss=g.last_col_loss.detach(), dtex=tex.grad.clone(), dimg=img.grad.clone())
out['gloss_cfg'] = dict(alex_seed=81, tex_seed=162, img_seed=163, tgt_seed=164, shape=(2, 3, 48, 40), w_tex=0.006, w_per=0.01)
lin_sd = torch.load(os.path.join(REF, 'PerceptualSimilarity/models/weights/v0.1/alex.pth'), map_location='cpu')
out['lins'] = [lin_sd['lin%d.model.1.weight' % i].clone() for i in range(5)]

# ---- FS discriminator with the avg_pool high-pass (include_pad False) ------------------------------------------------
net = ref_model.Discriminator(kernel_size=5, wgan=False, highpass=True, D_arch='FSD', norm_layer='Instance', filter_type='avg_pool')
sd = O.synth_state_dict(D.fsd_shapes(3), seed=151, gain=1.0)
net.load_state_dict(sd, strict=False)
x = O.synth_image((2, 3, 24, 16), 152).requires_grad_(True)
y = net(x)
pat = O.synth(tuple(y.shape), 153)
(y * pat).sum().backward()
out['fsd_avg'] = dict(w_seed=151, x_seed=152, x_shape=(2, 3, 24, 16), pat_seed=153, out=y.detach(), dx=x.grad.clone(),
                      grad_norms=OrderedDict((k, float(p.grad.double().norm())) for k, p in net.named_parameters() if k.startswith('net.')))

# ---- BatchNorm FS discriminator (train mode: batch statistics, running-stat update; then eval mode) -------------------
net = ref_model.Discriminator(kernel_size=5, wgan=False, highpass=True, D_arch='FSD', norm_layer='Batch', filter_type='gau')
keys = [k for k in net.state_dict().keys() if k.startswith('net.')]
shapes = OrderedDict((k, tuple(net.state_dict()[k].shape)) for k in keys if 'num_batches' not in k and 'running' not in k)
sd = OrderedDict()
for i, (k, shp) in enumerate(shapes.items()):
    if len(shp) == 4:
        fan = shp[1] * shp[2] * shp[3]
        sd[k] = O.synth(shp, 171000 + i, (2.0 / fan) ** 0.5 * 3 ** 0.5)
    elif k.endswith('weight'):                                   # BatchNorm gamma around 1
        sd[k] = O.synth(shp, 171000 + i, 0.3, 1.0)
    else:
        sd[k] = O.synth(shp, 171000 + i, 0.05)
net.load_state_dict(sd, strict=False)
net.train()
x = O.synth_image((3, 3, 20, 12), 172).requires_grad_(True)
y = net(x)
pat = O.synth(tuple(y.shape), 173)
(y * pat).sum().backward()
bn = dict(shapes=shapes, x_seed=172, x_shape=(3, 3, 20, 12), pat_seed=173, out=y.detach(), dx=x.grad.clone(),
          grads=OrderedDict((k, p.grad.clone()) for k, p in net.named_parameters() if k.startswith('net.') and p.dim() == 1),
          grad_norms=OrderedDict((k, float(p.grad.double().norm())) for k, p in net.named_parameters() if k.startswith('net.')),
          running=OrderedDict((k, v.clone()) for k, v in net.state_dict().items() if 'running' in k or 'num_batches' in k))
net.eval()
with torch.no_grad():
    bn['out_eval'] = net(O.synth_image((2, 3, 20, 12), 174))
bn['x_eval_seed'] = 174
out['fsd_bn'] = bn

path = os.path.join(ROOT, 'tests', 'golden', 'dsn_autorepro.pt')
torch.save(out, path)
print('dsn_autorepro.pt %.1f KB' % (os.path.getsize(path) / 1024))
for ft in ('avg_pool', 'gau'):
    print(ft, {k: float(v) for k, v in out['gloss_' + ft].items() if v.numel() == 1})
