"""Generate tests/golden/lpips_alex.pt from the UNMODIFIED reference LPIPS network
(<DASR checkout>/codes/PerceptualSimilarity/models/networks_basic.py: PNetLin(pnet_type='alex')) on CPU.
The AlexNet trunk gets synthetic weights (no torchvision checkpoint offline); the five linear layers are the reference's
own weights/v0.1/alex.pth (stored in the fixture: 1152 floats).  Test infrastructure only."""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF = os.path.join(os.environ.get('DASR_REFERENCE', 'DASR'), 'codes')   # a ShuhangGu/DASR checkout
sys.path.insert(0, os.path.join(HERE, 'ref_stubs'))
sys.path.insert(0, REF)
sys.path.insert(0, ROOT)

import torch  # noqa: E402
import torchvision  # noqa: E402

_orig = torchvision.models.alexnet
torchvision.models.alexnet = lambda pretrained=True, **k: _orig(weights=None)

from PerceptualSimilarity.models import networks_basic as nb  # noqa: E402

from oracle import lpips_oracle as LP  # noqa: E402
from oracle import srn_oracle as O  # noqa: E402

torch.set_num_threads(8)
net = nb.PNetLin(pnet_rand=True, pnet_tune=False, pnet_type='alex', use_dropout=True, spatial=False, version='0.1', lpips=True)
lin_sd = torch.load(os.path.join(REF, 'PerceptualSimilarity/models/weights/v0.1/alex.pth'), map_location='cpu')
net.load_state_dict(lin_sd, strict=False)
sd = O.synth_state_dict(LP.alex_shapes(), seed=81, gain=1.0)
own = [k for k in net.state_dict().keys() if k.startswith('net.slice')]
assert own == list(sd.keys()), (own, list(sd.keys()))
net.load_state_dict(sd, strict=False)
net.eval()
for p in net.parameters():
    p.requires_grad_(False)
pred = O.synth_image((2, 3, 64, 64), 82).requires_grad_(True)
target = O.synth_image((2, 3, 64, 64), 83)
val = net.forward(2 * target - 1, 2 * pred - 1)            # PerceptualLoss.forward(pred, target, normalize=True) -> model.forward(target, pred)
val.mean().backward()
out = dict(w_seed=81, pred_seed=82, target_seed=83, shape=(2, 3, 64, 64), value=val.detach(), dpred=pred.grad.clone(),
           lins=[lin_sd['lin%d.model.1.weight' % i].clone() for i in range(5)])
path = os.path.join(ROOT, 'tests', 'golden', 'lpips_alex.pt')
torch.save(out, path)
print('lpips_alex.pt %.1f KB  value %s' % (os.path.getsize(path) / 1024, val.flatten().tolist()))
