"""Generate tests/golden/ddm.pt from the UNMODIFIED reference <DASR checkout>/codes/DSN/receptive_cal.py (pure numpy) and
create_dataset_modified.py:14-24's handler logic.  Test infrastructure only.   python oracle/gen_golden_ddm.py"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(os.environ.get('DASR_REFERENCE', 'DASR'), 'codes', 'DSN'))   # a ShuhangGu/DASR checkout
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402
import receptive_cal as ref  # noqa: E402  (reference)
from oracle import srn_oracle as O  # noqa: E402

cases = []
# (fs_type, convnet, image hw, D_out hw as the discriminator of that configuration produces it)
for name, convnet, hw in (('fsd', [[5, 1, 2], [5, 1, 2], [5, 1, 2], [5, 1, 2]], (37, 29)),            # FSD 5x5 s1 p2 (create_dataset_modified.py:115)
                          ('nld_s1', [[4, 1, 1], [4, 1, 1], [4, 1, 1], [4, 1, 1]], (40, 33)),           # :117
                          ('nld_s2', [[4, 2, 1], [4, 2, 1], [4, 1, 1], [4, 1, 1]], (86, 56))):          # :119
    H, W = hw
    lh, lw = ref.receptive_cal(H, convnet), ref.receptive_cal(W, convnet)
    patch = O.synth_image((1, 1, lh[0], lw[0]), 500 + len(cases)).numpy()
    img = torch.zeros((1, 1, H, W))
    out = ref.getWeights(patch, img, lh, lw)
    cases.append(dict(name=name, convnet=convnet, hw=hw, patch_seed=500 + len(cases), patch_shape=(1, 1, lh[0], lw[0]),
                      layer_h=tuple(lh), layer_w=tuple(lw), ddm=torch.from_numpy(np.asarray(out, dtype=np.float64))))
    print(name, hw, 'patch', lh[0], lw[0], 'jump', lw[1], 'rf', lw[2], 'start', lh[3], lw[3], 'nan', int(np.isnan(out).sum()))
path = os.path.join(ROOT, 'tests', 'golden', 'ddm.pt')
torch.save(cases, path)
print('ddm.pt %.1f KB' % (os.path.getsize(path) / 1024))
