"""Per-stage device time of the dense-block launches of one forward (torch profiler, launch order folded modulo 5), and
of LR_conv and HR_conv0."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from torch.profiler import profile, ProfilerActivity
from oracle import srn_oracle as O
from dasr_b200 import engine
nb, shape = 23, (16, 3, 256, 256)
sd = O.synth_state_dict(O.rrdbnet_shapes(nb=nb), 1, 0.1)
params = [v.cuda() for v in sd.values()]
x = O.synth_image(shape, 2).cuda()
cache = engine._PackCache()
for _ in range(2):
    engine.rrdb_forward_bf16(x, params, nb, 4, cache)
torch.cuda.synchronize()
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    engine.rrdb_forward_bf16(x, params, nb, 4, cache)
    torch.cuda.synchronize()
ev = [e for e in prof.events() if 'conv_tc_kernel' in e.name or 'conv_tc2_kernel' in e.name]
ev.sort(key=lambda e: e.time_range.start)
durs = [e.device_time if hasattr(e, 'device_time') else e.cuda_time for e in ev]
trunk = durs[1:1 + 5 * 69]
per = [sum(trunk[j::5]) / 69 for j in range(5)]
print('stage us:', ' '.join('%.0f' % t for t in per), '| RDB %.0f us | trunk %.1f ms | other convs %.1f ms' %
      (sum(per), sum(trunk) / 1e3, (sum(durs) - sum(trunk)) / 1e3), flush=True)
# after the trunk: LR_conv, the two upconvs, HR_conv0, HR_conv1
print('LR_conv %.0f us | HR_conv0 %.0f us' % (durs[1 + 5 * 69], durs[1 + 5 * 69 + 3]), flush=True)
