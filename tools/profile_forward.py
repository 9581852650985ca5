"""One RRDBNet-23 bf16 forward (BASELINE configs[1] shape) between cudaProfilerStart/Stop, for ncu:
   ncu --profile-from-start off --metrics gpu__time_duration.sum,dram__bytes_read.sum,dram__bytes_write.sum \
       --clock-control none --csv --log-file profiling/launches.csv python tools/profile_forward.py
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from dasr_b200.srn.models.modules.architecture import RRDBNet  # noqa: E402
from oracle import srn_oracle as O  # noqa: E402

nb = int(os.environ.get('NB', 23))
batch = int(os.environ.get('BATCH', 16))
net = RRDBNet(3, 3, 64, nb)
net.load_state_dict(O.synth_state_dict(O.rrdbnet_shapes(nb=nb), 1, 0.1))
net.cuda().eval()
net.precision = os.environ.get('PREC', 'bf16')
x = O.synth_image((batch, 3, 256, 256), 100).cuda()
with torch.no_grad():
    net(x)
    torch.cuda.synchronize()
    torch.cuda.profiler.start()
    net(x)
    torch.cuda.synchronize()
    torch.cuda.profiler.stop()
print('done')
