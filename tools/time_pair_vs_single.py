"""dasr_conv_tc2 launch shapes on the CTA pair against one CTA per tile, across grid sizes.

For every conv launch that dasr_conv_tc2 may run on one CTA per tile (dense-block launches 2-4 of schedule 3, LR_conv,
HR_conv0, the DSN De_resnet trunk convs and their dgrads, the 64-channel VGG19 convs and their dgrads), times
ops.conv_tc(..., pair=False) (dasr_conv_tc: one CTA per tile) and ops.conv_tc(..., pair=True) (dasr_conv_tc2) with CUDA
events at 1, 2, 4, 8, 16 and 62 waves of pixel tiles (one wave = one tile per SM) and at the size the benchmark runs.
Dense-block launch 5 is timed too: its filters leave no room for one CTA per tile, so it stays on the pair.  For each
dasr_conv_tc2 point it also records, from the kernel name in a torch.profiler trace, whether the launch ran the pair's
half Cout tile ('pair') or the whole tile on one CTA ('single'); None when the profiler returned no kernel record, which
the later sessions of this long process often do (tests/test_gpu_conv_tc_single_feed.py checks the sides in fresh
interpreters).

    python tools/time_pair_vs_single.py --out /tmp/pair_vs_single.json

Prints the card name and its power limit, then one line per point; writes everything as JSON to --out."""
import argparse
import json
import os
import re
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from dasr_b200 import ops  # noqa: E402
from dasr_b200.ops import View  # noqa: E402

WAVES = (1, 2, 4, 8, 16, 62)
GC, CS = 32, 256          # dense-block growth channels, the [x | x1..x4 | conv5 partial sums] buffer of nf = 64


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        q = torch.cuda.get_device_name(0) + ', power limit not reported'
    return q


def _grid_shape(sms):
    """(H, W) of an image with exactly `sms` pixel tiles of 16 x 8, as square as the divisors of sms allow"""
    a = max(d for d in range(1, int(sms ** 0.5) + 1) if sms % d == 0)
    return 16 * a, 8 * (sms // a)


def _rnd(shape, dt, g):
    return (torch.randn(shape, generator=g) * 0.5).to(dt).cuda()


def _filters(cout, cin, kind, dt, g):
    w = torch.randn((cin, cout, 3, 3) if kind == ops.TC_DGRAD else (cout, cin, 3, 3), generator=g) * 0.05
    return ops.pack_filter_tc(w.cuda(), kind, dt)


# name -> (builder(N, H, W, dt, g) -> (inp, w, bias, out, kwargs), bench-size (N, H, W))
def _rdb(j):
    def build(N, H, W, dt, g):
        b = _rnd((N, H, W, CS), dt, g)
        chunks = {2: [64], 3: [64, 96], 4: [128], 5: [64, 96, 128, 160]}[j]
        cout = {2: 32, 3: 64, 4: 32, 5: 64}[j]
        w = _filters(cout, 32 * len(chunks), ops.TC_FPROP, dt, g)
        bias = torch.randn(cout, generator=g).cuda()
        if j < 5:
            o = View(b, cout, 64 + (j - 1) * GC)
            return b, w, bias, o, dict(act=ops.ACT_LRELU, slope=0.2, act_cols=GC, pre=o, chunks=chunks, tile_rev=j % 2 == 1)
        dst = _rnd((N, H, W, 64), dt, g)
        return b, w, bias, dst, dict(pre=View(b, 64, 192), chunks=chunks, tile_rev=True, alpha=0.2,
                                     res1=_rnd((N, H, W, 64), dt, g), beta1=1.0)
    return build


def _plain(cin, cout, kind=ops.TC_FPROP, act=ops.ACT_NONE, res1=False):
    def build(N, H, W, dt, g):
        x = _rnd((N, H, W, cin), dt, g)
        w = _filters(cout, cin, kind, dt, g)
        bias = torch.randn(cout, generator=g).cuda() if kind == ops.TC_FPROP else None
        o = torch.empty((N, H, W, cout), dtype=dt, device='cuda')
        kw = dict(kind=kind, act=act, slope=0.2)
        if res1:
            kw.update(res1=_rnd((N, H, W, cout), dt, g), beta1=1.0)
        return x, w, bias, o, kw
    return build


SHAPES = {
    'rdb_launch2 (32 -> 32, pre)': (_rdb(2), (16, 256, 256)),
    'rdb_launch3 (64 -> 64, pre)': (_rdb(3), (16, 256, 256)),
    'rdb_launch4 (32 -> 32, pre)': (_rdb(4), (16, 256, 256)),
    'rdb_launch5 (128 -> 64, pre, res1)': (_rdb(5), (16, 256, 256)),
    'LR_conv (64 -> 64, res1)': (_plain(64, 64, res1=True), (16, 256, 256)),
    'HR_conv0 (64 -> 64, lrelu)': (_plain(64, 64, act=ops.ACT_LRELU), (16, 1024, 1024)),
    'DSN conv1 (64 -> 64)': (_plain(64, 64), (8, 256, 256)),
    'DSN conv2 (64 -> 64, res1)': (_plain(64, 64, res1=True), (8, 256, 256)),
    'DSN dgrad conv2 (64 -> 64)': (_plain(64, 64, ops.TC_DGRAD), (8, 256, 256)),
    'DSN dgrad conv1 (64 -> 64, res1)': (_plain(64, 64, ops.TC_DGRAD, res1=True), (8, 256, 256)),
    'VGG conv1_1 (32 -> 64, relu)': (_plain(32, 64, act=ops.ACT_RELU), (32, 128, 128)),
    'VGG conv1_2 (64 -> 64, relu)': (_plain(64, 64, act=ops.ACT_RELU), (32, 128, 128)),
    'VGG dgrad conv1_2 (64 -> 64)': (_plain(64, 64, ops.TC_DGRAD), (32, 128, 128)),
    'VGG dgrad conv1_1 (64 -> 32)': (_plain(64, 32, ops.TC_DGRAD), (32, 128, 128)),
}


def _time(fn, target_ms=40.0):
    """median µs per call of three windows of about target_ms each"""
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(3):
        fn()
    e1.record()
    e1.synchronize()
    reps = max(3, min(2000, int(target_ms / max(e0.elapsed_time(e1) / 3, 1e-3))))
    ts = []
    for _ in range(3):
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        e1.synchronize()
        ts.append(e0.elapsed_time(e1) * 1e3 / reps)
    return sorted(ts)[1]


def _side(fn, nt):
    """'single' or 'pair' from the Cout tile of the conv_tc_kernel instantiation the call ran (None: no kernel record)"""
    from torch.profiler import ProfilerActivity, profile
    for _ in range(3):          # a profiler session can come back without any kernel record: trace again
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        for e in prof.events():
            m = re.search(r'conv_tc_kernel<([^>]*)>', e.name)
            if m:
                a = [s.strip() for s in m.group(1).split(',')]
                ntk = int(a[4]) if len(a) > 4 else 0
                return 'single' if ntk == nt else 'pair' if ntk == nt // 2 else 'other (NT=%d)' % ntk
    return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None, help='JSON file to write')
    ap.add_argument('--dtype', default='bf16', choices=('bf16', 'fp16'))
    ap.add_argument('--only', default=None, help='substring of the shape names to run')
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'needs a GPU'
    dt = torch.bfloat16 if args.dtype == 'bf16' else torch.float16
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    h1, w1 = _grid_shape(sms)
    info = card()
    print('card: %s; %d SMs; %s' % (info, sms, args.dtype), flush=True)
    res = {'card': info, 'sms': sms, 'dtype': args.dtype, 'waves': list(WAVES), 'points': []}
    g = torch.Generator().manual_seed(0)
    for name, (build, bench) in SHAPES.items():
        if args.only and args.only not in name:
            continue
        sizes = [(w, (w, h1, w1)) for w in WAVES] + [('bench', bench)]
        for label, (N, H, W) in sizes:
            inp, w, bias, out, kw = build(N, H, W, dt, g)
            tiles = N * -(-H // 16) * -(-W // 8)
            nt = ops.as_view(out).c
            one = lambda: ops.conv_tc(inp, w, bias, out, pair=False, **kw)
            two = lambda: ops.conv_tc(inp, w, bias, out, pair=True, **kw)
            t1, t2 = [], []
            for _ in range(2):              # alternate the arms: other work on the host moves both alike
                t1.append(_time(one))
                t2.append(_time(two))
            side = _side(two, nt)
            pt = dict(shape=name, size=label, N=N, H=H, W=W, tiles=tiles, waves=round(tiles / sms, 2),
                      us_single=round(min(t1), 2), us_pair=round(min(t2), 2), pair_true_ran=side)
            res['points'].append(pt)
            print('%-36s %6s %7d tiles %7.2f waves  one CTA %9.1f us  pair=True %9.1f us  (%s)  one/pair %.3f' % (
                name, label, tiles, tiles / sms, pt['us_single'], pt['us_pair'], side, pt['us_single'] / pt['us_pair']),
                flush=True)
            del inp, w, bias, out, kw
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
