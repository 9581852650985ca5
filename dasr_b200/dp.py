"""Data-parallel gradient exchange for the SRN / DSN train steps (SURVEY.md §8e).

One process per GPU (torchrun), pure data parallel.  All trainable networks of a model share ONE flat fp32 gradient
bucket ``[G | D_target | D_source]`` (17.4 M elements = 69.5 MB for the shipped DASR config):

  * construction broadcasts every parameter and buffer from rank 0, so replicas start identical even when each
    process drew its own random seed (train.py picks ``random.randint`` per process when ``manual_seed`` is null);
  * a network that can write its gradients straight into a caller-supplied flat buffer (``RRDBNet.set_grad_arena`` —
    the mixed-precision backward produces ONE flat gradient tensor anyway) is handed its bucket segment: autograd then
    installs ``.grad``s that are views of the bucket and the step does no per-tensor gather copies at all; the few
    tensors of the other networks (6 for the patch discriminator) are copied into their views;
  * ``reduce_segment(i)`` starts the NCCL all-reduce (AVG) of one network's segment asynchronously — the model calls
    it for G as soon as G's backward has finished, so the 66.8 MB exchange overlaps the discriminator's forward and
    backward — and ``finish()`` reduces whatever is left and makes the compute stream wait for everything;
    ``DASR_B200_DP_OVERLAP=0`` selects the single all-reduce of the whole bucket after the last backward instead.

Per-rank data sharding is the caller's job (each rank must see its own shard of the dataset; the reference has no
distributed sampler) and checkpoints are written by rank 0 only (``BaseModel.save_network``).
"""
import os

import torch
import torch.distributed as dist
import torch.nn as nn


def _unwrap(net):
    return net.module if isinstance(net, nn.DataParallel) else net


def is_active():
    return dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1


def rank():
    return dist.get_rank() if (dist.is_available() and dist.is_initialized()) else 0


def broadcast_module(net, src=0):
    """Every parameter and buffer of `net` from rank `src` (two flat broadcasts: parameters, floating buffers).  The
    tensors are written in place under no_grad, not through .data, so their version counters move and every cache
    keyed on them (packed filters, CUDA graphs) rebuilds."""
    net = _unwrap(net)
    with torch.no_grad():
        for group in (list(net.parameters()), [b for b in net.buffers() if b.is_floating_point()]):
            if not group:
                continue
            flat = torch.cat([t.reshape(-1).float() for t in group])
            dist.broadcast(flat, src)
            o = 0
            for t in group:
                t.copy_(flat[o:o + t.numel()].view_as(t))
                o += t.numel()


class GradBucket:
    def __init__(self, nets, broadcast=True):
        """`nets`: trainable modules in bucket order (or, for backward compatibility, a flat list of parameters)."""
        nets = list(nets)
        if nets and isinstance(nets[0], torch.Tensor):
            holder = nn.Module()
            holder._plist = nn.ParameterList(nets)
            nets = [holder]
        self.nets = [_unwrap(n) for n in nets]
        self.active = is_active()
        self.overlap = os.environ.get('DASR_B200_DP_OVERLAP', '1') != '0'
        self.flat = None
        self.segs = []          # per net: (offset, numel, [params], [parameter-order views])
        self.works = []
        self.reduced = set()
        self.copies = 0
        self.last_copies = 0    # per-tensor gather copies of the last finished step (only the non-arena networks: 6 for D)
        if self.active and self.nets:
            if broadcast:
                for n in self.nets:
                    broadcast_module(n)
            self._build()

    def _build(self):
        plists = [[p for p in n.parameters() if p.requires_grad] for n in self.nets]
        total = sum(p.numel() for ps in plists for p in ps)
        dev = next(p for ps in plists for p in ps).device
        self.flat = torch.zeros(total, dtype=torch.float32, device=dev)
        self._avg = dist.get_backend() == 'nccl'
        off = 0
        for net, ps in zip(self.nets, plists):
            n = sum(p.numel() for p in ps)
            seg = self.flat[off:off + n]
            views, o = [], 0
            for p in ps:
                views.append(seg[o:o + p.numel()].view_as(p))
                o += p.numel()
            if hasattr(net, 'set_grad_arena'):
                net.set_grad_arena(seg)
            self.segs.append((off, n, ps, views))
            off += n

    def numel(self):
        return 0 if self.flat is None else self.flat.numel()

    def segment(self, i):
        off, n, _, _ = self.segs[i]
        return self.flat[off:off + n]

    def _gather(self, i):
        """Make every .grad of net i a view of its bucket segment.  Gradients that already live in the segment (the net
        wrote them there) are left alone; anything else is copied into its parameter-order view."""
        off, n, ps, views = self.segs[i]
        lo = self.flat.data_ptr() + 4 * off
        hi = lo + 4 * n
        inside = [p.grad is not None and lo <= p.grad.data_ptr() < hi for p in ps]
        if all(inside):
            return
        if any(inside):      # mixed: the in-segment gradients use the net's own layout, which the views would overwrite
            for p, ins in zip(ps, inside):
                if ins:
                    p.grad = p.grad.clone()
        for p, v in zip(ps, views):
            if p.grad is None:
                v.zero_()
            else:
                v.copy_(p.grad)
                self.copies += 1
            p.grad = v

    def _all_reduce(self, t, async_op):
        if self._avg:
            return dist.all_reduce(t, op=dist.ReduceOp.AVG, async_op=async_op)
        w = dist.all_reduce(t, op=dist.ReduceOp.SUM, async_op=async_op)      # gloo (CPU tests): no AVG
        if async_op:
            w.wait()
            w = None
        t.mul_(1.0 / dist.get_world_size())
        return w

    def reduce_segment(self, i):
        """Start the all-reduce of net i's gradients (call right after its backward).  No-op when overlap is off."""
        if not self.active or not self.overlap or i in self.reduced:
            return
        self._gather(i)
        w = self._all_reduce(self.segment(i), True)
        if w is not None:
            self.works.append(w)
        self.reduced.add(i)

    def finish(self):
        """Reduce what has not been reduced yet and make the current stream wait for every pending collective."""
        if not self.active:
            return
        todo = [i for i in range(len(self.segs)) if i not in self.reduced]
        for i in todo:
            self._gather(i)
        if len(todo) == len(self.segs):
            self._all_reduce(self.flat, False)              # ONE all-reduce of [G | D] (overlap off / nothing started)
        else:
            for i in todo:
                self._all_reduce(self.segment(i), False)
        for w in self.works:
            w.wait()
        self.works = []
        self.reduced = set()
        self.last_copies, self.copies = self.copies, 0

    def all_reduce_mean(self):
        """One synchronous exchange of everything (the round-1 entry point)."""
        self.finish()
