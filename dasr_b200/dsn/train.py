"""The training iteration of codes/DSN/train.py:204-264 as a function (the reference has it inline
in a script).  Both gradients are taken with the D weights of the forward pass, then both Adam steps are applied
(train.py steps D before back-propagating the G loss through it, which PyTorch >= 1.5 rejects; see
oracle/dsn_oracle.py)."""
from collections import OrderedDict

import torch

from . import loss as dsn_loss


def train_iteration(model_g, model_d, g_loss_module, optimizer_g, optimizer_d, input_img, bicubic_img, disc_img,
                    grad_sync=None, log=True):
    """One DeResnet iteration (no ragan / wgan, disc_freq = gen_freq = 1).  grad_sync: optional callable run
    between the backward passes and the optimiser steps (data-parallel all-reduce of both gradient sets)."""
    import os
    from dasr_b200 import ops
    mixed = (getattr(model_g, 'precision', None) or os.environ.get('DASR_B200_TRAIN_PRECISION', 'fp32')) == 'bf16'
    # mixed precision: the fp32 layers (stride-2 tail, 5x5 FS discriminator) take tf32 tensor-core math
    with ops.f32_math(os.environ.get('DASR_B200_SIDE_MATH', 'tf32') if mixed else 'default'):
        return _train_iteration(model_g, model_d, g_loss_module, optimizer_g, optimizer_d, input_img, bicubic_img, disc_img,
                                grad_sync, log)


def _train_iteration(model_g, model_d, g_loss_module, optimizer_g, optimizer_d, input_img, bicubic_img, disc_img, grad_sync, log):
    fake_img = model_g(input_img)                                                   # :218
    real_tex = model_d(disc_img)                                                    # :226
    fake_tex = model_d(fake_img)                                                    # :227
    pd = [p for p in model_d.parameters() if p.requires_grad]
    pg = [p for p in model_g.parameters() if p.requires_grad]
    d_tex_loss = dsn_loss.discriminator_loss(real_tex, fake_tex)                    # :242
    g_d = torch.autograd.grad(d_tex_loss, pd, retain_graph=True)
    g_loss = g_loss_module(fake_tex, fake_img, bicubic_img)                         # :257
    g_g = torch.autograd.grad(g_loss, pg)
    for p, g in zip(pd, g_d):
        p.grad = g
    for p, g in zip(pg, g_g):
        p.grad = g
    if grad_sync is not None:
        grad_sync()
    optimizer_d.step()                                                              # :244
    optimizer_g.step()                                                              # :264
    if not log:
        return None
    return OrderedDict(d_tex_loss=float(d_tex_loss), g_loss=float(g_loss), perceptual_loss=float(g_loss_module.last_per_loss),
                       color_loss=float(g_loss_module.last_col_loss), g_tex_loss=float(g_loss_module.last_tex_loss),
                       real=float(real_tex.mean()), fake=float(fake_tex.mean())), fake_img.detach()
