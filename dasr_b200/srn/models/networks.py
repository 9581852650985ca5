"""Network factories + weight init (reference: codes/SRN/models/networks.py).

define_G / define_D / define_pairD / define_F keep their names, option keys and error behaviour for the
networks the SRN hot path uses; other ``which_model_*`` values raise NotImplementedError exactly like an
unknown name does in the reference.  ``gpu_ids`` truthy still wraps the net in nn.DataParallel (callers
unwrap with isinstance checks, base_model.py:44,53,61) — with ONE device it is a pass-through; multi-GPU
runs use one process per GPU + dasr_b200.dp instead.
"""
import functools
import logging

import torch
import torch.nn as nn
from torch.nn import init

from .modules import architecture as arch

logger = logging.getLogger('base')


def weights_init_normal(m, std=0.02):
    name = m.__class__.__name__
    if name.find('Conv') != -1 or name.find('Linear') != -1:
        init.normal_(m.weight.data, 0.0, std)
        if m.bias is not None:
            m.bias.data.zero_()
    elif name.find('BatchNorm2d') != -1:
        init.normal_(m.weight.data, 1.0, std)
        init.constant_(m.bias.data, 0.0)


def weights_init_kaiming(m, scale=1):
    name = m.__class__.__name__
    if name.find('Conv') != -1 or name.find('Linear') != -1:
        init.kaiming_normal_(m.weight.data, a=0, mode='fan_in')
        m.weight.data *= scale
        if m.bias is not None:
            m.bias.data.zero_()
    elif name.find('BatchNorm2d') != -1:
        init.constant_(m.weight.data, 1.0)
        init.constant_(m.bias.data, 0.0)


def weights_init_orthogonal(m):
    name = m.__class__.__name__
    if name.find('Conv') != -1 or name.find('Linear') != -1:
        init.orthogonal_(m.weight.data, gain=1)
        if m.bias is not None:
            m.bias.data.zero_()
    elif name.find('BatchNorm2d') != -1:
        init.constant_(m.weight.data, 1.0)
        init.constant_(m.bias.data, 0.0)


def init_weights(net, init_type='kaiming', scale=1, std=0.02):
    logger.info('Initialization method [{:s}]'.format(init_type))
    if init_type == 'normal':
        net.apply(functools.partial(weights_init_normal, std=std))
    elif init_type == 'kaiming':
        net.apply(functools.partial(weights_init_kaiming, scale=scale))
    elif init_type == 'orthogonal':
        net.apply(weights_init_orthogonal)
    else:
        raise NotImplementedError('initialization method [{:s}] not implemented'.format(init_type))


def _wrap(net, gpu_ids):
    if gpu_ids:
        assert torch.cuda.is_available()
        if len(gpu_ids) > 1:
            raise NotImplementedError('dasr_b200 scales with one process per GPU (torchrun + dasr_b200.dp), '
                                      'not nn.DataParallel over gpu_ids=%s' % (gpu_ids,))
        net = nn.DataParallel(net, device_ids=[torch.cuda.current_device()])
    return net


def define_G(opt):
    opt_net = opt['network_G']
    which = opt_net['which_model_G']
    if which in ('RRDB_net', 'RRDB_mask'):
        netG = arch.RRDBNet(in_nc=opt_net['in_nc'], out_nc=opt_net['out_nc'], nf=opt_net['nf'], nb=opt_net['nb'],
                            gc=opt_net['gc'], upscale=opt_net['scale'], norm_type=opt_net['norm_type'],
                            act_type='leakyrelu', mode=opt_net['mode'], upsample_mode='upconv')
    elif which in ('RRDB_Residual_conv', 'RRDB_Residual_conv_concat'):
        # networks.py:131-138: only the concat variant receives ada_nb; RRDB_Residual_conv always has ONE adaptive block
        cls = arch.RRDBNet_Residual_conv_concat if which == 'RRDB_Residual_conv_concat' else arch.RRDBNet_Residual_conv
        kw = {'nb_ada': opt_net['ada_nb']} if which == 'RRDB_Residual_conv_concat' else {}
        netG = cls(in_nc=opt_net['in_nc'], out_nc=opt_net['out_nc'], nf=opt_net['nf'], nb=opt_net['nb'], gc=opt_net['gc'],
                   upscale=opt_net['scale'], norm_type=opt_net['norm_type'], act_type='leakyrelu', mode=opt_net['mode'],
                   upsample_mode='upconv', **kw)
    elif which == 'sr_resnet':      # networks.py:88-91
        netG = arch.SRResNet(in_nc=opt_net['in_nc'], out_nc=opt_net['out_nc'], nf=opt_net['nf'], nb=opt_net['nb'],
                             upscale=opt_net['scale'], norm_type=opt_net['norm_type'], act_type='relu', mode=opt_net['mode'],
                             upsample_mode='pixelshuffle')
    else:
        raise NotImplementedError('Generator model [{:s}] not recognized'.format(str(which)))
    if opt['is_train']:
        init_weights(netG, init_type='kaiming', scale=0.1)
    return _wrap(netG, opt['gpu_ids'])


def _patch_discriminator(opt_net, key):
    which = opt_net[key]
    if which == 'discriminator_patch':
        return arch.NLayerDiscriminator(opt_net['in_nc'], n_layers=opt_net['n_layers'])
    if which == 'discriminator_vgg_128':      # networks.py:156-159
        return arch.Discriminator_VGG_128(in_nc=opt_net['in_nc'], nf=opt_net['nf'])
    if which == 'discriminator_vgg_192':      # networks.py:170-172
        return arch.Discriminator_VGG_192(in_nc=opt_net['in_nc'], base_nf=opt_net['nf'], norm_type=opt_net['norm_type'],
                                          mode=opt_net['mode'], act_type=opt_net['act_type'])
    raise NotImplementedError('Discriminator model [{:s}] not recognized'.format(str(which)))


def define_D(opt):
    netD = _patch_discriminator(opt['network_D'], 'which_model_D')
    init_weights(netD, init_type='kaiming', scale=1)
    return _wrap(netD, opt['gpu_ids'])


def define_pairD(opt):
    netD = _patch_discriminator(opt['network_D'], 'which_model_pairD')
    init_weights(netD, init_type='kaiming', scale=1)
    return _wrap(netD, opt['gpu_ids'])


def define_patchD(opt):
    """FS_Discriminator (networks.py:229-245 / architecture.py:922-980): frequency-separation filter + patch
    discriminator + sigmoid; shared with the DSN drop-in (dasr_b200/dsn/model.py)."""
    from dasr_b200.dsn.model import Discriminator as FS_Discriminator
    opt_net = opt['network_patchD']
    if opt_net['which_patchD'] != 'FSD':
        raise NotImplementedError('Patch Discriminator model [{:s}] not recognized'.format(str(opt_net)))
    net = FS_Discriminator(kernel_size=opt_net['kernel_size'], D_arch='FSD', filter_type=opt_net['FS_type'],
                           norm_layer=opt_net['norm_layer'])
    init_weights(net, init_type='kaiming', scale=1)
    return _wrap(net, opt['gpu_ids'])


def define_F(opt, use_bn=False):
    gpu_ids = opt['gpu_ids']
    device = torch.device('cuda' if gpu_ids else 'cpu')
    weights = opt['path']['pretrain_model_F'] if opt['path'] else None
    netF = arch.VGGFeatureExtractor(feature_layer=49 if use_bn else 34, use_bn=use_bn, use_input_norm=True,
                                    device=device, weights=weights)
    netF = _wrap(netF, gpu_ids)
    netF.eval()
    return netF
