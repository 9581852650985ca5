"""DASR_Adaptive_Model — the test path of the adaptive-weight generators (reference: codes/SRN/models/DASR_Adaptive_model.py).

The map network net_patchD (the FS patch discriminator of a DSN checkpoint) turns the LR input into a per-pixel weight map,
and netG (RRDBNet_Residual_conv_concat / RRDBNet_Residual_conv) super-resolves the input under that map.  Like the
reference, net_patchD is never switched to eval(): its BatchNorm layers normalise with the statistics of the current batch
and update their running statistics on every test() call.

Training is not built: the shipped train config has no `FS` block, so the reference cannot construct it either
(DASR_Adaptive_model.py:61), and the backward through the weight-map epilogue does not exist.
"""
import logging
from collections import OrderedDict

import torch
import torch.nn as nn

from . import networks
from .base_model import BaseModel
from .modules.architecture import FilterHigh

logger = logging.getLogger('base')


class DASR_Adaptive_Model(BaseModel):
    def __init__(self, opt):
        super().__init__(opt)
        if self.is_train:
            raise NotImplementedError(
                'DASR_Adaptive_Model training is not built: the shipped train_DASR_Adaptive.json has no `FS` block (the '
                'reference fails on opt["FS"]["fs"] as well), and the backward of the adaptive generators is not built')
        self.chop = opt['chop']
        self.scale = opt['scale']
        self.val_lpips = opt['val_lpips']
        self.use_domain_distance_map = opt['use_domain_distance_map']
        self.netG = networks.define_G(opt).to(self.device)
        self.net_patchD = networks.define_patchD(opt).to(self.device)
        self.load()
        fs = opt['FS'] or {}
        self.filter_high = FilterHigh(kernel_size=fs.get('fs_kernel_size') or 5, gaussian=True).to(self.device)
        self.print_network()
        self.fake_H = None
        if self.val_lpips:      # DASR_Adaptive_model.py:173-174
            from dasr_b200.lpips import PerceptualLoss as val_lpips
            self.cri_fea_lpips = val_lpips(model='net-lin', net='alex').to(self.device)

    def feed_data(self, data, istrain):
        if istrain and 'HR' in data:
            raise NotImplementedError('DASR_Adaptive_Model: training batches are not supported (test path only)')
        self.var_L = self._to_device(data['LR'])
        self.needHR = 'HR' in data
        if self.needHR:
            self.var_H = self._to_device(data['HR'])

    def test(self, tsamples=False):
        self._log_eval_precision(self.netG)
        self.netG.eval()
        with torch.no_grad():
            self.adaptive_weights = self.net_patchD(self.var_L)
            if self.chop:
                # the reference calls forward_chop(var_L, scale, netG) without the map, which fails inside netG
                raise NotImplementedError('chop is not supported for DASR_Adaptive_Model (the reference raises a TypeError)')
            self.fake_H = self.netG(self.var_L, self.adaptive_weights)
            if not tsamples and self.val_lpips:
                from .SR_model import _val_lpips
                self.LPIPS = _val_lpips(self.cri_fea_lpips, self.fake_H, self.var_H, self.device)
        self.netG.train()

    def get_current_log(self):
        return OrderedDict()

    def get_current_visuals(self, need_HR=True, tsamples=False):
        out = OrderedDict()
        out['LR'] = self.var_L.detach()[0].float().cpu()
        if tsamples:
            out['hf'] = self.filter_high(self.fake_H).float().cpu()
            out['gt_hf'] = self.filter_high(self.var_H).float().cpu()
            out['HR'] = self.var_H.detach()[0].float().cpu()
            out['HR_hf'] = self.filter_high(self.var_H).detach().float().cpu()
            out['SR'] = self.fake_H.detach().float().cpu()
        else:
            out['SR'] = self.fake_H.detach()[0].float().cpu()
            if self.val_lpips:
                out['LPIPS'] = self.LPIPS.detach().float().cpu()
            if self.needHR:
                out['HR'] = self.var_H.detach()[0].float().cpu()
        if self.use_domain_distance_map:
            out['adaptive_weights'] = torch.mean(self.adaptive_weights.float().cpu())
        return out

    def print_network(self):
        self._log_network(self.netG, 'G')

    def load(self):
        path = self.opt['path']
        if path['pretrain_model_G'] is not None:
            logger.info('Loading pretrained model for G [{:s}] ...'.format(path['pretrain_model_G']))
            self.load_network(path['pretrain_model_G'], self.netG)
        if path['Patch_Discriminator'] is not None:
            # a DSN checkpoint (codes/DSN/train.py:368): the discriminator's weights under 'models_d_state_dict'
            logger.info('Loading pretrained model for Patch_Discriminator [{:s}] ...'.format(path['Patch_Discriminator']))
            checkpoint = torch.load(path['Patch_Discriminator'], map_location='cpu')
            if isinstance(self.net_patchD, nn.DataParallel):
                self.net_patchD = self.net_patchD.module
            self.net_patchD.load_state_dict(checkpoint['models_d_state_dict'])

    def save(self, iter_step):
        self.save_network(self.netG, 'G', iter_step)

