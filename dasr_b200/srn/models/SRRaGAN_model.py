"""SRRaGANModel (ESRGAN: relativistic average GAN) and its non-relativistic sibling SRGANModel — reference:
codes/SRN/models/SRRaGAN_model.py:18-253 and SRGAN_model.py.  `"model": "srragan"` is what the shipped train_SRGAN.json
asks for (G = RRDB_net, D = discriminator_vgg_192, VGG19 feature loss, vanilla GAN).

Same attributes / methods / log keys / checkpoint names (`{iter}_G.pth`, `{iter}_D.pth`).  Every network and loss runs on
the dasr_b200 kernels; the relativistic terms `pred - mean(other)` are arithmetic on the [N, 1] logits.  Differences, all
behaviour-preserving: while G's loss is back-propagated through D, D's filter gradients (which the reference computes and
then discards with optimizer_D.zero_grad()) are not computed; the BatchNorm running statistics of D see the same sequence
of forward passes as in the reference (2 + 2 per step, 1 + 2 for SRGAN, one more D forward with wgan-gp).

gan_type wgan-gp adds the reference's gradient penalty (SRRaGAN_model.py:156-165): gp_weigth * GradientPenaltyLoss at
interp = r * fake_H + (1 - r) * var_ref, one uniform r per sample drawn on the device, differentiated twice through
the layer-list discriminator; logged as l_d_gp."""
import logging
from collections import OrderedDict

import torch
import torch.nn as nn

from . import networks
from .base_model import BaseModel
from .DASR_model import _params_frozen
from .modules import loss as L

logger = logging.getLogger('base')


class SRRaGANModel(BaseModel):
    relativistic = True

    def __init__(self, opt):
        super().__init__(opt)
        train_opt = opt['train']
        self.val_lpips = opt['val_lpips']
        self.netG = networks.define_G(opt).to(self.device)
        if self.is_train:
            self.netD = networks.define_D(opt).to(self.device)
            self.netG.train()
            self.netD.train()
        self.load()
        # the reference builds the LPIPS validation metric unconditionally (SRRaGAN_model.py:28); here it is built when
        # its weights exist or val_lpips asks for it, otherwise test() reports nan
        self.cri_fea_lpips = None
        if self.val_lpips:
            from dasr_b200.lpips import PerceptualLoss
            self.cri_fea_lpips = PerceptualLoss(model='net-lin', net='alex').to(self.device)
        if self.is_train:
            self.cri_pix = self._criterion(train_opt['pixel_criterion']) if train_opt['pixel_weight'] > 0 else None
            self.l_pix_w = train_opt['pixel_weight']
            if self.cri_pix is None:
                logger.info('Remove pixel loss.')
            self.cri_fea = self._criterion(train_opt['feature_criterion']) if train_opt['feature_weight'] > 0 else None
            self.l_fea_w = train_opt['feature_weight']
            if self.cri_fea is None:
                logger.info('Remove feature loss.')
            else:
                self.netF = networks.define_F(opt, use_bn=False).to(self.device)
            if train_opt['gan_type'] == 'wgan-gp':
                if opt['network_D']['which_model_D'] == 'discriminator_patch':
                    raise NotImplementedError('wgan-gp needs a twice-differentiable discriminator: discriminator_vgg_128 / '
                                              '_192 (the NLayer patch discriminator has no double backward)')
                self.random_pt = torch.Tensor(1, 1, 1, 1).to(self.device)
                self.cri_gp = L.GradientPenaltyLoss(device=self.device).to(self.device)
                self.l_gp_w = train_opt['gp_weigth']
            self.cri_gan = L.GANLoss(train_opt['gan_type'], 1.0, 0.0).to(self.device)
            self.l_gan_w = train_opt['gan_weight']
            self.D_update_ratio = train_opt['D_update_ratio'] or 1
            self.D_init_iters = train_opt['D_init_iters'] or 0
            self.optimizer_G = self._adam(self.netG, train_opt['lr_G'], train_opt['weight_decay_G'], train_opt['beta1_G'])
            self.optimizer_D = self._adam(self.netD, train_opt['lr_D'], train_opt['weight_decay_D'], train_opt['beta1_D'])
            self._make_schedulers(train_opt)
            self.log_dict = OrderedDict()
        self.print_network()

    def feed_data(self, data, istrain=True):
        self.var_L = self._to_device(data['LR'])
        self.var_H = self._to_device(data['HR'])
        if istrain:
            self.var_ref = self._to_device(data['ref'] if 'ref' in data else data['HR'])

    def _g_gan(self):
        """generator GAN term (SRRaGAN_model.py:133-138 / SRGAN_model.py:131-133), D's filters frozen"""
        with _params_frozen(self.netD):
            pred_g_fake = self.netD(self.fake_H)
            if not self.relativistic:
                return self.l_gan_w * self.cri_gan(pred_g_fake, True)
            pred_d_real = self.netD(self.var_ref).detach()
        return self.l_gan_w * (self.cri_gan(pred_d_real - torch.mean(pred_g_fake), False) +
                               self.cri_gan(pred_g_fake - torch.mean(pred_d_real), True)) / 2

    def optimize_parameters(self, step):
        self.optimizer_G.zero_grad()
        self.fake_H = self.netG(self.var_L)
        do_g = step % self.D_update_ratio == 0 and step > self.D_init_iters
        if do_g:
            l_g_total = 0
            if self.cri_pix:
                l_g_pix = self.l_pix_w * self.cri_pix(self.fake_H, self.var_H)
                l_g_total = l_g_total + l_g_pix
            if self.cri_fea:
                real_fea = self.netF(self.var_H).detach()
                fake_fea = self.netF(self.fake_H)
                l_g_fea = self.l_fea_w * self.cri_fea(fake_fea, real_fea)
                l_g_total = l_g_total + l_g_fea
            l_g_gan = self._g_gan()
            l_g_total = l_g_total + l_g_gan
            l_g_total.backward()
            self.optimizer_G.step()
        # D
        self.optimizer_D.zero_grad()
        pred_d_real = self.netD(self.var_ref)
        pred_d_fake = self.netD(self.fake_H.detach())
        if self.relativistic:
            l_d_real = self.cri_gan(pred_d_real - torch.mean(pred_d_fake), True)
            l_d_fake = self.cri_gan(pred_d_fake - torch.mean(pred_d_real), False)
            l_d_total = (l_d_real + l_d_fake) / 2
        else:
            l_d_real = self.cri_gan(pred_d_real, True)
            l_d_fake = self.cri_gan(pred_d_fake, False)
            l_d_total = l_d_real + l_d_fake
        wgan_gp = self.opt['train']['gan_type'] == 'wgan-gp'
        if wgan_gp:
            batch_size = self.var_ref.size(0)
            if self.random_pt.size(0) != batch_size:
                self.random_pt.resize_(batch_size, 1, 1, 1)
            self.random_pt.uniform_()
            interp = self.random_pt * self.fake_H.detach() + (1 - self.random_pt) * self.var_ref
            interp.requires_grad = True
            interp_crit = self.netD(interp)
            l_d_gp = self.l_gp_w * self.cri_gp(interp, interp_crit)
            l_d_total = l_d_total + l_d_gp
        l_d_total.backward()
        self.optimizer_D.step()
        if do_g:
            if self.cri_pix:
                self.log_dict['l_g_pix'] = l_g_pix.item()
            if self.cri_fea:
                self.log_dict['l_g_fea'] = l_g_fea.item()
            self.log_dict['l_g_gan'] = l_g_gan.item()
        self.log_dict['l_d_real'] = l_d_real.item()
        self.log_dict['l_d_fake'] = l_d_fake.item()
        if wgan_gp:
            self.log_dict['l_d_gp'] = l_d_gp.item()
        self.log_dict['D_real'] = torch.mean(pred_d_real.detach())
        self.log_dict['D_fake'] = torch.mean(pred_d_fake.detach())

    def test(self):
        self.netG.eval()
        with torch.no_grad():
            self.fake_H = self.netG(self.var_L)
            if self.cri_fea_lpips is not None:
                self.LPIPS = self.cri_fea_lpips(self.fake_H, self.var_H)
            else:
                self.LPIPS = torch.full((self.fake_H.shape[0], 1, 1, 1), float('nan'))
        self.netG.train()

    def get_current_log(self):
        return self.log_dict

    def get_current_visuals(self, need_HR=True):
        out = OrderedDict()
        out['LR'] = self.var_L.detach()[0].float().cpu()
        out['SR'] = self.fake_H.detach()[0].float().cpu()
        if need_HR:
            out['HR'] = self.var_H.detach()[0].float().cpu()
            out['LPIPS'] = self.LPIPS.detach().float().cpu()
        return out

    def print_network(self):
        self._log_network(self.netG, 'G')
        if self.is_train:
            self._log_network(self.netD, 'D')
            if self.cri_fea:
                self._log_network(self.netF, 'F')

    def load(self):
        path = self.opt['path']
        if path['pretrain_model_G'] is not None:
            logger.info('Loading pretrained model for G [{:s}] ...'.format(path['pretrain_model_G']))
            self.load_network(path['pretrain_model_G'], self.netG)
        if self.opt['is_train'] and path['pretrain_model_D'] is not None:
            logger.info('Loading pretrained model for D [{:s}] ...'.format(path['pretrain_model_D']))
            self.load_network(path['pretrain_model_D'], self.netD)

    def save(self, iter_step):
        self.save_network(self.netG, 'G', iter_step)
        self.save_network(self.netD, 'D', iter_step)
