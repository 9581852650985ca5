"""DASR_Model — the SRN GAN training step + test path (reference: codes/SRN/models/DASR_model.py).

Same attributes (netG, netD_target, netD_source, netF, optimizers, schedulers, log_dict), same methods
(feed_data, optimize_parameters, test, get_current_log, get_current_visuals, save, load, ...), same loss
arithmetic including the reference's quirks (pixel weight applied twice, :214-218).  Differences, all
behaviour-preserving:
  * every network / loss / frequency split runs on dasr_b200 kernels;
  * b_split on the fixed [0]*B+[1]*B mask is a view, not a per-sample cat (:200-207);
  * while G's loss is back-propagated through D, D's filter gradients (which the reference computes and
    then discards with optimizer_D_target.zero_grad(), :282) are not computed;
  * log values are kept as device scalars and only synchronised in get_current_log();
  * under torch.distributed (one process per GPU) the G and D gradients live in one flat bucket and are averaged over
    NCCL before both optimiser steps (dasr_b200.dp; G's segment is exchanged while the discriminator step runs) —
    equivalent to the reference order because the D step only consumes tensors detached before the G update
    (SURVEY.md §8e); rank 0's initial weights are broadcast, checkpoints are written by rank 0 only.
"""
import contextlib
import logging
from collections import OrderedDict

import torch
import torch.nn as nn

from dasr_b200 import dp, ops
from dasr_b200.srn.utils.util import b_split, forward_chop
from . import networks
from .base_model import BaseModel
from .modules import loss as L
from .modules.architecture import FilterHigh, FilterLow

logger = logging.getLogger('base')


@contextlib.contextmanager
def _params_frozen(net):
    ps = [p for p in net.parameters() if p.requires_grad]
    for p in ps:
        p.requires_grad_(False)
    try:
        yield
    finally:
        for p in ps:
            p.requires_grad_(True)


def _side_math(netG):
    """'tf32' when the generator trains in mixed precision (DASR_B200_SIDE_MATH overrides: fma | tf32 | tf32x3), else the
    library default (exact FMA unless DASR_B200_F32_MATH says otherwise)."""
    import os
    net = netG.module if hasattr(netG, 'module') else netG
    tp = getattr(net, 'train_precision', None) or os.environ.get('DASR_B200_TRAIN_PRECISION', 'fp32')
    if tp != 'bf16':
        return 'default'
    return os.environ.get('DASR_B200_SIDE_MATH', 'tf32')


def _ragan_pair(cri_gan, pred_real, pred_fake, for_G):
    """Relativistic average GAN term of the generator (DASR_model.py:242-246): each set's scores relative to the batch
    mean (dim 0, per patch position) of the other set; the real scores carry no gradient."""
    pred_real = pred_real.detach()
    return (cri_gan(pred_fake - pred_real.mean(0, keepdim=True), True) +
            cri_gan(pred_real - pred_fake.mean(0, keepdim=True), False)) / 2


class DASR_Model(BaseModel):
    def __init__(self, opt):
        super().__init__(opt)
        train_opt = opt['train'] if opt['train'] is not None else {}
        self.chop = opt['chop']
        self.scale = opt['scale']
        self.val_lpips = opt['val_lpips']
        self.adaptive_weights = opt['adaptive_weights']
        self.multiweights = opt['multiweights']

        self.ragan = train_opt.get('ragan')
        self.l_gan_H_target_w = train_opt.get('gan_H_target') or 0
        self.l_gan_H_source_w = train_opt.get('gan_H_source') or 0
        if self.is_train:
            self.cri_gan = L.GANLoss(train_opt['gan_type'], 1.0, 0.0).to(self.device)
            if train_opt['gan_type'] == 'wgan-gp':
                raise NotImplementedError('wgan-gp gradient penalty (double backward) is not on the H100 path')

        self.netG = networks.define_G(opt).to(self.device)
        if self.is_train:
            if self.l_gan_H_target_w > 0:
                self.netD_target = networks.define_D(opt).to(self.device)
                self.netD_target.train()
            if self.l_gan_H_source_w > 0:
                self.netD_source = networks.define_pairD(opt).to(self.device)
                self.netD_source.train()
            self.netG.train()
        self.load()

        # frequency separation.  fs_kernel_size defaults to 5: the shipped wavelet configs omit it and the
        # reference then crashes in FilterHigh(kernel_size=None) (SURVEY §5.6b).
        self.norm = train_opt.get('norm')
        fs = train_opt.get('fs') or 'wavelet'
        ks = train_opt.get('fs_kernel_size') or 5
        if fs == 'wavelet':
            self.fs = self.wavelet_s
            self.filter_high = FilterHigh(kernel_size=ks, gaussian=True).to(self.device)
        elif fs in ('gau', 'avgpool'):
            g = fs == 'gau'
            self.filter_low = FilterLow(kernel_size=ks, gaussian=g).to(self.device)
            self.filter_high = FilterHigh(kernel_size=ks, gaussian=g).to(self.device)
            self.fs = self.filter_func
        else:
            raise NotImplementedError('FS type [{:s}] not recognized.'.format(str(fs)))

        if self.is_train:
            self._init_training(opt, train_opt)
        self.print_network()
        if self.val_lpips:      # DASR_model.py:158-159
            from dasr_b200.lpips import PerceptualLoss as val_lpips
            self.cri_fea_lpips = val_lpips(model='net-lin', net='alex').to(self.device)

    def _init_training(self, opt, cfg):
        """Losses, perceptual network, update cadence, optimisers and schedulers of the GAN step (DASR_model.py:75-151)."""
        # pixel / LL losses
        self.cri_pix = None
        if cfg['pixel_weight'] > 0:
            self.cri_pix = self._criterion(cfg['pixel_criterion'])
            self.l_pix_w, self.l_pix_LL_w, self.sup_LL = cfg['pixel_weight'], cfg['pixel_LL_weight'], cfg['sup_LL']
        else:
            logger.info('Remove pixel loss.')
        # perceptual loss on VGG19 features
        self.cri_fea, self.l_fea_type = None, cfg['feature_criterion']
        if cfg['feature_weight'] > 0:
            self.l_fea_w = cfg['feature_weight']
            if self.l_fea_type == 'LPIPS':       # DASR_model.py:97: PerceptualLoss() = mean LPIPS(alex) of [0,1] images
                from dasr_b200.lpips import PerceptualLossAug
                self.cri_fea = PerceptualLossAug().to(self.device)
            else:
                self.cri_fea = self._criterion(self.l_fea_type)
                self.netF = networks.define_F(opt, use_bn=False).to(self.device)
        else:
            logger.info('Remove feature loss.')
        # update cadence
        self.G_update_inter = cfg['G_update_inter'] or 1
        self.D_update_inter = cfg['D_update_inter'] or 1
        self.D_update_ratio = cfg['D_update_ratio'] or 1
        self.D_init_iters = cfg['D_init_iters'] or 0
        # optimisers: G first, then the discriminators that are switched on (order = checkpoint order)
        self.optimizer_G = self._adam(self.netG, cfg['lr_G'], cfg['weight_decay_G'], cfg['beta1_G'])
        trained = [self.netG]
        for weight, attr in ((self.l_gan_H_target_w, 'target'), (self.l_gan_H_source_w, 'source')):
            if weight > 0:
                net = getattr(self, 'netD_' + attr)
                setattr(self, 'optimizer_D_' + attr, self._adam(net, cfg['lr_D'], cfg['weight_decay_D'], cfg['beta1_D']))
                trained.append(net)
        self._make_schedulers(cfg)
        self.log_dict, self._log_t = OrderedDict(), OrderedDict()
        # data parallel: one flat gradient bucket over [G | D_target | D_source]
        # (construction broadcasts rank 0's weights; G's mixed-precision backward writes straight into its bucket segment)
        self.grad_sync = dp.GradBucket(trained)

    # ------------------------------------------------------------------------------------------ data
    def feed_data(self, data, istrain):
        if istrain and 'HR' in data:
            HR_pair = self._to_device(data['HR'])
            HR_unpair = self._to_device(data['HR_unpair'])
            fake_w = self._to_device(data['fake_w']).float().contiguous()
            real_LR = self._to_device(data['LR_real'])
            fake_LR = self._to_device(data['LR_fake'])
            self.var_L = torch.cat([fake_LR, real_LR], dim=0)
            self.var_H = torch.cat([HR_pair, HR_unpair], dim=0)
            # bilinear (align_corners=False) resize of the domain-distance map to the HR crop
            self.weights = torch.empty((fake_w.shape[0], fake_w.shape[1], HR_pair.shape[2], HR_pair.shape[3]),
                                       dtype=torch.float32, device=self.device)
            ops.bilinear(fake_w, self.weights)
            B = self.var_L.shape[0]
            self.mask = [0] * (B // 2) + [1] * (B - B // 2)
        else:
            self.var_L = self._to_device(data['LR'])
            if 'HR' in data:
                self.var_H = self._to_device(data['HR'])
                self.needHR = True
            else:
                self.needHR = False

    # ------------------------------------------------------------------------------------------ step
    def optimize_parameters(self, step):
        # mixed-precision training: the fp32 side nets (discriminator, Cin-3 / strided layers) take tf32 tensor-core math
        with ops.f32_math(_side_math(self.netG)):
            self._optimize_parameters(step)

    def _optimize_parameters(self, step):
        with ops.nvtx('G/forward'):
            self.fake_H = self.netG(self.var_L)
        with ops.nvtx('frequency_separation'):
            self.fake_LL, self.fake_Hc = self.fs(self.fake_H, norm=self.norm)
            self.real_LL, self.real_Hc = self.fs(self.var_H, norm=self.norm)

        self.fake_SR_source, _ = b_split(self.fake_H, self.mask)
        self.fake_SR_LL_source, _ = b_split(self.fake_LL, self.mask)
        self.fake_SR_Hf_source, self.fake_SR_Hf_target = b_split(self.fake_Hc, self.mask)
        self.real_HR_source, _ = b_split(self.var_H, self.mask)
        self.real_HR_LL_source, _ = b_split(self.real_LL, self.mask)
        self.real_HR_Hf_source, self.real_HR_Hf_target = b_split(self.real_Hc, self.mask)

        do_G = step % self.G_update_inter == 0
        do_D = step % self.D_update_inter == 0
        log = self._log_t
        if do_G:
            l_g_total = 0
            if self.cri_pix:
                if self.multiweights:
                    l_g_pix = self.l_pix_w * L.weighted_l1(self.fake_SR_source, self.real_HR_source, self.weights)
                else:
                    l_g_pix = self.cri_pix(self.fake_SR_source, self.real_HR_source)
                l_g_total += self.l_pix_w * l_g_pix
                if self.sup_LL:
                    l_g_LL_pix = self.cri_pix(self.fake_SR_LL_source, self.real_HR_LL_source)
                    l_g_total += self.l_pix_LL_w * l_g_LL_pix
            if self.cri_fea and self.l_fea_type in ['l1', 'l2']:
                real_fea = self.netF(self.real_HR_source).detach()
                fake_fea = self.netF(self.fake_SR_source)
                l_g_fea = self.cri_fea(fake_fea, real_fea)
                l_g_total += self.l_fea_w * l_g_fea
            elif self.cri_fea and self.l_fea_type == 'LPIPS':
                l_g_fea = self.cri_fea(self.fake_SR_source, self.real_HR_source)
                l_g_total += self.l_fea_w * l_g_fea
            if self.l_gan_H_target_w > 0:
                with _params_frozen(self.netD_target):
                    pred_g_Hf_target_fake = self.netD_target(self.fake_SR_Hf_target)
                    if self.ragan:
                        with torch.no_grad():
                            pred_g_Hf_target_real = self.netD_target(self.real_HR_Hf_target)
                if self.ragan:
                    # relativistic average: scores relative to the other set's batch mean (DASR_model.py:242-246; the weight
                    # is applied here AND below, as the reference does)
                    l_g_gan_target_Hf = self.l_gan_H_target_w * _ragan_pair(self.cri_gan, pred_g_Hf_target_real,
                                                                             pred_g_Hf_target_fake, True)
                else:
                    l_g_gan_target_Hf = self.cri_gan(pred_g_Hf_target_fake, True)
                l_g_total += self.l_gan_H_target_w * l_g_gan_target_Hf
            if self.l_gan_H_source_w > 0:
                with _params_frozen(self.netD_source):
                    pred_g_Hf_source_fake = self.netD_source(self.fake_SR_Hf_source)
                    if self.ragan:
                        with torch.no_grad():
                            pred_g_Hf_source_real = self.netD_source(self.real_HR_Hf_source)
                if self.ragan:
                    l_g_gan_source_Hf = self.l_gan_H_source_w * _ragan_pair(self.cri_gan, pred_g_Hf_source_real,
                                                                             pred_g_Hf_source_fake, True)
                else:
                    l_g_gan_source_Hf = self.l_gan_H_source_w * self.cri_gan(pred_g_Hf_source_fake, True)
                l_g_total += l_g_gan_source_Hf
            self.optimizer_G.zero_grad()
            with ops.nvtx('G/backward'):
                l_g_total.backward()
            if not self.grad_sync.active:
                self.optimizer_G.step()
            else:
                self.grad_sync.reduce_segment(0)      # G's all-reduce starts now and overlaps the discriminator step

        if do_D:
            if self.l_gan_H_target_w > 0:
                # (NVTX: the D step is everything between 'G/backward' and 'dp/finish+optimizers')
                # one discriminator pass over [real | fake] (DASR_model.py:271-272 runs two): InstanceNorm statistics are
                # per sample, so the scores and the parameter gradients are the same sums
                nreal = self.real_HR_Hf_target.shape[0]
                pred_d = self.netD_target(torch.cat([self.real_HR_Hf_target.detach(), self.fake_SR_Hf_target.detach()], 0))
                pred_d_target_real, pred_d_target_fake = pred_d[:nreal], pred_d[nreal:]
                if self.ragan:
                    l_d_target_real = self.cri_gan(pred_d_target_real - pred_d_target_fake.mean(0, keepdim=True), True)
                    l_d_target_fake = self.cri_gan(pred_d_target_fake - pred_d_target_real.mean(0, keepdim=True), False)
                else:
                    l_d_target_real = self.cri_gan(pred_d_target_real, True)
                    l_d_target_fake = self.cri_gan(pred_d_target_fake, False)
                l_d_target_total = (l_d_target_real + l_d_target_fake) / 2
                self.optimizer_D_target.zero_grad()
                l_d_target_total.backward()
                if not self.grad_sync.active:
                    self.optimizer_D_target.step()
            if self.l_gan_H_source_w > 0:
                pred_d_source_real = self.netD_source(self.real_HR_Hf_source.detach())
                pred_d_source_fake = self.netD_source(self.fake_SR_Hf_source.detach())
                if self.ragan:
                    l_d_source_real = self.cri_gan(pred_d_source_real - pred_d_source_fake.mean(0, keepdim=True), True)
                    l_d_source_fake = self.cri_gan(pred_d_source_fake - pred_d_source_real.mean(0, keepdim=True), False)
                else:
                    l_d_source_real = self.cri_gan(pred_d_source_real, True)
                    l_d_source_fake = self.cri_gan(pred_d_source_fake, False)
                l_d_source_total = (l_d_source_fake + l_d_source_real) / 2
                self.optimizer_D_source.zero_grad()
                l_d_source_total.backward()
                if not self.grad_sync.active:
                    self.optimizer_D_source.step()

        if self.grad_sync.active:
            # gradient exchange over NCCL (G's segment already in flight, D's now; DASR_B200_DP_OVERLAP=0: one all-reduce of
            # the whole [G | D] bucket here), then the deferred optimiser steps
            with ops.nvtx('dp/finish+optimizers'):
                self.grad_sync.finish()
                if do_G:
                    self.optimizer_G.step()
                if do_D and self.l_gan_H_target_w > 0:
                    self.optimizer_D_target.step()
                if do_D and self.l_gan_H_source_w > 0:
                    self.optimizer_D_source.step()

        if do_G:
            if self.cri_pix:
                log['loss/l_g_pix'] = l_g_pix.detach()
                if self.sup_LL:
                    log['loss/l_g_LL_pix'] = l_g_LL_pix.detach()
            if self.cri_fea:
                log['loss/l_g_fea'] = l_g_fea.detach()
            if self.l_gan_H_target_w > 0:
                log['loss/l_g_gan_target_Hf'] = l_g_gan_target_Hf.detach()
            if self.l_gan_H_source_w > 0:
                log['loss/l_g_gan_source_H'] = l_g_gan_source_Hf.detach()
        if do_D:
            if self.l_gan_H_target_w > 0:
                log['loss/l_d_target_total'] = l_d_target_total.detach()
                log['disc_Score/D_real_target_H'] = L.mean(pred_d_target_real.detach())
                log['disc_Score/D_fake_target_H'] = L.mean(pred_d_target_fake.detach())
            if self.l_gan_H_source_w > 0:
                log['loss/l_d_total'] = l_d_source_total.detach()
                log['disc_Score/D_real_source_H'] = L.mean(pred_d_source_real.detach())
                log['disc_Score/D_fake_source_H'] = L.mean(pred_d_source_fake.detach())

    def test(self, tsamples=False):
        self._log_eval_precision(self.netG)
        self.netG.eval()
        with torch.no_grad():
            if self.chop:
                self.fake_H = forward_chop(self.var_L, self.scale, self.netG, min_size=320000)
            else:
                self.fake_H = self.netG(self.var_L)
            if not tsamples and self.val_lpips:
                from .SR_model import _val_lpips
                self.LPIPS = _val_lpips(self.cri_fea_lpips, self.fake_H, self.var_H, self.device)
            self.netG.train()

    def get_current_log(self):
        """One device->host synchronisation for the whole dict (the reference does 7-10 .item() per step)."""
        for k, v in self._log_t.items():
            self.log_dict[k] = float(v)
        return self.log_dict

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
        return out

    def print_network(self):
        nets = [('G', self.netG)]
        if self.is_train:
            if self.l_gan_H_target_w > 0:
                nets.append(('D_target', self.netD_target))
            if self.l_gan_H_source_w > 0:
                nets.append(('D_source', self.netD_source))
            if self.cri_fea and self.l_fea_type in ['l1', 'l2']:
                nets.append(('F', self.netF))
        for label, net in nets:
            self._log_network(net, label)

    def load(self):
        path = self.opt['path']
        if path['pretrain_model_G'] is not None:
            logger.info('Loading pretrained model for G [{:s}] ...'.format(path['pretrain_model_G']))
            self.load_network(path['pretrain_model_G'], self.netG)
        if self.opt['is_train'] and path['pretrain_model_D_target'] is not None:
            logger.info('Loading pretrained model for D_target [{:s}] ...'.format(path['pretrain_model_D_target']))
            self.load_network(path['pretrain_model_D_target'], self.netD_target)
        if self.opt['is_train'] and path['pretrain_model_D_source'] is not None:
            logger.info('Loading pretrained model for D_source [{:s}] ...'.format(path['pretrain_model_D_source']))
            self.load_network(path['pretrain_model_D_source'], self.netD_source)

    def save(self, iter_step):
        self.save_network(self.netG, 'G', iter_step)
        if self.l_gan_H_target_w > 0:
            self.save_network(self.netD_target, 'D_target', iter_step)
        if self.l_gan_H_source_w > 0:
            self.save_network(self.netD_source, 'D_source', iter_step)

    # ------------------------------------------------------------------------- frequency separation
    def wavelet_s(self, x, norm=False):
        """(LL, cat(LH,HL,HH)) with LL*0.5 and Hc*0.5+0.5 when norm — one fused kernel."""
        return L.haar_split(x, norm)

    def filter_func(self, x, norm=False):
        low_f, high_f = self.filter_low(x), self.filter_high(x)
        if norm:
            high_f = high_f * 0.5 + 0.5
        return low_f, high_f
