"""create_model(opt) — same dispatch on opt['model'] as codes/SRN/models/__init__.py:5-26 for the models
of the SRN hot path.  'DASR_FS_ESRGAN_patchGAN' (the name the shipped train_DASR*.json files use, which
the reference's create_model does not know — SURVEY.md §5.6a) is accepted as an alias of 'DASR'."""
import logging

logger = logging.getLogger('base')


def create_model(opt):
    model = opt['model']
    if model == 'sr':
        from .SR_model import SRModel as M
    elif model == 'srgan':
        from .SRGAN_model import SRGANModel as M
    elif model == 'srragan':
        from .SRRaGAN_model import SRRaGANModel as M
    elif model in ('DASR', 'DASR_FS_ESRGAN_patchGAN'):
        from .DASR_model import DASR_Model as M
    elif model == 'DASR_Adaptive_Model':
        from .DASR_Adaptive_model import DASR_Adaptive_Model as M
    else:
        raise NotImplementedError('Model [{:s}] not recognized.'.format(str(model)))
    m = M(opt)
    logger.info('Model [{:s}] is created.'.format(m.__class__.__name__))
    return m


def _see_reference_package(name):
    """When this mirror shadows the reference package of the same name (dasr_b200.launch / PYTHONPATH overlay), keep the
    reference's OTHER submodules importable (e.g. utils.receptive_cal, which test.py imports): append the shadowed
    directory to this package's search path — files that exist here still win."""
    import os
    import sys
    here = [os.path.abspath(p) for p in __path__]
    for d in sys.path:
        cand = os.path.abspath(os.path.join(d or '.', name))
        if os.path.isdir(cand) and cand not in here and os.path.exists(os.path.join(cand, '__init__.py')):
            __path__.append(cand)


if __name__ == 'models':          # imported as the top-level package, i.e. as the drop-in
    _see_reference_package('models')
