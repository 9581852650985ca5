"""Import overlay: makes an UNMODIFIED ShuhangGu/DASR checkout resolve its hot-path modules to the dasr_b200 mirrors, also
for the entry points that `codes/Auto_Reproduce.py` starts with `os.system` (Auto_Reproduce.py:38-40:
`cd ./DSN; sh auto_reproduce_launcher_<dataset>.sh`, `cd ./SRN; python train.py -opt ...`).

Python puts the running script's directory first on sys.path, so `codes/SRN/models` always wins over any PYTHONPATH
entry.  A `sys.meta_path` finder runs BEFORE the path-based import system: when the running script lives in a directory
that `python -m dasr_b200.install` has marked (a `.dasr_b200` file naming the flavour, SRN or DSN), the top-level imports

    SRN:  models, options, utils        ->  dasr_b200/srn/{models,options,utils}
    DSN:  model, loss, receptive_cal    ->  dasr_b200/dsn/{model,loss,receptive_cal}.py

are served from this repository; everything else (data/, scripts/, utils/receptive_cal.py, DSN/utils.py, ...) keeps
coming from the checkout (the mirror packages append the shadowed reference directory to their own __path__).
Unmarked directories are not affected.  DASR_B200_OVERLAY=0 disables the finder; DASR_B200_OVERLAY_LOG=<file> appends
one line per redirected import (used by the tests)."""
import importlib.abc
import importlib.util
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
MARKER = '.dasr_b200'
TABLE = {
    'SRN': {'models': os.path.join(HERE, 'srn', 'models'), 'options': os.path.join(HERE, 'srn', 'options'),
            'utils': os.path.join(HERE, 'srn', 'utils')},
    'DSN': {'model': os.path.join(HERE, 'dsn', 'model.py'), 'loss': os.path.join(HERE, 'dsn', 'loss.py'),
            'receptive_cal': os.path.join(HERE, 'dsn', 'receptive_cal.py')},
}
_NAMES = {n for t in TABLE.values() for n in t}


def _script_dir():
    argv0 = sys.argv[0] if getattr(sys, 'argv', None) else ''
    if argv0 and argv0 not in ('-c', '-m') and os.path.exists(argv0):
        return os.path.dirname(os.path.abspath(argv0))
    return os.path.abspath(sys.path[0] or os.getcwd()) if sys.path else os.getcwd()


class MirrorFinder(importlib.abc.MetaPathFinder):
    def __init__(self):
        self._flavour = {}

    def flavour(self, sdir):
        f = self._flavour.get(sdir)
        if f is None:
            f = ''
            try:
                with open(os.path.join(sdir, MARKER)) as fh:
                    f = fh.read().split()[0].strip()
            except (OSError, IndexError):
                pass
            self._flavour[sdir] = f
        return f

    def find_spec(self, name, path=None, target=None):
        if path is not None or name not in _NAMES or os.environ.get('DASR_B200_OVERLAY', '1') == '0':
            return None
        sdir = _script_dir()
        tab = TABLE.get(self.flavour(sdir))
        if not tab or name not in tab:
            return None
        dst = tab[name]
        if ROOT not in sys.path:
            sys.path.append(ROOT)                       # the mirrors import `dasr_b200...`
        if os.path.isdir(dst):
            spec = importlib.util.spec_from_file_location(name, os.path.join(dst, '__init__.py'), submodule_search_locations=[dst])
        else:
            spec = importlib.util.spec_from_file_location(name, dst)
        log = os.environ.get('DASR_B200_OVERLAY_LOG')
        if log:
            with open(log, 'a') as fh:
                fh.write('%s -> %s (script dir %s)\n' % (name, dst, sdir))
        return spec


def activate():
    if not any(isinstance(f, MirrorFinder) for f in sys.meta_path):
        sys.meta_path.insert(0, MirrorFinder())
        _drop_in_defaults()


def _drop_in_defaults():
    """Defaults of the drop-in entry points (this overlay, dasr_b200.launch): reference scripts train in the mixed-precision
    mode (wgmma fprop / dgrad / wgrad, tf32 side nets).  The library default stays the exact
    fp32 mode; DASR_B200_TRAIN_PRECISION=fp32 selects it for a script, too."""
    os.environ.setdefault('DASR_B200_TRAIN_PRECISION', 'bf16')
