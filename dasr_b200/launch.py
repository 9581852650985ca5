"""Run one of the reference's entry scripts on the H100 path without touching the reference checkout:

    python -m dasr_b200.launch /path/to/DASR/codes/SRN/test.py  -opt options/test/test_sr.json
    python -m dasr_b200.launch /path/to/DASR/codes/SRN/train.py -opt options/train/train_DASR_auto_reproduce_realsr.json
    python -m dasr_b200.launch /path/to/DASR/codes/DSN/train.py --per_type VGG --filter wavelet ...

Python always puts the script's own directory first on sys.path, so a PYTHONPATH overlay cannot shadow the reference's
`models` / `options` / `utils` (SRN) or `model` / `loss` (DSN) modules.  This launcher puts the mirrors in front of the
script directory and then executes the script unchanged (runpy), in the script's directory (its relative paths keep working).
The mirrors fall back to the reference's own submodules for everything they do not replace (`data/`, `scripts/`,
`utils/receptive_cal.py`, ...)."""
import os
import runpy
import sys


def main(argv):
    if not argv:
        print(__doc__)
        return 2
    script = os.path.abspath(argv[0])
    sdir = os.path.dirname(script)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    here = os.path.dirname(os.path.abspath(__file__))
    mirrors = [os.path.join(here, 'dsn')] if os.path.basename(sdir) == 'DSN' else [os.path.join(here, 'srn')]
    sys.path[:0] = mirrors + [root, sdir]
    sys.argv = [script] + list(argv[1:])
    from dasr_b200.overlay import _drop_in_defaults
    _drop_in_defaults()                      # reference scripts train in mixed precision unless DASR_B200_TRAIN_PRECISION=fp32
    os.chdir(sdir)
    runpy.run_path(script, run_name='__main__')
    return 0


if __name__ == '__main__':
    sys.exit(main(sys.argv[1:]))
