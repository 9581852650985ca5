"""python -m dasr_b200.install <path/to/DASR/codes> [--pth] [--uninstall]

Marks `codes/SRN` and `codes/DSN` of a reference checkout for the dasr_b200 import overlay (dasr_b200/overlay.py) and
makes the overlay start with every interpreter, so that `python Auto_Reproduce.py --dataset ... --artifact ...` — which
shells out to `cd ./DSN; sh auto_reproduce_launcher_*.sh` and `cd ./SRN; python train.py -opt ...`
(Auto_Reproduce.py:38-40) — runs the H100 modules without a single edit in the checkout's sources.

  * writes `<codes>/SRN/.dasr_b200` ("SRN") and `<codes>/DSN/.dasr_b200` ("DSN")  — the only files added to the checkout;
  * interpreter hook, one of
      --pth      : `dasr_b200_overlay.pth` in this interpreter's site-packages (permanent for this environment), or
      (default)  : prints the `export PYTHONPATH=...` line that activates it through sitecustomize for one shell.
  * --uninstall removes the markers and the .pth file.
"""
import argparse
import os
import site
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
PTH = 'dasr_b200_overlay.pth'


def _pth_path():
    return os.path.join(site.getsitepackages()[0], PTH)


def install(codes, pth=False, out=sys.stdout):
    codes = os.path.abspath(codes)
    done = []
    for flavour in ('SRN', 'DSN'):
        d = os.path.join(codes, flavour)
        if not os.path.isdir(d):
            raise SystemExit('%s is not a DASR codes directory (no %s/)' % (codes, flavour))
        with open(os.path.join(d, '.dasr_b200'), 'w') as fh:
            fh.write(flavour + '\n')
        done.append(d)
    site_dir = os.path.join(HERE, 'overlay_site')
    if pth:
        with open(_pth_path(), 'w') as fh:
            fh.write('import sys; sys.path.append(%r); import dasr_b200.overlay as _o; _o.activate()\n' % ROOT)
        out.write('overlay hook written to %s\n' % _pth_path())
    else:
        out.write('activate the overlay for this shell with:\n  export PYTHONPATH=%s:%s${PYTHONPATH:+:$PYTHONPATH}\n' % (site_dir, ROOT))
    out.write('marked: %s\n' % ', '.join(done))
    return site_dir


def uninstall(codes, out=sys.stdout):
    codes = os.path.abspath(codes)
    for flavour in ('SRN', 'DSN'):
        m = os.path.join(codes, flavour, '.dasr_b200')
        if os.path.exists(m):
            os.remove(m)
            out.write('removed %s\n' % m)
    try:
        p = _pth_path()
        if os.path.exists(p):
            os.remove(p)
            out.write('removed %s\n' % p)
    except Exception:
        pass


def main(argv=None):
    ap = argparse.ArgumentParser(prog='python -m dasr_b200.install', description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('codes', help='the `codes` directory of a ShuhangGu/DASR checkout')
    ap.add_argument('--pth', action='store_true', help='install a site-packages .pth hook instead of printing the PYTHONPATH line')
    ap.add_argument('--uninstall', action='store_true')
    a = ap.parse_args(argv)
    if a.uninstall:
        uninstall(a.codes)
    else:
        install(a.codes, a.pth)
    return 0


if __name__ == '__main__':
    sys.exit(main())
