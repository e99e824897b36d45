"""Run an UNCHANGED reference script (VBx/vbhmm.py) with `VBx` bound to the H100 implementation:

    python -m vbx_b200.dropin.run /path/to/VBx/vbhmm.py --init AHC+VB --out-rttm-dir exp ...

`python VBx/vbhmm.py` puts the script's directory at sys.path[0], ahead of PYTHONPATH, so `from VBx import VBx`
(VBx/vbhmm.py:45) would still find the reference's VBx.py next to it.  This launcher registers the shadow module as
`sys.modules['VBx']` first - an import statement consults sys.modules before any path - then executes the script as
__main__ with its own directory on sys.path, exactly as the interpreter would."""
import importlib
import os
import runpy
import sys


def main(argv=None):
    argv = sys.argv[1:] if argv is None else list(argv)
    if not argv or argv[0] in ('-h', '--help'):
        print(__doc__)
        return 2
    script = os.path.abspath(argv[0])
    if not os.path.isfile(script):
        print(f'vbx_b200.dropin.run: no such script: {script}', file=sys.stderr)
        return 2
    shadow = importlib.import_module('vbx_b200.dropin.VBx')
    sys.modules['VBx'] = shadow
    sys.path.insert(0, os.path.dirname(script))
    sys.argv = [script] + argv[1:]
    runpy.run_path(script, run_name='__main__')
    return 0


if __name__ == '__main__':
    sys.exit(main())
