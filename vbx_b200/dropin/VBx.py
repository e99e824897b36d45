"""Shadow of the reference module VBx/VBx.py: `from VBx import VBx` (VBx/vbhmm.py:45) resolves to the H100
implementation when this module is what `VBx` names.  For the unchanged `python VBx/vbhmm.py ...` use the launcher
(`python -m vbx_b200.dropin.run VBx/vbhmm.py ...`): a script's own directory comes first on sys.path, so PYTHONPATH
alone cannot shadow a module that sits next to the script."""
import os
import sys

_ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if _ROOT not in sys.path:
    sys.path.insert(0, _ROOT)

from vbx_b200.api import VBx, DER, forward_backward  # noqa: E402,F401
