"""vbx_b200: the VB-HMM EM loop of BUTSpeechFIT/VBx (VBx/VBx.py) as hand-written sm_90a CUDA kernels
behind a C ABI (include/vbx_b200.h), with a drop-in `VBx()` (+ `forward_backward`, `DER`), a batched `VbxBatch` /
`make_batch`, whole-archive `diarize_batch` and the command line `python -m vbx_b200.cli`."""
from ._lib import VbxError, LIB_PATH  # noqa: F401


def __getattr__(name):
    # torch is imported lazily so that `import vbx_b200.formats` etc. stay light
    if name in ('VBx', 'DER', 'forward_backward'):
        from . import api
        return getattr(api, name)
    if name in ('VbxBatch', 'vbx_batch'):
        from . import batch
        return getattr(batch, name)
    if name in ('make_batch', 'PartitionedBatch'):
        from . import parts
        return getattr(parts, name)
    if name in ('diarize_batch', 'diarize_recording'):
        from . import pipeline
        return getattr(pipeline, name)
    raise AttributeError(name)
