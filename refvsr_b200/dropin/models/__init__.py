"""Put `<repo>/refvsr_b200/dropin` in front of the reference checkout on sys.path and the reference's
`from models.SRNet import SRNet` / `importlib.import_module('models.archs.RefVSR')` resolve to the CUDA
implementation; run.py / eval.py / trainers / ckpt_manager stay untouched (INTEGRATION.md).

Only `models/SRNet.py` and `models/archs/RefVSR.py` are overridden.  The reference's `models/` directory (a namespace
package: it has no __init__.py) is appended to this package's `__path__`, so `models.utils`, `models.loss.Loss`
(`trainers/trainer.py:20-21`) and every other `models.archs.<name>` (`models/SRNet.py:20-21`) still resolve to the
reference's own files."""
import os
import sys

_here = os.path.dirname(os.path.abspath(__file__))
REFERENCE_DIR = None
for _p in list(sys.path) + [os.getcwd()]:
    _cand = os.path.join(_p or os.getcwd(), 'models')
    if (os.path.isdir(_cand) and os.path.abspath(_cand) != _here
            and os.path.isfile(os.path.join(_cand, 'archs', 'RefVSR.py')) and os.path.isfile(os.path.join(_cand, 'utils.py'))):
        __path__.append(_cand)          # noqa: F821  (package attribute)
        REFERENCE_DIR = _cand
        break
# (no reference checkout on sys.path: the package still serves SRNet / archs.RefVSR on their own)
