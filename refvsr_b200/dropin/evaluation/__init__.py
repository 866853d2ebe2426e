"""Drop-in for the reference's `evaluation` package (SURVEY 8f row 1: the evaluation loop around the hot path).

With `<repo>/refvsr_b200/dropin` in front of the reference checkout on sys.path this package takes the place of `evaluation`;
`eval_qual_quan.py` (the default `qual_quan` mode), `eval_quan_FOV.py` (`--eval_mode FOV`) and `eval_quan_conf_map.py`
(`--eval_mode conf`) are overridden, every other sub-module (`init`, `metrics`) resolves to the reference's file through
`__path__`."""
import os
import sys

_here = os.path.dirname(os.path.abspath(__file__))
REFERENCE_DIR = None
for _p in list(sys.path) + [os.getcwd()]:
    _cand = os.path.join(_p or os.getcwd(), 'evaluation')
    if os.path.isdir(_cand) and os.path.abspath(_cand) != _here and os.path.isfile(os.path.join(_cand, 'eval_qual_quan.py')):
        __path__.append(_cand)          # noqa: F821
        REFERENCE_DIR = _cand
        break
else:
    raise ImportError('refvsr_b200.dropin.evaluation: the reference checkout (evaluation/eval_qual_quan.py) is not on sys.path')
