"""refvsr_b200 - H100-native (sm_90a) implementation of RefVSR's per-frame forward hot path.

Public surface (mirrors the reference's module contract, SURVEY.md 8b):
    SRNet(config).forward(x, ref, is_first_frame=True, is_log=False, is_train=False) -> OrderedDict
    models.archs.RefVSR.Network(config)              (via refvsr_b200/dropin on sys.path)
    get_config(name)                                  config_RefVSR_* factories for standalone use
"""
from .config import get_config  # noqa: F401
from .network import Network  # noqa: F401
from .srnet import SRNet  # noqa: F401

__version__ = '0.1.0'
