"""univtg_b200 - H100-native (sm_90a) implementation of the UniVTG cross-modal encoder + heads hot path.

Public surface mirrors the reference plugin boundary (reference main/config.py:341-342, model/univtg.py:409-450):

    from univtg_b200 import build_model
    model, criterion = build_model(args)

The compute path is the CUDA library behind include/univtg_b200.h; there is no CPU / eager fallback.
"""
from ._lib import load_library, LIB_PATH  # noqa: F401


def build_model(args):
    from .plugin import build_model as _bm

    return _bm(args)
