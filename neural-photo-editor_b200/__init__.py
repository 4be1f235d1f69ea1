"""neural-photo-editor_b200: H100-native (sm_90a) implementation of the IAN hot path of
ajbrock/Neural-Photo-Editor behind the reference's own API.IAN surface.

    import importlib; npe = importlib.import_module("neural-photo-editor_b200")
    model = npe.IAN('IAN_simple.py', dnn=True)
"""
from .API import IAN  # noqa: F401
from ._lib import IanError, LIB_PATH, SIGNATURES, load  # noqa: F401
