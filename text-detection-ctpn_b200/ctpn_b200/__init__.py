"""ctpn_b200: H100-native (sm_90a) CTPN text-detection hot path (drop-in for the detection path of
eragonruan/text-detection-ctpn).  Importing the package loads libctpn_b200.so; there is no
CPU fallback."""
from ._native import CtpnError, LIB_PATH, lib  # noqa: F401
from .engine import YUV420, Engine, frontend_plan, load_weight_file, ragged_plan  # noqa: F401
from .session import Session  # noqa: F401

__all__ = ["Engine", "Session", "CtpnError", "YUV420", "load_weight_file", "ragged_plan", "frontend_plan", "LIB_PATH"]
