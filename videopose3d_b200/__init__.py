"""videopose3d_b200 — H100-native (sm_90a) execution of VideoPose3D's temporal-convolution models.

Public surface = the reference's ``common/model.py`` classes; everything else stays the reference's.
"""
from .temporal_model import TemporalModel, TemporalModelBase, TemporalModelOptimized1f
from .data_parallel import GradientReducer, broadcast_buffers
from .streaming import StreamingSession

__all__ = ["TemporalModelBase", "TemporalModel", "TemporalModelOptimized1f", "GradientReducer",
           "broadcast_buffers", "StreamingSession"]
__version__ = "0.1.0"
