"""malio_b200 — H100-native (sm_90a) MA-LIO measurement hot path (k-NN over a flattened ikd-Tree, plane fit +
point-wise uncertainty, fused H^T R^-1 H reduction, host IESKF) behind the C-ABI of include/malio_b200.h."""
from . import capi, plugin, synth  # noqa: F401
from .plugin import MeasurementModel, MapSnapshot, build_static_snapshot  # noqa: F401
