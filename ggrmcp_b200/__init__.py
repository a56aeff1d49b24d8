"""ggrmcp_b200 - GPU-native JSON<->protobuf transcoding engine for ggRMCP's tools/call hot path.

The package is a thin host layer over libggrmcp_b200.so (hand-written sm_90a kernels for the H100 behind the C
ABI of include/ggrmcp_b200.h).  There is no CPU fallback: creating an Engine without a CUDA device
raises.
"""
from .engine import (Engine, Schema, EngineError, STATUS_NAMES, F_COMMA_SPACE, ORDER_FIELD_NUMBER, ORDER_GO_LEGACY,
                     lib_path)

__all__ = ["Engine", "Schema", "EngineError", "STATUS_NAMES", "F_COMMA_SPACE", "ORDER_FIELD_NUMBER",
           "ORDER_GO_LEGACY", "lib_path"]
