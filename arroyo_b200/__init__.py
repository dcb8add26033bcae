"""arroyo_b200: H100-native (sm_90a) window-assign / keyed-aggregate / windowed-join operators behind
Arroyo's ArrowOperator surface.  The compute lives in libarroyo_b200.so (hand-written CUDA behind a C ABI,
include/arroyo_b200.h); this package is the Python host-side mirror of the reference's operator interface
(arroyo-operator/src/operator.rs:1143-1257, context.rs) used by the tests and the benchmark.

There is no CPU fallback: operators raise if the CUDA library or a CUDA device is missing."""
from .config import Agg, JoinConfig, SessionConfig, WindowAggConfig, WindowFunctionConfig  # noqa: F401
from .context import (FINAL_WATERMARK, IDLE, Collector, OperatorContext, WatermarkGenerator,  # noqa: F401
                      WatermarkHolder)

__all__ = ["Agg", "WindowAggConfig", "SessionConfig", "JoinConfig", "WindowFunctionConfig", "Collector", "OperatorContext",
           "WatermarkGenerator", "WatermarkHolder", "FINAL_WATERMARK", "IDLE"]
