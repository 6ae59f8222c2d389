"""graph_weather_b200 -- the encode-process-decode GNN forward of openclimatefix/graph_weather, rebuilt for H100 (sm_90a).

Public names mirror graph_weather/__init__.py:3-9 and graph_weather/models/__init__.py:3-17 for the hot path only.
"""

from .constraint import PhysicalConstraintLayer  # noqa: F401
from .losses import NormalizedMSELoss  # noqa: F401
from .dynamic_graph_builder import DynamicGraphBuilder  # noqa: F401
from .models import (  # noqa: F401
    AssimilatorDecoder,
    AssimilatorEncoder,
    Decoder,
    Encoder,
    GraphCast,
    GraphCastConfig,
    GraphWeatherAssimilator,
    GraphWeatherAssimilatorConfig,
    GraphWeatherForecaster,
    GraphWeatherForecasterConfig,
    Processor,
)
from .regional import BoundaryNudgingLayer, RegionalForecaster, RegionalForecasterConfig  # noqa: F401

__all__ = [
    "GraphWeatherForecaster", "GraphWeatherForecasterConfig", "GraphWeatherAssimilator", "GraphWeatherAssimilatorConfig",
    "GraphCast", "GraphCastConfig", "Encoder", "Processor", "Decoder", "AssimilatorEncoder", "AssimilatorDecoder",
    "NormalizedMSELoss", "PhysicalConstraintLayer", "DynamicGraphBuilder", "RegionalForecaster", "RegionalForecasterConfig",
    "BoundaryNudgingLayer",
]  # fmt: skip
