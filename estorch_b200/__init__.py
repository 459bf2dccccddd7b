"""estorch_b200 -- Blackwell-native Evolution Strategies engine behind the estorch API.

Public names mirror the reference package (estorch/__init__.py:1-2,
docs/index.rst:4-15): ``ES``, ``NS_ES``, ``NSR_ES``, ``NSRA_ES``,
``rank_transformation``, ``VirtualBatchNorm``; plus the device-agent and population-agent protocols.
"""
from .agents import DeviceAgent, PopulationAgent, SequenceAgent, SyntheticAgent
from .estorch import ES, NS_ES, NSR_ES, NSRA_ES, rank_transformation
from .vbn import VirtualBatchNorm

__version__ = "0.1.0"
__all__ = ["ES", "NS_ES", "NSR_ES", "NSRA_ES", "rank_transformation", "VirtualBatchNorm",
           "DeviceAgent", "PopulationAgent", "SequenceAgent", "SyntheticAgent"]
