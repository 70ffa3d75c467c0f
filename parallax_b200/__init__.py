"""parallax_b200 — a Hopper-native sparsity-aware data-parallel training
engine with the capabilities and API of snuspl/parallax.

Public surface (parity with `parallax/parallax/__init__.py:16-26`):
`parallel_run`, `Config`, `PSConfig`, `MPIConfig`, `CommunicationConfig`,
`CheckPointConfig`, `ProfileConfig`, `get_partitioner`, `shard`, `log`; plus
the torch-side pieces a TF graph provided implicitly: `Graph`, `optim`, `nn`.
"""
from . import consts as _consts
_consts.adopt_horovod_env()          # HOROVOD_TIMELINE & co. work under their own names

from .partitions import get_partitioner
from .runner import parallel_run
from . import shard
from .log import parallax_log as log

from .config import ParallaxConfig as Config
from .config import PSConfig
from .config import MPIConfig
from .config import CommunicationConfig
from .config import CheckPointConfig
from .config import ProfileConfig

from .graph import (Graph, ClipByGlobalNorm, ClipByValue, ScaleGradients,
                    ExponentialMovingAverage)
from . import optim
from . import nn

__version__ = "0.1.0"

__all__ = [
    "get_partitioner", "parallel_run", "shard", "log", "Config", "PSConfig",
    "MPIConfig", "CommunicationConfig", "CheckPointConfig", "ProfileConfig",
    "Graph", "ClipByGlobalNorm", "ClipByValue", "ScaleGradients", "ExponentialMovingAverage",
    "optim", "nn",
]
