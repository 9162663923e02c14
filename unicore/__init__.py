"""unicore: Uni-Core compatible training framework, Hopper-native underneath.

Importing the package populates the registries (optimizers, LR schedulers, losses, built-in tasks)
and installs the historical module aliases ``unicore.distributed_utils / meters / metrics /
progress_bar`` (reference ``unicore/__init__.py:21-35``).
"""
import sys

from .version import __version__  # noqa: F401

__all__ = []

from unicore.distributed import utils as distributed_utils  # noqa: E402
from unicore.logging import meters, metrics, progress_bar  # noqa: E402,F401

sys.modules["unicore.distributed_utils"] = distributed_utils
sys.modules["unicore.meters"] = meters
sys.modules["unicore.metrics"] = metrics
sys.modules["unicore.progress_bar"] = progress_bar

import unicore.ops  # noqa: E402,F401
import unicore.losses  # noqa: E402,F401
import unicore.distributed  # noqa: E402,F401
import unicore.models  # noqa: E402,F401
import unicore.modules  # noqa: E402,F401
import unicore.optim  # noqa: E402,F401
import unicore.optim.lr_scheduler  # noqa: E402,F401
import unicore.tasks  # noqa: E402,F401
