"""Data-parallel execution on one 8×H100 node (one process per GPU)."""
from .data_parallel import DataParallel  # noqa
