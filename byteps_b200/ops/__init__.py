"""Python faces of the sm_90a kernels."""
from .compress import GpuCompressor  # noqa: F401
from .pushpull import all_gather, pushpull_inplace, reduce_scatter  # noqa: F401
