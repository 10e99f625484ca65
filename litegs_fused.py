"""Drop-in module: ``import litegs_fused`` resolves to the H100-native implementation.

The reference imports its CUDA extension by this name (litegs/utils/wrapper.py:8-12).  With this repository
root on ``sys.path`` -- ahead of any installed ``litegs_fused`` -- the reference's wrapper.py, render/__init__.py,
statistic_helper.py and optimizer.py bind to ``litegs_b200.fused`` without modification.  See INTEGRATION.md.
"""
from litegs_b200.fused import *  # noqa: F401,F403
from litegs_b200.fused import CONFIG, EXPORTS  # noqa: F401
from litegs_b200 import fused as _impl

globals().update({name: getattr(_impl, name) for name in EXPORTS})
__all__ = list(EXPORTS)
