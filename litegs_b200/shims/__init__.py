"""Stand-ins for the four third-party modules the reference imports at package import time but that are absent from this
image and cannot be installed offline (SURVEY 8f row 3): ``plyfile``, ``torchmetrics``, ``matplotlib``, ``simple_knn``.

They exist so that the UNMODIFIED reference package (``import litegs``; ``litegs/__init__.py:1-6``,
``litegs/training/trainer.py:3-10``, ``litegs/io_manager/ply.py:4``, ``litegs/scene/__init__.py:3``) imports and trains on
top of ``litegs_fused`` / ``fused_ssim`` from this repository.  Each shim implements exactly the calls the reference makes:

  plyfile        PlyElement.describe, PlyData([...]).write, PlyData.read, element["name"], element.properties[i].name
  torchmetrics   torchmetrics.image.psnr.PeakSignalNoiseRatio(data_range=...)  (+ functional form)
  matplotlib     import matplotlib.pyplot as plt  (imported by trainer.py:10, never called on the training path)
  simple_knn     simple_knn._C.distCUDA2(points[N,3]) -> mean squared distance to the 3 nearest neighbours

``install()`` appends this directory to ``sys.path`` -- AFTER site-packages, so a real installation of any of the four
always wins -- and makes the repository root importable so that ``litegs_fused`` and ``fused_ssim`` resolve to this
implementation.  Nothing in ``litegs_b200`` itself imports these shims."""
from __future__ import annotations

import importlib.util
import os
import sys

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(os.path.dirname(_HERE))
NAMES = ("plyfile", "torchmetrics", "matplotlib", "simple_knn")


def install(verbose: bool = False) -> list:
    """Make the shims importable for the modules that are really missing; returns the names that were shimmed."""
    missing = [n for n in NAMES if n not in sys.modules and importlib.util.find_spec(n) is None]
    if missing and _HERE not in sys.path:
        sys.path.append(_HERE)                       # after site-packages: real packages take precedence
    if _ROOT not in sys.path:
        sys.path.insert(0, _ROOT)                    # litegs_fused.py / fused_ssim.py live at the repository root
    if verbose:
        print(f"[litegs_b200.shims] standing in for: {', '.join(missing) if missing else 'nothing (all installed)'}")
    return missing
