"""CPU restatement of the depth mode in numpy (fp32 or fp64), for the depth tests.

The mode (DESIGN.md section 1, "Depth") renders D = sum_i w_i z_i with the colour's blend weights w_i and the view-space z_i.
That is the oracle's own composite with the colour replaced by z: ``depth_forward`` draws the colour (z / zs, 0, 0) with zs a
power of two above every z, so the composite stays below the min(c, 1) clamp and scaling back by zs is exact.  Both channels
use the same weights, so the backward is the sum of the oracle's colour backward and the same backward of that depth-as-colour
image; its colour gradient is sum_pixels w g_z = dL/dz (times zs), which joins the view-space z gradient of the position and the
camera.  tests/fused_oracle.py renders D and adds that backward.  The oracle library itself has no depth mode.
"""
import numpy as np

import oracle


def _zscale(z):
    m = float(np.abs(z).max()) if z.size else 1.0
    return 2.0 ** (int(np.ceil(np.log2(max(m, 1e-30)))) + 1)


def depth_colour(z, dt):
    """(the colour [1,3,N] whose composite is D / zs, zs) for view-space z [N]."""
    zs = _zscale(z)
    col = np.zeros((1, 3, z.shape[-1]), dt)
    col[0, 0] = (z / zs).astype(dt)
    return col, zs


def depth_forward(sorted_pid, ranges, ndc, inv_cov2d, opacity, z, H, W, th, tw, specific_tiles=None):
    """D [V,1,Hp,Wp] of the records (ndc, inv_cov2d, opacity) with view-space z [N] over the given tile lists."""
    col, zs = depth_colour(z, ndc.dtype)
    img = oracle.rasterize_forward(sorted_pid, ranges, ndc, inv_cov2d, col, opacity, specific_tiles, H, W, th, tw)[0]
    return img[:, :1] * zs
