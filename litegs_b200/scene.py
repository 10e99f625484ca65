"""Synthetic scenes and cameras for parity tests and ``bench.py`` (numpy, no GPU needed).

Follows the input specification of BASELINE.md ("Synthetic inputs"): seed 0, N Gaussians uniform in
[-1,1]^3, cameras on a radius-3 Fibonacci sphere looking at the origin, fov_x 60 deg, z_near 0.01,
z_far 5000, log-scale ~ U(ln 0.002, ln 0.02), quaternion ~ N(0,1), opacity logit ~ U(-2,4),
sh_0 ~ N(0,1), sh_rest ~ N(0,0.1), sh_degree 3.

Conventions are the reference's (DX style, row vectors): ``p_view = p_world @ view_matrix`` and
``p_hom = p_view @ proj_matrix``; both matrices are the transposes of the COLMAP/OpenGL ones
(reference ``litegs/data.py:13,43-46,77``).  Parameters are kept in the reference's clustered layout
``[..., chunks, chunk_size]`` (``litegs/scene/cluster.py:7-22``).
"""
from __future__ import annotations

import math

import numpy as np


def look_at_view_matrix(eye: np.ndarray, target=(0.0, 0.0, 0.0), up=(0.0, 1.0, 0.0)) -> np.ndarray:
    """World->camera, camera looks along +z with y down (COLMAP); returned in row-vector form [4,4]."""
    eye = np.asarray(eye, np.float64)
    f = np.asarray(target, np.float64) - eye
    f /= np.linalg.norm(f)
    upv = np.asarray(up, np.float64)
    if abs(np.dot(f, upv)) > 0.999:
        upv = np.array([1.0, 0.0, 0.0])
    r = np.cross(f, upv); r /= np.linalg.norm(r)      # camera +x
    d = np.cross(f, r)                                  # camera +y (down)
    R = np.stack([r, d, f], axis=0)                     # rows: camera axes in world coords
    t = -R @ eye
    Rt = np.eye(4)
    Rt[:3, :3] = R
    Rt[:3, 3] = t
    return Rt.T.astype(np.float32)                      # row-vector convention


def proj_matrix(width: int, height: int, fov_x_deg: float = 60.0, z_near: float = 0.01, z_far: float = 5000.0) -> np.ndarray:
    """Reference ``PinHoleCameraInfo`` (litegs/data.py:33-51) with square pixels; row-vector form."""
    fx = 1.0 / math.tan(math.radians(fov_x_deg) * 0.5)          # recp_tan_half_fov_x
    fy = fx * width / height
    P = np.array([[fx, 0, 0, 0],
                  [0, fy, 0, 0],
                  [0, 0, z_far / (z_far - z_near), -z_far * z_near / (z_far - z_near)],
                  [0, 0, 1, 0]], dtype=np.float32)
    return P.T.copy()


def frustum_planes(view: np.ndarray, proj: np.ndarray) -> np.ndarray:
    """Six planes from the view-projection matrix, reference litegs/data.py:139-177; [6,4]."""
    vp = view.astype(np.float32) @ proj.astype(np.float32)
    fp = np.zeros((6, 4), np.float32)
    for k in range(4):
        fp[0, k] = vp[k, 3] + vp[k, 0]
        fp[1, k] = vp[k, 3] - vp[k, 0]
        fp[2, k] = vp[k, 3] + vp[k, 1]
        fp[3, k] = vp[k, 3] - vp[k, 1]
        fp[4, k] = vp[k, 2]
        fp[5, k] = vp[k, 3] - vp[k, 2]
    return fp


def fibonacci_camera(i: int, n: int, radius: float = 3.0) -> np.ndarray:
    """Eye position of view i out of n on the Fibonacci lattice."""
    golden = math.pi * (3.0 - math.sqrt(5.0))
    y = 1.0 - 2.0 * (i + 0.5) / n
    r = math.sqrt(max(0.0, 1.0 - y * y))
    th = golden * i
    return radius * np.array([math.cos(th) * r, y, math.sin(th) * r])


def make_camera(i: int, n_views: int, width: int, height: int, radius: float = 3.0, fov_x_deg: float = 60.0):
    """dict(view [1,4,4], proj [1,4,4], frustumplane [1,6,4]) for lattice view i."""
    V = look_at_view_matrix(fibonacci_camera(i, n_views, radius))
    P = proj_matrix(width, height, fov_x_deg)
    return dict(view=V[None].copy(), proj=P[None].copy(), frustumplane=frustum_planes(V, P)[None].copy())


def morton_order(xyz: np.ndarray, bits: int = 10) -> np.ndarray:
    """Stable Morton-code order of points [3,N] (what the reference's spatial_refine establishes)."""
    lo = xyz.min(axis=1, keepdims=True); hi = xyz.max(axis=1, keepdims=True)
    q = ((xyz - lo) / np.maximum(hi - lo, 1e-12) * ((1 << bits) - 1)).astype(np.int64)
    code = np.zeros(xyz.shape[1], np.int64)
    for b in range(bits):
        code |= ((q[0] >> b) & 1) << (3 * b) | ((q[1] >> b) & 1) << (3 * b + 1) | ((q[2] >> b) & 1) << (3 * b + 2)
    return np.argsort(code, kind="stable")


def cluster(a: np.ndarray, chunk: int) -> np.ndarray:
    """[...,N] -> [...,chunks,chunk]; the tail chunk is padded by repeating trailing points
    (reference litegs/scene/cluster.py:7-22)."""
    n = a.shape[-1]
    pad = (-n) % chunk
    if pad:
        a = np.concatenate([a, a[..., -pad:]], axis=-1)
    return np.ascontiguousarray(a.reshape(*a.shape[:-1], a.shape[-1] // chunk, chunk))


def quat_to_R(q: np.ndarray) -> np.ndarray:
    """Unit quaternion (r,x,y,z) [4,N] -> [3,3,N], reference wrapper.py:198-220."""
    r, x, y, z = q
    return np.stack([
        np.stack([1 - 2 * (y * y + z * z), 2 * (x * y + r * z), 2 * (x * z - r * y)]),
        np.stack([2 * (x * y - r * z), 1 - 2 * (x * x + z * z), 2 * (y * z + r * x)]),
        np.stack([2 * (x * z + r * y), 2 * (y * z - r * x), 1 - 2 * (x * x + y * y)]),
    ])


def cluster_aabb(xyz_c: np.ndarray, scale_c: np.ndarray, rot_c: np.ndarray, filter_3d=None):
    """Chunk AABBs from raw (log-scale, unnormalised quaternion) clustered params;
    semantics of reference litegs/scene/cluster.py:29-46 -> (origin [3,C], extend [3,C]).
    filter_3d ([1,C,S] or None): the boxes cover the splats widened by the 3D smoothing filter, scale sqrt(s^2 + f^2)."""
    C, S = xyz_c.shape[-2:]
    xyz = xyz_c.reshape(3, -1).astype(np.float64)
    s = np.exp(scale_c.reshape(3, -1).astype(np.float64))
    if filter_3d is not None:
        s = np.sqrt(s * s + np.asarray(filter_3d, np.float64).reshape(1, -1) ** 2)
    q = rot_c.reshape(4, -1).astype(np.float64)
    q = q / np.linalg.norm(q, axis=0, keepdims=True)
    T = quat_to_R(q) * s[:, None, :]
    ext = np.abs(T * math.sqrt(2 * math.log(255))).sum(axis=0)
    hi = (xyz + ext).reshape(3, C, S).max(-1)
    lo = (xyz - ext).reshape(3, C, S).min(-1)
    return ((hi + lo) / 2).astype(np.float32), ((hi - lo) / 2).astype(np.float32)


def cluster_aabb_torch(xyz_c, scale_c, rot_c, filter_3d=None):
    """cluster_aabb on torch tensors of any device (the chunk maintenance step of a training loop: positions and shapes
    move, the culling boxes follow without a host round trip).  Same semantics, float32 -> (origin [3,C], extend [3,C]).
    filter_3d ([1,C,S] or None): as in cluster_aabb."""
    import torch
    C, S = xyz_c.shape[-2:]
    xyz = xyz_c.reshape(3, -1).float()
    s = torch.exp(scale_c.reshape(3, -1).float())
    if filter_3d is not None:
        s = torch.sqrt(s * s + filter_3d.reshape(1, -1).float().square())
    q = rot_c.reshape(4, -1).float()
    q = q / q.norm(dim=0, keepdim=True)
    r, x, y, z = q[0], q[1], q[2], q[3]
    R = torch.stack([torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y + r * z), 2 * (x * z - r * y)]),
                     torch.stack([2 * (x * y - r * z), 1 - 2 * (x * x + z * z), 2 * (y * z + r * x)]),
                     torch.stack([2 * (x * z + r * y), 2 * (y * z - r * x), 1 - 2 * (x * x + y * y)])])          # [3,3,N], as quat_to_R
    ext = (R * s[:, None, :] * math.sqrt(2 * math.log(255))).abs().sum(dim=0)
    hi = (xyz + ext).reshape(3, C, S).amax(-1)
    lo = (xyz - ext).reshape(3, C, S).amin(-1)
    return ((hi + lo) * 0.5).contiguous(), ((hi - lo) * 0.5).contiguous()


def make_scene(n: int, sh_degree: int = 3, chunk: int = 128, seed: int = 0, log_scale_range=(0.002, 0.02),
               morton: bool = True, cube: float = 1.0, sh_rest_sigma: float = 0.1):
    """Random clustered Gaussian parameters following BASELINE.md.  Returns a dict of float32 arrays
    xyz[3,C,S] scale[3,C,S] rot[4,C,S] sh_0[1,3,C,S] sh_rest[K-1,3,C,S] opacity[1,C,S] plus the chunk
    AABBs and the true point count."""
    rng = np.random.default_rng(seed)
    K = (sh_degree + 1) ** 2
    xyz = rng.uniform(-cube, cube, (3, n))
    if morton:
        xyz = xyz[:, morton_order(xyz)]
    scale = rng.uniform(math.log(log_scale_range[0]), math.log(log_scale_range[1]), (3, n))
    rot = rng.normal(size=(4, n))
    opacity = rng.uniform(-2.0, 4.0, (1, n))
    sh_0 = rng.normal(size=(1, 3, n))
    sh_rest = rng.normal(scale=sh_rest_sigma, size=(max(K - 1, 0), 3, n))
    p = dict(xyz=xyz, scale=scale, rot=rot, sh_0=sh_0, sh_rest=sh_rest, opacity=opacity)
    p = {k: cluster(v.astype(np.float32), chunk) for k, v in p.items()}
    origin, extend = cluster_aabb(p["xyz"], p["scale"], p["rot"])
    p["cluster_origin"] = origin
    p["cluster_extend"] = extend
    p["n_points"] = n
    return p


# ---------------------------------------------------------------------------------------------------
# chunk maintenance on the device (SURVEY 8f rank 4): Morton re-clustering and chunk AABBs as single kernels
# ---------------------------------------------------------------------------------------------------

def cluster_aabb_device(xyz_c, scale_c, rot_c):
    """get_cluster_AABB (litegs/scene/cluster.py:29-46) in one kernel (csrc/scene.cu) from the RAW clustered parameters
    xyz/scale [3,C,S], rot [4,C,S] (float32 CUDA) -> (origin [3,C], extend [3,C])."""
    import torch
    from . import _lib
    from .fused import _f32c, _ptr, _stream
    x, s, q = _f32c(xyz_c.detach(), "xyz"), _f32c(scale_c.detach(), "scale"), _f32c(rot_c.detach(), "rot")
    C, S = x.shape[-2:]
    dev = x.device
    with torch.cuda.device(dev):
        origin = torch.empty((3, C), dtype=torch.float32, device=dev)
        extend = torch.empty((3, C), dtype=torch.float32, device=dev)
        _lib.call("lgs_cluster_aabb", _ptr(x), _ptr(s), _ptr(q), C, S, _ptr(origin), _ptr(extend), _stream(dev))
    return origin, extend


def filter_3d_device(xyz_c, views, projs, hw, out=None):
    """Mip-Splatting's 3D smoothing filter (compute_3D_filter) in two kernels (csrc/scene.cu, DESIGN.md section 1): xyz_c
    f32[3,C,S] on CUDA (every slot, the tail padding included), the training cameras views / projs f32[V,4,4] (row-vector
    convention) and hw (V image sizes (height, width): i32[V,2] tensor or sequence) -> f32[1,C,S], no gradient.

    out: an f32[1,C,S] tensor to write in place (keeps the data pointer, so CUDA graphs captured with it stay valid).  No host
    synchronisation: it can run inside a training step."""
    import torch
    from . import _lib
    from .fused import _f32c, _ptr, _stream
    x = _f32c(xyz_c.detach(), "xyz")
    C, S = x.shape[-2:]
    dev = x.device
    V = _f32c(views.detach().to(dev), "views").reshape(-1, 4, 4)
    P = _f32c(projs.detach().to(dev), "projs").reshape(-1, 4, 4)
    hw_t = torch.as_tensor(hw, dtype=torch.int32).to(dev).reshape(-1, 2).contiguous()
    nv = V.shape[0]
    if nv < 1 or P.shape[0] != nv or hw_t.shape[0] != nv:
        raise RuntimeError(f"filter_3d_device: {V.shape[0]} views, {P.shape[0]} projections and {hw_t.shape[0]} image sizes")
    if out is None:
        out = torch.empty((1, C, S), dtype=torch.float32, device=dev)
    elif not (out.device == dev and out.dtype == torch.float32 and out.is_contiguous() and out.numel() == C * S):
        raise RuntimeError(f"filter_3d_device: out must be a contiguous float32 tensor of {C * S} elements on {dev}")
    with torch.cuda.device(dev):
        _lib.call("lgs_filter_3d", _ptr(x), C, S, _ptr(V), _ptr(P), _ptr(hw_t), nv, _ptr(out), _stream(dev))
    return out


def morton_codes_device(xyz, bits: int = 21):
    """_gen_morton_code (litegs/scene/point.py:38-81) for xyz f32[3,N] on CUDA -> int64[N]."""
    import torch
    from . import _lib
    from .fused import _f32c, _ptr, _stream
    p = _f32c(xyz.detach(), "xyz")
    if p.dim() != 2 or p.shape[0] != 3:
        raise RuntimeError("positions must be a (3, N) tensor")
    dev, N = p.device, p.shape[1]
    with torch.cuda.device(dev):
        lo = p.amin(dim=1).contiguous()
        hi = p.amax(dim=1).contiguous()
        codes = torch.empty(N, dtype=torch.int64, device=dev)
        _lib.call("lgs_morton_codes", _ptr(p), _ptr(lo), _ptr(hi), N, int(bits), _ptr(codes), _stream(dev))
    return codes


def spatial_refine_device(tensors: dict, xyz_key: str = "xyz"):
    """spatial_refine (litegs/scene/point.py:85-154) for clustered tensors: every entry of `tensors` is [..., C, S] float32 CUDA
    (parameters, their gradients, Adam moments ...); all are re-ordered by the stable Morton order of tensors[xyz_key] and
    re-clustered.  Returns (dict of new tensors, the permutation int64[C*S]).  Each tensor is permuted by ONE launch."""
    import torch
    from . import _lib
    from .fused import _f32c, _ptr, _stream
    xyz = tensors[xyz_key]
    C, S = xyz.shape[-2:]
    N = C * S
    dev = xyz.device
    codes = morton_codes_device(xyz.detach().reshape(3, N))
    _, order = codes.sort(stable=True)                                     # point.py:92 (torch.sort: integer keys, exact)
    out = {}
    with torch.cuda.device(dev):
        for k, t in tensors.items():
            src = _f32c(t.detach(), k)
            if tuple(src.shape[-2:]) != (C, S):
                raise RuntimeError(f"spatial_refine_device: '{k}' is not clustered like '{xyz_key}'")
            R = src.numel() // N
            dst = torch.empty_like(src)
            _lib.call("lgs_permute_rows", _ptr(src), _ptr(order), R, N, _ptr(dst), _stream(dev))
            out[k] = dst
    return out, order
