"""Mesh extraction from the rendered expected depth, on the kernels of csrc/mesh.cu (DESIGN.md section 1, "Mesh extraction"):
TSDF fusion of batches of views into a dense lattice and marching tetrahedra on its cells, the last step of the 2DGS / PGSR
surface-reconstruction recipe.

    vol = TSDFVolume(origin, voxel_size, dims, sdf_trunc=None, color=True)
    vol.integrate(depth, trans, views, projs, rgb=None, alpha_min=0.5, depth_far=inf)     # one launch per batch of V views
    vertices, faces, colors = vol.extract(weight_min=1.0)                                  # f32[M,3], i32[F,3], u8[M,3] or None
    mesh_from_views(params, cameras, hw, pp, vol, batch=16, filter_3d=None)               # render + integrate every camera

depth, trans: the depth mode's D and the transmittance T, f32[V,1,H,W]; rgb: the rendered images f32[V,3,H,W]; views, projs:
f32[V,4,4] (row-vector convention).  The mesh is closed where the volume was observed, wound with its normals toward free space,
and in a canonical order (vertices by lattice point and edge, faces by cell, tetrahedron and triangle), so the same volume always
gives the same arrays.  CUDA float32 only; there is no CPU path.
"""
from __future__ import annotations

import copy
import math

import torch

from . import _lib, render, scene
from .fused import _on, _ptr, _stream

_MAX_POINTS = (1 << 31) - 1


def _tensor(t, name: str, shape, dev) -> torch.Tensor:
    """t as a contiguous float32 CUDA tensor of the given shape on dev (entries None in shape: any size)."""
    if not isinstance(t, torch.Tensor):
        raise RuntimeError(f"mesh (litegs_b200): {name} must be a torch tensor, got {type(t).__name__}")
    if not t.is_cuda or t.dtype != torch.float32:
        raise RuntimeError(f"mesh (litegs_b200): {name} must be a float32 CUDA tensor, got {t.dtype} on {t.device}")
    if t.dim() != len(shape) or any(s is not None and t.shape[d] != s for d, s in enumerate(shape)):
        want = "[" + ",".join("?" if s is None else str(s) for s in shape) + "]"
        raise RuntimeError(f"mesh (litegs_b200): {name} must be {want}, got {list(t.shape)}")
    if t.device != dev:
        raise RuntimeError(f"mesh (litegs_b200): {name} is on {t.device}, the volume on {dev}")
    return t.contiguous()


class TSDFVolume:
    """A dense TSDF volume of dims = (nx, ny, nz) lattice points, x fastest; point (i, j, k) sits at origin + (i, j, k) voxel_size.
    tsdf f32[nz,ny,nx] starts at 1, weight f32[nz,ny,nx] at 0 and, with color=True, color f32[3,nz,ny,nx] at 0.  sdf_trunc is
    the truncation distance in world units (default 5 voxel_size, as 2DGS)."""

    def __init__(self, origin, voxel_size: float, dims, sdf_trunc: float | None = None, color: bool = True, device=None):
        dev = torch.device(device if device is not None else "cuda")
        if dev.type != "cuda":
            raise RuntimeError(f"TSDFVolume (litegs_b200): the volume lives on a CUDA device, got {dev}")
        if dev.index is None:
            dev = torch.device("cuda", torch.cuda.current_device())
        self.origin = tuple(float(x) for x in origin)
        self.dims = tuple(int(n) for n in dims)
        if len(self.origin) != 3 or len(self.dims) != 3:
            raise RuntimeError("TSDFVolume (litegs_b200): origin and dims need three entries each")
        if min(self.dims) < 1:
            raise RuntimeError(f"TSDFVolume (litegs_b200): dims {self.dims} must be positive")
        n = math.prod(self.dims)
        if n > _MAX_POINTS:
            raise RuntimeError(f"TSDFVolume (litegs_b200): {n} lattice points exceed 2^31 - 1")
        self.voxel_size = float(voxel_size)
        self.sdf_trunc = 5.0 * self.voxel_size if sdf_trunc is None else float(sdf_trunc)
        if not (self.voxel_size > 0 and self.sdf_trunc > 0 and math.isfinite(self.voxel_size) and math.isfinite(self.sdf_trunc)):
            raise RuntimeError(f"TSDFVolume (litegs_b200): voxel_size = {voxel_size} and sdf_trunc = {sdf_trunc} must be positive")
        self.device = dev
        nx, ny, nz = self.dims
        with _on(dev):
            self.tsdf = torch.ones((nz, ny, nx), dtype=torch.float32, device=dev)
            self.weight = torch.zeros((nz, ny, nx), dtype=torch.float32, device=dev)
            self.color = torch.zeros((3, nz, ny, nx), dtype=torch.float32, device=dev) if color else None

    def integrate(self, depth, trans, views, projs, rgb=None, alpha_min: float = 0.5, depth_far: float = math.inf) -> None:
        """Fuse V >= 1 views in one launch, in index order (the result is that of V single-view calls, bit for bit).  depth,
        trans f32[V,1,H,W]; views, projs f32[V,4,4]; rgb f32[V,3,H,W], required exactly when the volume has colour.  Pixels with
        1 - T <= alpha_min and expected depths D / (1 - T) beyond depth_far are skipped."""
        dev = self.device
        D = _tensor(depth, "depth", (None, 1, None, None), dev)
        V, _, H, W = D.shape
        if V < 1 or H < 1 or W < 1:
            raise RuntimeError(f"mesh (litegs_b200): depth must be a non-empty [V,1,H,W] batch, got {list(D.shape)}")
        T = _tensor(trans, "trans", (V, 1, H, W), dev)
        Vm = _tensor(views, "views", (V, 4, 4), dev)
        Pm = _tensor(projs, "projs", (V, 4, 4), dev)
        if (rgb is None) != (self.color is None):
            raise RuntimeError("mesh (litegs_b200): rgb is required for a volume with colour, and refused for one without")
        C = None if rgb is None else _tensor(rgb, "rgb", (V, 3, H, W), dev)
        if not 0.0 <= float(alpha_min) < 1.0:
            raise RuntimeError(f"mesh (litegs_b200): alpha_min = {alpha_min} outside [0, 1)")
        if not float(depth_far) > 0.0:
            raise RuntimeError(f"mesh (litegs_b200): depth_far = {depth_far} must be positive")
        with _on(dev):
            _lib.call("lgs_tsdf_integrate", _ptr(self.tsdf), _ptr(self.weight), _ptr(self.color), *self.dims, *self.origin,
                      self.voxel_size, self.sdf_trunc, _ptr(D), _ptr(T), _ptr(C), _ptr(Vm), _ptr(Pm), V, H, W, float(alpha_min),
                      float(depth_far), _stream(dev))

    def extract(self, weight_min: float = 1.0):
        """Marching tetrahedra over the cells whose 8 corners all have weight >= weight_min -> (vertices f32[M,3], faces i32[F,3],
        colors u8[M,3] or None for a volume without colour).  Reads the two totals back once (an offline step); an empty or
        unobserved volume gives empty arrays."""
        dev = self.device
        N = self.tsdf.numel()
        with _on(dev):
            vmask = torch.empty(N, dtype=torch.uint8, device=dev)
            vcount = torch.empty(N, dtype=torch.uint8, device=dev)
            fcount = torch.empty(N, dtype=torch.uint8, device=dev)
            _lib.call("lgs_mesh_count", _ptr(self.tsdf), _ptr(self.weight), *self.dims, float(weight_min), _ptr(vmask), _ptr(vcount),
                      _ptr(fcount), _stream(dev))
            vert_end = torch.cumsum(vcount, 0, dtype=torch.int64)
            del vcount
            face_end = torch.cumsum(fcount, 0, dtype=torch.int64)
            M, F = (int(x) for x in torch.stack((vert_end[-1], face_end[-1])).tolist())
            check_totals(M, F)
            vertices = torch.empty((M, 3), dtype=torch.float32, device=dev)
            faces = torch.empty((F, 3), dtype=torch.int32, device=dev)
            colors = None if self.color is None else torch.empty((M, 3), dtype=torch.uint8, device=dev)
            _lib.call("lgs_mesh_emit", _ptr(self.tsdf), _ptr(self.color), *self.dims, *self.origin, self.voxel_size, _ptr(vmask),
                      _ptr(fcount), _ptr(vert_end), _ptr(face_end), M, F, _ptr(vertices), _ptr(faces), _ptr(colors), _stream(dev))
        return vertices, faces, colors


def check_totals(n_vertices: int, n_faces: int) -> None:
    """The mesh's vertex and face indices are int32: refuse totals of 2^31 or more before anything is allocated."""
    if n_vertices >= 1 << 31 or n_faces >= 1 << 31:
        raise RuntimeError(f"mesh (litegs_b200): {n_vertices} vertices and {n_faces} faces; int32 indices need both below 2^31 "
                           "(use a coarser or smaller volume)")


def bounding_volume(xyz, resolution: int = 512, trunc_voxels: float = 5.0, bounds=None, color: bool = True) -> TSDFVolume:
    """A TSDFVolume with `resolution` lattice points along the longest axis of bounds = (x0, y0, z0, x1, y1, z1); without bounds,
    the box of the points xyz (f32[3,...] CUDA) padded on every side by 2 sdf_trunc, where sdf_trunc = trunc_voxels voxels."""
    if resolution < 2:
        raise RuntimeError(f"mesh (litegs_b200): resolution = {resolution} must be at least 2")
    if bounds is None:
        p = xyz.detach().reshape(3, -1)
        lo, hi = p.amin(dim=1).double().tolist(), p.amax(dim=1).double().tolist()
        ext = max(h - l for l, h in zip(lo, hi))
        # (ext + 4 trunc_voxels h) / (resolution - 1) = h
        if resolution - 1 <= 4 * trunc_voxels:
            raise RuntimeError(f"mesh (litegs_b200): resolution = {resolution} leaves no room for a {trunc_voxels}-voxel truncation band")
        h = max(ext, 1e-6) / (resolution - 1 - 4 * trunc_voxels)
        pad = 2 * trunc_voxels * h
        lo, hi = [l - pad for l in lo], [x + pad for x in hi]
        device = xyz.device
    else:
        lo, hi = [float(b) for b in bounds[:3]], [float(b) for b in bounds[3:]]
        if len(lo) != 3 or len(hi) != 3 or any(b <= a for a, b in zip(lo, hi)):
            raise RuntimeError(f"mesh (litegs_b200): bounds {list(bounds)} must be x0 y0 z0 x1 y1 z1 with x0 < x1, y0 < y1, z0 < z1")
        h = max(b - a for a, b in zip(lo, hi)) / (resolution - 1)
        device = xyz.device if xyz is not None else None
    dims = [int(math.floor((b - a) / h + 1e-9)) + 1 for a, b in zip(lo, hi)]
    return TSDFVolume(lo, h, dims, sdf_trunc=trunc_voxels * h, color=color, device=device)


def mesh_from_views(params: dict, cameras, hw, pp, volume: TSDFVolume, batch: int = 16, filter_3d=None, alpha_min: float = 0.5,
                    depth_far: float = math.inf) -> TSDFVolume:
    """Render every camera forward only through render.render_view with the depth mode and the transmittance on, and fuse the
    views into volume, `batch` views per launch.  params: the six clustered parameter tensors (xyz, scale, rot, sh_0, sh_rest,
    opacity) and, optionally, cluster_origin / cluster_extend (computed from the parameters and filter_3d when absent); cameras:
    dicts of view [1,4,4], proj [1,4,4], frustumplane [1,6,4] on the device; hw = (H, W); pp: the pipeline parameters the model
    is drawn with (antialiased, tile size ...).  Returns volume."""
    if batch < 1:
        raise RuntimeError(f"mesh_from_views: batch = {batch} must be at least 1")
    H, W = int(hw[0]), int(hw[1])
    pp = copy.copy(pp)
    pp.render_depth = True
    pp.enable_transmitance = True
    if "cluster_origin" in params and "cluster_extend" in params:
        origin, extend = params["cluster_origin"], params["cluster_extend"]
    else:
        origin, extend = scene.cluster_aabb_torch(params["xyz"], params["scale"], params["rot"], filter_3d=filter_3d)
    deg = int(round(math.sqrt(params["sh_rest"].shape[0] + 1))) - 1
    args = [params[k] for k in ("xyz", "scale", "rot", "sh_0", "sh_rest", "opacity")]
    cams = list(cameras)
    with torch.no_grad():
        for b0 in range(0, len(cams), batch):
            outs = []
            for c in cams[b0:b0 + batch]:
                img, trans, depth, _, _ = render.render_view(origin, extend, c["frustumplane"], c["view"], c["proj"], *args, deg, (H, W), pp,
                                                             filter_3d=filter_3d)
                outs.append((img, trans, depth, c["view"].reshape(1, 4, 4), c["proj"].reshape(1, 4, 4)))
            img, trans, depth, views, projs = (torch.cat(x) for x in zip(*outs))
            volume.integrate(depth, trans, views, projs, rgb=img if volume.color is not None else None, alpha_min=alpha_min,
                             depth_far=depth_far)
    return volume
