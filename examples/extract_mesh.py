"""Extract a triangle mesh from a 3DGS point cloud (.ply): render the expected depth of every camera, fuse it into a TSDF volume
and run marching tetrahedra, on the GPU (litegs_b200.mesh, DESIGN.md section 1, "Mesh extraction").

    python examples/extract_mesh.py --ply point_cloud.ply --colmap /path/to/colmap --out mesh.ply
    python examples/extract_mesh.py --ply point_cloud.ply --views 64 --width 960 --height 540 --resolution 384
    python examples/extract_mesh.py --ply surface.ply --colmap DIR --bounds -2 -2 -2 2 2 2 --sdf-trunc 4 --depth-far 6

Cameras: the poses of a COLMAP model when --colmap is given, else the Fibonacci lattice of scene.make_camera (as render_ply.py).
The volume has --resolution lattice points along the longest axis of --bounds (default: the box of the Gaussian centres padded by
twice the truncation distance on every side); --sdf-trunc is the truncation distance in voxels.  The mesh is written as a binary
PLY with vertex colours (MeshLab, Open3D and Blender read it).
"""
import argparse
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from litegs_b200 import colmap, mesh, ply, scene  # noqa: E402
from litegs_b200.arguments import PipelineParams  # noqa: E402
from litegs_b200.dist import PARAM_ORDER  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ply", required=True)
    ap.add_argument("--colmap", default=None)
    ap.add_argument("--views", type=int, default=64, help="lattice cameras (without --colmap), or the first N COLMAP images")
    ap.add_argument("--width", type=int, default=960)
    ap.add_argument("--height", type=int, default=540)
    ap.add_argument("--sh-degree", type=int, default=3)
    ap.add_argument("--resolution", type=int, default=512, help="lattice points along the longest axis of the volume")
    ap.add_argument("--bounds", type=float, nargs=6, default=None, metavar=("X0", "Y0", "Z0", "X1", "Y1", "Z1"))
    ap.add_argument("--sdf-trunc", type=float, default=5.0, help="truncation distance in voxels")
    ap.add_argument("--depth-far", type=float, default=float("inf"), help="skip expected depths beyond this")
    ap.add_argument("--alpha-min", type=float, default=0.5, help="skip pixels with 1 - T at or below this")
    ap.add_argument("--batch", type=int, default=16, help="views fused per launch")
    ap.add_argument("--antialiased", action="store_true", help="render with the antialiased mode's opacity compensation")
    ap.add_argument("--filter-3d", action="store_true", help="apply the file's filter_3D property (Mip-Splatting)")
    ap.add_argument("--out", default="mesh.ply")
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    g = ply.params_from_ply(a.ply, a.sh_degree)
    P = {k: torch.from_numpy(g[k]).to(dev) for k in PARAM_ORDER}
    filt = None
    if a.filter_3d:
        if "filter_3D" not in g:
            ap.error(f"--filter-3d: {a.ply} has no filter_3D property")
        filt = torch.from_numpy(g["filter_3D"]).to(dev)
    P["cluster_origin"], P["cluster_extend"] = scene.cluster_aabb_torch(P["xyz"], P["scale"], P["rot"], filter_3d=filt)
    if a.colmap:
        cs, ims, _ = colmap.read_model(a.colmap)
        cams = []
        for im in sorted(ims.values(), key=lambda v: v.name)[: a.views]:
            c = cs[im.camera_id]
            cams.append((colmap.camera_from_colmap(im.qvec, im.tvec, c.params, c.width, c.height), (c.height, c.width)))
        if len({hw for _, hw in cams}) > 1:
            ap.error("--colmap: the images have different sizes; mesh extraction fuses one image size")
        hw = cams[0][1]
        cams = [c for c, _ in cams]
    else:
        hw = (a.height, a.width)
        cams = [scene.make_camera(i, a.views, a.width, a.height) for i in range(a.views)]
    cams = [{k: torch.from_numpy(v).to(dev) for k, v in c.items()} for c in cams]
    vol = mesh.bounding_volume(P["xyz"].reshape(3, -1)[:, : g["n_points"]], resolution=a.resolution, trunc_voxels=a.sdf_trunc,
                               bounds=a.bounds)
    pp = PipelineParams(tile_size=(8, 16), antialiased=a.antialiased)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    mesh.mesh_from_views(P, cams, hw, pp, vol, batch=a.batch, filter_3d=filt, alpha_min=a.alpha_min, depth_far=a.depth_far)
    torch.cuda.synchronize()
    t1 = time.perf_counter()
    v, f, c = vol.extract()
    torch.cuda.synchronize()
    t2 = time.perf_counter()
    ply.save_mesh_ply(a.out, v, f, c)
    nx, ny, nz = vol.dims
    print(f"{len(cams)} views {hw[1]}x{hw[0]} fused into {nx}x{ny}x{nz} (voxel {vol.voxel_size:.4g}, truncation {vol.sdf_trunc:.4g}) "
          f"in {(t1 - t0) * 1e3:.1f} ms (rendering included), extracted in {(t2 - t1) * 1e3:.1f} ms: {len(v)} vertices, {len(f)} faces "
          f"-> {a.out}")


if __name__ == "__main__":
    main()
