"""Render a 3DGS point cloud (.ply, the layout shared by every 3DGS code base) with the fused forward pipeline.

    python examples/render_ply.py --ply point_cloud.ply --out /tmp/renders --views 8 [--colmap /path/to/colmap]
    python examples/render_ply.py --make /tmp/demo.ply --out /tmp/renders        # writes a synthetic cloud first
    python examples/render_ply.py --ply mip_splatting.ply --filter-3d --antialiased    # a Mip-Splatting checkpoint
    python examples/render_ply.py --make /tmp/demo.ply --out /tmp/renders --depth      # also depth maps (e.g. for TSDF fusion)
    python examples/render_ply.py --ply point_cloud.ply --depth-normal                  # also the normals of the rendered depth

Cameras: the poses of a COLMAP model when --colmap is given, else the Fibonacci lattice of scene.make_camera.  Forward only
(the reference's example_metrics.py path): project -> bin -> sort -> composite, no gradients kept.  With --depth each view also
writes <name>_depth.npy (D = sum w z, the accumulated view-space depth, f32[H,W]) and <name>_alpha.npy (1 - T, f32[H,W]); the
expected depth is D / alpha where alpha > 0.  With --normal each view also writes <name>_normal.npy, the expected view-space
normal N / (1 - T) (f32[3,H,W], zero where nothing was blended; DESIGN.md section 1, "Normals").  With --depth-normal each view
also writes <name>_depth_normal.npy, the unit view-space normal n_d of the surface the expected depth unprojects to (f32[3,H,W],
zero where it is undefined: the border, 1 - T <= 0.5 at the pixel or a neighbour; DESIGN.md section 1, "Depth-normal consistency").
"""
import argparse
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from litegs_b200 import colmap, geometry, pipeline, ply, scene  # noqa: E402
from litegs_b200.dist import PARAM_ORDER  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ply", default=None)
    ap.add_argument("--make", default=None, help="write a synthetic cloud to this .ply first")
    ap.add_argument("--colmap", default=None)
    ap.add_argument("--out", default="renders")
    ap.add_argument("--views", type=int, default=8)
    ap.add_argument("--width", type=int, default=960)
    ap.add_argument("--height", type=int, default=540)
    ap.add_argument("--sh-degree", type=int, default=3)
    ap.add_argument("--antialiased", action="store_true",
                    help="opacity compensation of the 2D filter (for models trained in that mode, or renders at another resolution)")
    ap.add_argument("--filter-3d", action="store_true",
                    help="apply the file's filter_3D property (Mip-Splatting's 3D smoothing filter); the file must have it")
    ap.add_argument("--depth", action="store_true", help="also write the accumulated depth D and 1 - T of each view as .npy")
    ap.add_argument("--normal", action="store_true", help="also write the expected view-space normal N / (1 - T) of each view as .npy")
    ap.add_argument("--depth-normal", action="store_true", help="also write the normal n_d of the rendered expected depth of each view as .npy")
    a = ap.parse_args()
    path = a.ply
    if a.make:
        sc = scene.make_scene(200_000, sh_degree=3, seed=0)
        ply.params_to_ply(a.make, sc)
        path = a.make
    if path is None:
        ap.error("give --ply or --make")
    dev = torch.device("cuda:0")
    g = ply.params_from_ply(path, a.sh_degree)
    P = {k: torch.from_numpy(g[k]).to(dev) for k in PARAM_ORDER}
    A = [torch.from_numpy(g[k]).to(dev) for k in ("cluster_origin", "cluster_extend")]
    filt = None
    if a.filter_3d:
        if "filter_3D" not in g:
            ap.error(f"--filter-3d: {path} has no filter_3D property")
        filt = torch.from_numpy(g["filter_3D"]).to(dev)
        A = list(scene.cluster_aabb_torch(P["xyz"], P["scale"], P["rot"], filter_3d=filt))       # boxes of the widened splats
    cams = []
    if a.colmap:
        cs, ims, _ = colmap.read_model(a.colmap)
        for im in sorted(ims.values(), key=lambda v: v.name)[: a.views]:
            c = cs[im.camera_id]
            cams.append((colmap.camera_from_colmap(im.qvec, im.tvec, c.params, c.width, c.height), (c.height, c.width), im.name))
    else:
        cams = [(scene.make_camera(i, a.views, a.width, a.height), (a.height, a.width), f"view_{i:04d}.png") for i in range(a.views)]
    import PIL.Image
    os.makedirs(a.out, exist_ok=True)
    imgs, depths, normals, depth_normals = [], [], [], []
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    with torch.no_grad():
        for cam, hw, _ in cams:
            c = {k: torch.from_numpy(v).to(dev) for k, v in cam.items()}
            img, st, _ = pipeline.render_view_forward(P, A[0], A[1], c["frustumplane"], c["view"], c["proj"], a.sh_degree, hw, (8, 16),
                                                      clamp_zero=True, antialiased=a.antialiased, filter_3d=filt,
                                                      render_depth=a.depth or a.depth_normal, render_normal=a.normal)
            imgs.append(img[0, :, : hw[0], : hw[1]])
            if a.depth:
                depths.append((st.depth[0, 0, : hw[0], : hw[1]], 1.0 - st.T[0, 0, : hw[0], : hw[1]]))
            if a.normal:
                alpha = 1.0 - st.T[0, :, : hw[0], : hw[1]]
                nrm = st.normal[0, :, : hw[0], : hw[1]]
                normals.append(torch.where(alpha > 0, nrm / alpha.clamp_min(1e-12), torch.zeros_like(nrm)))
            if a.depth_normal:
                depth_normals.append(geometry.depth_normal(st.depth[..., : hw[0], : hw[1]], st.T[..., : hw[0], : hw[1]], c["proj"])[0][0])
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    for (cam, hw, name), img in zip(cams, imgs):
        PIL.Image.fromarray((img.permute(1, 2, 0) * 255.0 + 0.5).clamp(0, 255).to(torch.uint8).cpu().numpy()).save(
            os.path.join(a.out, os.path.splitext(name)[0] + ".png"))
    for (_, _, name), (d, alpha) in zip(cams, depths):
        np.save(os.path.join(a.out, os.path.splitext(name)[0] + "_depth.npy"), d.cpu().numpy())
        np.save(os.path.join(a.out, os.path.splitext(name)[0] + "_alpha.npy"), alpha.cpu().numpy())
    for (_, _, name), en in zip(cams, normals):
        np.save(os.path.join(a.out, os.path.splitext(name)[0] + "_normal.npy"), en.cpu().numpy())
    for (_, _, name), nd in zip(cams, depth_normals):
        np.save(os.path.join(a.out, os.path.splitext(name)[0] + "_depth_normal.npy"), nd.cpu().numpy())
    print(f"{g['n_points']} Gaussians, {len(cams)} views rendered in {dt * 1e3:.1f} ms ({len(cams) / dt:.0f} views/s forward only) -> {a.out}")


if __name__ == "__main__":
    main()
