"""From a COLMAP directory to a trained set of Gaussians on the litegs_b200 stack (BASELINE.json config 5 in spirit).

    python examples/train_colmap.py --make /tmp/synth_colmap          # writes a synthetic dataset first (renders of a hidden scene)
    python examples/train_colmap.py --data /path/to/colmap --iters 2000
    python examples/train_colmap.py --make /tmp/noisy --pose-noise 1 0.02 --refine-poses     # learn the camera poses too
    python examples/train_colmap.py --make /tmp/noisy --pose-noise 1 0.02 --refine-poses --exact-grad   # ... with the J and SH terms
    python examples/train_colmap.py --make /tmp/synth_depth --depth-weight 0.1     # also supervise the expected depth
    python examples/train_colmap.py --make /tmp/synth_normal --normal-weight 0.1   # also supervise the rendered normals
    python examples/train_colmap.py --data /path/to/colmap --depth-normal-weight 0.1   # self-supervised depth-normal consistency
    python examples/train_colmap.py --data /path/to/colmap --depth-normal-weight 0.1 --mesh mesh.ply   # ... and write a mesh

Reads ``sparse/0/{cameras,images,points3D}.bin`` and ``images/*`` (litegs_b200.colmap; same files and conventions as the
reference's ``litegs/io_manager/colmap.py`` + ``litegs/data.py``), initialises Gaussians from the SfM points the way
``litegs/scene/point.py:7-19`` does, and trains appearance + geometry with the fused L1+SSIM loss and the fused Adam step.
No densification (that policy is out of scope, SURVEY 2.1): the point count stays what COLMAP delivered.
With ``--depth-weight W`` and a ``depths/`` directory beside ``images/`` (``depths/<image stem>.npy``, f32[H,W] expected depth,
NaN where unknown -- ``--make`` writes the hidden scene's), the loss gains W * mean |ED - target| over the known pixels, with
ED = D / (1 - T) from the depth mode (DESIGN.md section 1, "Depth").
With ``--normal-weight W`` and a ``normals/`` directory (``normals/<image stem>.npy``, f32[3,H,W] unit view-space normal, NaN
where unknown -- ``--make`` writes the hidden scene's N / |N|), the loss gains W * mean(1 - cos(N / |N|, target)) over the known
pixels, with N from the normal mode (DESIGN.md section 1, "Normals"); it composes with ``--depth-weight``.
With ``--depth-normal-weight W`` the loss gains W * mean(1 - n_d . N / |N|), n_d the normal of the surface the rendered expected
depth unprojects to (litegs_b200.geometry, DESIGN.md section 1, "Depth-normal consistency"): it turns depth and normals on and
needs no ``depths/`` or ``normals/`` directory, so it trains the geometry of a real capture; it composes with every option above.
With ``--mesh PATH`` the trained model's expected depth from every training camera (the refined poses with ``--refine-poses``, the
3D filter with ``--filter-3d``) is fused into a TSDF volume over the Gaussian centres and written as a coloured triangle mesh
(litegs_b200.mesh, DESIGN.md section 1, "Mesh extraction").
"""
import argparse
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from litegs_b200 import colmap, dist as lgs_dist, geometry, mesh as lgs_mesh, optimizer, ply, render, scene, ssim  # noqa: E402
from litegs_b200.arguments import PipelineParams  # noqa: E402
from litegs_b200.dist import PARAM_ORDER  # noqa: E402


def make_dataset(root, n_gaussians=60_000, n_views=24, hw=(270, 480), n_points=20_000, seed=0, dev=None, log_scale_range=(0.01, 0.04),
                 pose_noise=None):
    """A hidden scene rendered from the lattice cameras -> COLMAP model + PNGs.  The 'SfM points' are a subsample of the
    hidden Gaussians' centres with their band-0 colours (what a real reconstruction would roughly deliver).

    pose_noise = (degrees, fraction): the poses written to the model are off by a rotation of that many degrees about a random
    axis and a translation of that fraction of the camera's distance, as noisy SfM poses are; the images stay exact."""
    dev = dev or torch.device("cuda:0")
    H, W = hw
    pp = PipelineParams(tile_size=(8, 16), sparse_grad=True, render_depth=True, enable_transmitance=True, render_normal=True)
    truth = scene.make_scene(n_gaussians, sh_degree=3, seed=seed, log_scale_range=log_scale_range)
    T = {k: torch.from_numpy(truth[k]).to(dev) for k in PARAM_ORDER}
    A = [torch.from_numpy(truth[k]).to(dev) for k in ("cluster_origin", "cluster_extend")]

    eds, nrms = {}, {}

    def render_fn(i, cam):
        c = {k: torch.from_numpy(v).to(dev) for k, v in cam.items()}
        with torch.no_grad():
            img, trans, depth, normal, _ = render.render_view(A[0], A[1], c["frustumplane"], c["view"], c["proj"], T["xyz"], T["scale"],
                                                              T["rot"], T["sh_0"], T["sh_rest"], T["opacity"], 3, (H, W), pp)
            alpha = 1.0 - trans[0, 0]
            # the hidden scene's expected depth and unit normal where it is mostly opaque, unknown elsewhere
            eds[i] = torch.where(alpha > 0.5, depth[0, 0] / alpha.clamp_min(0.5), torch.full_like(alpha, float("nan"))).cpu().numpy()
            un = normal[0] / normal[0].norm(dim=0, keepdim=True).clamp_min(1e-12)
            nrms[i] = torch.where(alpha[None] > 0.5, un, torch.full_like(un, float("nan"))).cpu().numpy()
        return (img[0].permute(1, 2, 0) * 255.0 + 0.5).clamp(0, 255).to(torch.uint8).cpu().numpy()

    rng = np.random.default_rng(seed + 7)
    xyz = truth["xyz"].reshape(3, -1).T
    sel = rng.choice(xyz.shape[0], size=min(n_points, xyz.shape[0]), replace=False)
    rgb = np.clip((truth["sh_0"].reshape(3, -1).T[sel] * colmap.SH_C0 + 0.5) * 255.0, 0, 255).astype(np.uint8)
    names = colmap.write_synthetic_dataset(root, xyz[sel].astype(np.float64), rgb, n_views, W, H, render_fn=render_fn)
    os.makedirs(os.path.join(root, "depths"), exist_ok=True)
    for i, name in enumerate(names):
        np.save(os.path.join(root, "depths", os.path.splitext(name)[0] + ".npy"), eds[i].astype(np.float32))
    os.makedirs(os.path.join(root, "normals"), exist_ok=True)
    for i, name in enumerate(names):
        np.save(os.path.join(root, "normals", os.path.splitext(name)[0] + ".npy"), nrms[i].astype(np.float32))
    if pose_noise is not None:
        deg, frac = pose_noise
        cams, images, pts = colmap.read_model(root)
        for k, im in images.items():
            axis = rng.normal(size=3)
            axis /= np.linalg.norm(axis)
            a = np.radians(deg)
            c, s_ = np.cos(a), np.sin(a)
            K = np.array([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]])
            dR = np.eye(3) + s_ * K + (1 - c) * K @ K
            d = rng.normal(size=3)
            t = np.asarray(im.tvec, np.float64)
            t = t + frac * np.linalg.norm(t) * d / np.linalg.norm(d)
            images[k] = im._replace(qvec=colmap.rotmat_to_qvec(dR @ colmap.qvec_to_rotmat(im.qvec)), tvec=t)
        colmap.write_model(root, cams, images, pts)
    return root


def load_dataset(root, image_dir="images", dev=None):
    import PIL.Image
    dev = dev or torch.device("cuda:0")
    cams, images, pts = colmap.read_model(root)
    frames = []
    for im in sorted(images.values(), key=lambda v: v.name):
        c = cams[im.camera_id]
        if c.model != "PINHOLE":
            continue                                     # as the reference (colmap.py:222-224)
        cam = colmap.camera_from_colmap(im.qvec, im.tvec, c.params, c.width, c.height)
        gt = np.array(PIL.Image.open(os.path.join(root, image_dir, im.name)).convert("RGB"), np.uint8)
        frames.append(({k: torch.from_numpy(v).to(dev) for k, v in cam.items()},
                       torch.from_numpy(gt).to(dev).permute(2, 0, 1)[None].float().div_(255.0).contiguous(), (c.height, c.width)))
    P = list(pts.values())
    return frames, np.stack([p.xyz for p in P]), np.stack([p.rgb for p in P])


def load_depths(root, dev=None, sub="depths"):
    """Expected-depth targets f32[1,1,H,W] (NaN = unknown) aligned with load_dataset's frames, from root/depths/<image stem>.npy;
    None when the dataset has no depths directory.  sub="normals": the unit-normal targets f32[1,3,H,W] of root/normals."""
    if not os.path.isdir(os.path.join(root, sub)):
        return None
    dev = dev or torch.device("cuda:0")
    cams, images, _ = colmap.read_model(root)
    out = []
    for im in sorted(images.values(), key=lambda v: v.name):
        if cams[im.camera_id].model != "PINHOLE":
            continue
        d = np.load(os.path.join(root, sub, os.path.splitext(im.name)[0] + ".npy")).astype(np.float32)
        d = d[None] if d.ndim == 2 else d
        out.append(torch.from_numpy(d).to(dev)[None].contiguous())
    return out


def normal_loss_and_grad(normal, target, weight, upstream=1.0):
    """weight * mean(1 - cos(N / |N|, target)) over the pixels with a finite target and |N| > 1e-6 -> (loss, d_normal) with the
    gradient scaled by upstream; also the mean angle in degrees (for the evaluation)."""
    norm = normal.norm(dim=1, keepdim=True)
    valid = torch.isfinite(target[:, :1]) & (norm > 1e-6)
    n = valid.sum().clamp_min(1)
    nn = norm.clamp_min(1e-6)
    u = normal / nn
    t = torch.nan_to_num(target)
    cos = (u * t).sum(1, keepdim=True)
    loss = weight * torch.where(valid, 1.0 - cos, torch.zeros_like(cos)).sum() / n
    g = torch.where(valid, -(t - u * cos) / nn, torch.zeros_like(u)) * (weight * upstream / n)
    angle = torch.where(valid, torch.rad2deg(torch.arccos(cos.clamp(-1, 1))), torch.zeros_like(cos)).sum() / n
    return loss, g, angle


def depth_loss_and_grad(depth, trans, target, weight, upstream=1.0):
    """weight * mean |ED - target| over the pixels with a finite target and 1 - T > 1e-3, ED = depth / (1 - trans) ->
    (loss, d_depth, d_trans), each gradient scaled by upstream."""
    alpha = 1.0 - trans
    valid = torch.isfinite(target) & (alpha > 1e-3)
    n = valid.sum().clamp_min(1)
    a = alpha.clamp_min(1e-3)
    ed = depth / a
    r = torch.where(valid, ed - torch.nan_to_num(target), torch.zeros_like(ed))
    loss = weight * r.abs().sum() / n
    g_ed = torch.where(valid, torch.sign(r), torch.zeros_like(r)) * (weight * upstream / n)
    return loss, g_ed / a, g_ed * ed / a


def depth_normal_angle(depth, trans, normal, proj):
    """Mean angle in degrees between N / |N| and the depth normal n_d over the pixels where n_d is defined and |N| > 1e-6."""
    nd, mask = geometry.depth_normal(depth, trans, proj)
    norm = normal.norm(dim=1, keepdim=True)
    valid = mask & (norm > 1e-6)
    cos = (nd * normal / norm.clamp_min(1e-6)).sum(1, keepdim=True).clamp(-1, 1)
    return float(torch.rad2deg(torch.arccos(cos))[valid].mean()) if bool(valid.any()) else float("nan")


def train(root, iters=300, views_per_step=8, log=print, refine_poses=False, antialiased=False, filter_3d=False, exact_grad=False,
          depth_weight=0.0, metrics=None, normal_weight=0.0, depth_normal_weight=0.0, mesh=None, mesh_resolution=256):
    """Returns (loss history, PSNR).  depth_weight > 0 adds the expected-depth term (the dataset must have depths/), normal_weight
    > 0 the normal term (the dataset must have normals/), depth_normal_weight > 0 the depth-normal consistency term (no targets).
    mesh (a PLY path, optional): at the end, the mesh fused from all training cameras in a volume of mesh_resolution lattice
    points along the longest axis of the Gaussian centres' box.
    metrics (a dict, optional) receives "ed_error": mean |ED - target| over the known pixels of 8 training views, when the dataset
    has depths, "normal_angle": their mean angle in degrees between N / |N| and the target, when it has normals, and
    "depth_normal_angle": the mean angle in degrees between N / |N| and n_d where both are defined, with depth_normal_weight > 0."""
    from litegs_b200 import fused
    if refine_poses and int(os.environ.get("WORLD_SIZE", "1")) > 1:
        raise ValueError("--refine-poses runs on one GPU: multi-GPU pose refinement is not supported")
    keep = fused.CONFIG["true_sigmoid_grad"]
    fused.CONFIG["true_sigmoid_grad"] = True               # our own loops train with the true sigmoid derivative (SURVEY Q15)
    try:
        return _train(root, iters, views_per_step, log, refine_poses, antialiased, filter_3d, exact_grad, depth_weight, metrics,
                      normal_weight, depth_normal_weight, mesh, mesh_resolution)
    finally:
        fused.CONFIG["true_sigmoid_grad"] = keep


class _Poses:
    """Learnable extrinsics f32[n_frames,7] (qw qx qy qz tx ty tz, initialised from the COLMAP poses) with their own Adam.  Each
    view's camera comes from create_viewproj_forward; render_views' camera gradients are mapped back through
    create_viewproj_backward.  The field of view stays fixed, as in the reference (trainer.py:161-162)."""
    Z_NEAR, Z_FAR = 0.01, 5000.0

    def __init__(self, frames, hw, dev, lr=1e-4):
        self.hw = hw
        H, W = hw
        ext, recp = [], None
        for cam, _, _ in frames:
            q, t, intr = colmap.camera_to_colmap({k: v.cpu().numpy() for k, v in cam.items()}, W, H)
            ext.append(np.concatenate([q, t]))
            recp = intr[0] / (W * 0.5)
        self.extr = torch.tensor(np.stack(ext), dtype=torch.float32, device=dev).requires_grad_(True)
        self.recp = torch.tensor([recp], dtype=torch.float32, device=dev)
        self.opt = torch.optim.Adam([self.extr], lr=lr)

    def cameras(self, idx):
        from litegs_b200 import fused
        v, p, _, planes = fused.create_viewproj_forward(self.extr.detach()[idx], self.recp, *self.hw, self.Z_NEAR, self.Z_FAR)
        return [dict(view=v[i:i + 1], proj=p[i:i + 1], frustumplane=planes[i:i + 1]) for i in range(len(idx))]

    def step(self, idx, camera_grads):
        from litegs_b200 import fused
        ix = torch.tensor(idx, dtype=torch.int64, device=self.extr.device)
        g, _ = fused.create_viewproj_backward(camera_grads[:, 0], camera_grads[:, 1], torch.zeros_like(camera_grads[:, 0]),
                                              self.extr.detach()[ix], self.recp, *self.hw, self.Z_NEAR, self.Z_FAR)
        self.extr.grad = torch.zeros_like(self.extr).index_add_(0, ix, g)
        self.opt.step()


def _train(root, iters, views_per_step, log, refine_poses=False, antialiased=False, filter_3d=False, exact_grad=False,
           depth_weight=0.0, metrics=None, normal_weight=0.0, depth_normal_weight=0.0, mesh=None, mesh_resolution=256):
    dev = torch.device("cuda", int(os.environ.get("LOCAL_RANK", 0)))
    torch.cuda.set_device(dev)
    frames, xyz, rgb = load_dataset(root, dev=dev)
    targets = load_depths(root, dev=dev)
    if depth_weight > 0 and targets is None:
        raise ValueError(f"--depth-weight needs expected-depth targets in {os.path.join(root, 'depths')}")
    use_depth = depth_weight > 0
    ntargets = load_depths(root, dev=dev, sub="normals")
    if normal_weight > 0 and ntargets is None:
        raise ValueError(f"--normal-weight needs unit-normal targets in {os.path.join(root, 'normals')}")
    use_normal = normal_weight > 0
    use_dn = depth_normal_weight > 0
    H, W = frames[0][2]
    poses = _Poses(frames, (H, W), dev) if refine_poses else None
    extr0 = poses.extr.detach().clone() if poses else None
    cgrads = torch.empty((views_per_step, 2, 4, 4), dtype=torch.float32, device=dev) if poses else None
    g = colmap.gaussians_from_points(xyz, rgb, sh_degree=3)
    P = {k: torch.from_numpy(g[k]).to(dev) for k in PARAM_ORDER}
    pp = PipelineParams(tile_size=(8, 16), sparse_grad=True, antialiased=antialiased, exact_grad=exact_grad,
                        render_depth=use_depth or use_dn, render_normal=use_normal or use_dn)
    acc = lgs_dist.GradAccumulator(P)
    extent = float(np.linalg.norm(xyz.max(0) - xyz.min(0)) * 0.5)
    opt, sched = optimizer.get_optimizer(P, spatial_lr_scale=extent)
    hist = []
    # Mip-Splatting's 3D smoothing filter: recomputed from ALL training cameras (every rank computes the same values, no
    # collective) into the same tensor, so the captured per-view graphs keep reading it
    filt = torch.empty_like(P["opacity"]) if filter_3d else None
    hw_all = torch.tensor([[H, W]] * len(frames), dtype=torch.int32, device=dev) if filter_3d else None
    t0 = time.perf_counter()
    for it in range(iters):
        idx = [(it * views_per_step + j) % len(frames) for j in range(views_per_step)]
        if filter_3d and it % 100 == 0:
            all_cams = poses.cameras(list(range(len(frames)))) if poses else [f[0] for f in frames]
            scene.filter_3d_device(P["xyz"], torch.cat([c["view"] for c in all_cams]), torch.cat([c["proj"] for c in all_cams]), hw_all,
                                   out=filt)
        # positions and shapes move, so the chunk AABBs used for culling are refreshed from the parameters now and then
        if it % 50 == 0:
            A = list(scene.cluster_aabb_torch(P["xyz"], P["scale"], P["rot"], filter_3d=filt))
        cams = poses.cameras(idx) if poses else [frames[j][0] for j in idx]

        def colour_loss(i, img):
            return ssim.l1_ssim_loss_and_grad(img.contiguous(), frames[idx[i]][1], 0.2, upstream=1.0 / views_per_step)

        def colour_and_depth_loss(i, img, depth, trans):
            loss, d_img = colour_loss(i, img)
            ld, d_depth, d_trans = depth_loss_and_grad(depth, trans, targets[idx[i]], depth_weight, upstream=1.0 / views_per_step)
            return loss + ld, d_img, d_depth, d_trans

        def with_normal_loss(i, img, depth, trans, normal):
            if use_depth:
                loss, d_img, d_depth, d_trans = colour_and_depth_loss(i, img, depth, trans)
            else:
                (loss, d_img), d_depth, d_trans = colour_loss(i, img), None, None
            d_normal = None
            if use_normal:
                ln, d_normal, _ = normal_loss_and_grad(normal, ntargets[idx[i]], normal_weight, upstream=1.0 / views_per_step)
                loss = loss + ln
            if use_dn:
                lc, gd, gt, gn = geometry.depth_normal_loss_and_grad(depth, trans, normal, cams[i]["proj"], depth_normal_weight,
                                                                     upstream=1.0 / views_per_step)
                add = lambda a, b: b if a is None else a + b
                loss, d_depth, d_trans, d_normal = loss + lc, add(d_depth, gd), add(d_trans, gt), add(d_normal, gn)
            return loss, d_img, d_depth, d_trans, d_normal

        fn = with_normal_loss if (use_normal or use_dn) else (colour_and_depth_loss if use_depth else colour_loss)
        losses = render.render_views(views_per_step, lambda i: cams[i], None, A[0], A[1], P["xyz"], P["scale"], P["rot"],
                                     P["sh_0"], P["sh_rest"], P["opacity"], 3, (H, W), pp, acc.grads(),
                                     loss_and_grad_fn=fn, camera_grads=cgrads, filter_3d=filt)
        opt.step(acc)
        if poses:
            poses.step(idx, cgrads)
        sched.step()
        hist.append(float(torch.stack(losses).mean()))
        if it % 50 == 0 or it == iters - 1:
            log(f"iter {it:5d}  loss {hist[-1]:.5f}")
    torch.cuda.synchronize(dev)
    dt = time.perf_counter() - t0
    pp_eval = PipelineParams(tile_size=(8, 16), sparse_grad=True, antialiased=antialiased, render_depth=targets is not None or use_dn,
                             enable_transmitance=targets is not None or use_dn, render_normal=ntargets is not None or use_dn)
    with torch.no_grad():
        mse, ed_err, n_err, dn_err = [], [], [], []
        for j, (cam, gt, _) in enumerate(frames[:8]):
            cam = poses.cameras([j])[0] if poses else cam
            img, trans, depth, normal, _ = render.render_view(A[0], A[1], cam["frustumplane"], cam["view"], cam["proj"], P["xyz"],
                                                              P["scale"], P["rot"], P["sh_0"], P["sh_rest"], P["opacity"], 3, (H, W),
                                                              pp_eval, filter_3d=filt)
            mse.append(float(((img - gt) ** 2).mean()))
            if targets is not None:
                ed_err.append(float(depth_loss_and_grad(depth, trans, targets[j], 1.0)[0]))
            if ntargets is not None:
                n_err.append(float(normal_loss_and_grad(normal, ntargets[j], 1.0)[2]))
            if use_dn:
                dn_err.append(depth_normal_angle(depth, trans, normal, cam["proj"]))
    psnr = -10.0 * np.log10(np.mean(mse))
    if ed_err:
        log(f"expected-depth error over 8 training views: {np.mean(ed_err):.4f}")
        if metrics is not None:
            metrics["ed_error"] = float(np.mean(ed_err))
    if n_err:
        log(f"mean angle between N / |N| and the target normals over 8 training views: {np.mean(n_err):.2f} degrees")
        if metrics is not None:
            metrics["normal_angle"] = float(np.mean(n_err))
    if dn_err:
        log(f"mean angle between N / |N| and the depth normal n_d over 8 training views: {np.mean(dn_err):.2f} degrees")
        if metrics is not None:
            metrics["depth_normal_angle"] = float(np.mean(dn_err))
    log(f"{iters} iterations x {views_per_step} views in {dt:.1f} s ({iters * views_per_step / dt:.0f} views/s incl. loss + optimizer); "
        f"{xyz.shape[0]} Gaussians, PSNR over 8 training views {psnr:.2f} dB")
    if poses:
        moved = (poses.extr.detach() - extr0).abs()
        log(f"poses refined: mean |change| of the quaternions {float(moved[:, :4].mean()):.2e}, of the translations {float(moved[:, 4:].mean()):.2e}")
    if mesh:
        all_cams = poses.cameras(list(range(len(frames)))) if poses else [f[0] for f in frames]
        vol = lgs_mesh.bounding_volume(P["xyz"], resolution=mesh_resolution)
        A = list(scene.cluster_aabb_torch(P["xyz"], P["scale"], P["rot"], filter_3d=filt))
        lgs_mesh.mesh_from_views(dict(P, cluster_origin=A[0], cluster_extend=A[1]), all_cams, (H, W),
                                 PipelineParams(tile_size=(8, 16), antialiased=antialiased), vol, filter_3d=filt)
        v, f, c = vol.extract()
        ply.save_mesh_ply(mesh, v, f, c)
        log(f"mesh fused from {len(all_cams)} training views in a {'x'.join(map(str, vol.dims))} volume: {len(v)} vertices, "
            f"{len(f)} faces -> {mesh}")
    return hist, psnr


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--make", default=None, help="write a synthetic COLMAP dataset to this directory first and train on it")
    ap.add_argument("--data", default=None)
    ap.add_argument("--iters", type=int, default=300)
    ap.add_argument("--refine-poses", action="store_true", help="also optimise the camera extrinsics (one GPU)")
    ap.add_argument("--antialiased", action="store_true", help="train (and evaluate) in the antialiased mode")
    ap.add_argument("--filter-3d", action="store_true",
                    help="Mip-Splatting's 3D smoothing filter, from all training cameras at iteration 0 and every 100 iterations")
    ap.add_argument("--exact-grad", action="store_true",
                    help="exact position and camera gradients: also through the ray-space Jacobian and the SH view direction")
    ap.add_argument("--depth-weight", type=float, default=0.0,
                    help="weight of the mean |expected depth - target| term (needs depths/<image stem>.npy, written by --make)")
    ap.add_argument("--normal-weight", type=float, default=0.0,
                    help="weight of the mean (1 - cos) term between N / |N| and the target normals (needs normals/<image stem>.npy, "
                         "written by --make)")
    ap.add_argument("--depth-normal-weight", type=float, default=0.0,
                    help="weight of the mean (1 - cos) term between N / |N| and the normal of the rendered expected depth (needs no "
                         "targets)")
    ap.add_argument("--mesh", default=None, metavar="PATH", help="after training, write the mesh fused from the training views (PLY)")
    ap.add_argument("--mesh-resolution", type=int, default=256, help="lattice points along the longest axis of the --mesh volume")
    ap.add_argument("--pose-noise", type=float, nargs=2, default=None, metavar=("DEG", "FRAC"),
                    help="with --make: perturb the written poses by DEG degrees and FRAC of the camera distance")
    a = ap.parse_args()
    root = a.data
    if a.make:
        root = make_dataset(a.make, pose_noise=a.pose_noise)
    if root is None:
        ap.error("give --data or --make")
    h, _ = train(root, a.iters, refine_poses=a.refine_poses, antialiased=a.antialiased, filter_3d=a.filter_3d,
                 exact_grad=a.exact_grad, depth_weight=a.depth_weight, normal_weight=a.normal_weight,
                 depth_normal_weight=a.depth_normal_weight, mesh=a.mesh, mesh_resolution=a.mesh_resolution)
    assert h[-1] < h[0]
