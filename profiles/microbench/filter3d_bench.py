"""Cost of Mip-Splatting's 3D smoothing filter.  At C2 (1M Gaussians, 1920x1080, SH degree 3, 8x16 tiles): the per-view forward
(the whole synchronising render_view_forward) and backward (raster + project backward) of the same views without and with a
filter computed from 24 lattice cameras, the two arms alternated in one run, timed with CUDA events after warm-up, and the
(tile, splat) pair counts.  Then lgs_filter_3d at 1M Gaussians for 24, 300 and 1000 cameras.  Prints the GPU's name and power
limit beside the numbers."""
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import torch

from litegs_b200 import pipeline, scene

KEYS = ("xyz", "scale", "rot", "sh_0", "sh_rest", "opacity")


def _cameras(n, hw, dev):
    cams = [scene.make_camera(i, n, hw[1], hw[0]) for i in range(n)]
    cat = lambda k: torch.cat([torch.from_numpy(c[k]) for c in cams]).to(dev)
    return cat("view"), cat("proj"), torch.tensor([list(hw)] * n, dtype=torch.int32, device=dev)


def main(n_views=8, reps=20):
    dev = torch.device("cuda:0")
    try:
        plim = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    except OSError:
        plim = "unknown"
    print(f"GPU: {torch.cuda.get_device_name(0)}, power limit {plim}")
    H, W, tile = 1080, 1920, (8, 16)
    p = scene.make_scene(1_000_000, sh_degree=3, seed=0, log_scale_range=(0.002, 0.02))
    P = {k: torch.from_numpy(p[k]).to(dev) for k in KEYS}
    F = scene.filter_3d_device(P["xyz"], *_cameras(24, (H, W), dev))
    boxes = {None: [torch.from_numpy(p[k]).to(dev) for k in ("cluster_origin", "cluster_extend")],
             "f": list(scene.cluster_aabb_torch(P["xyz"], P["scale"], P["rot"], filter_3d=F))}
    acc = {k: torch.zeros_like(P[k]) for k in KEYS}
    cams = [{k: torch.from_numpy(x).to(dev) for k, x in scene.make_camera(v, 64, W, H).items()} for v in range(n_views)]
    g = torch.Generator(device="cpu").manual_seed(0)
    d_imgs = [torch.randn((1, 3, H, W + (-W) % tile[1]), generator=g).to(dev) for _ in range(n_views)]
    arms = (None, "f")

    def forward(arm):
        A = boxes[arm]
        out = []
        for cam in cams:
            img, st, _ = pipeline.render_view_forward(P, A[0], A[1], cam["frustumplane"], cam["view"], cam["proj"], 3, (H, W), tile,
                                                      clamp_zero=True, filter_3d=F if arm else None)
            out.append((img, st))
        return out

    def backward(views):
        for (img, st), d in zip(views, d_imgs):
            pipeline.render_view_backward(P, st, d[..., :img.shape[-2], :img.shape[-1]].contiguous(), accumulate_into=acc, clamped_img=img)

    pairs = {arm: [st.n_pairs for _, st in forward(arm)] for arm in arms}
    for _ in range(3):
        for arm in arms:
            backward(forward(arm))
    torch.cuda.synchronize()
    tf, tb = {a: [] for a in arms}, {a: [] for a in arms}
    for r in range(reps):
        for arm in (arms if r % 2 == 0 else arms[::-1]):
            e0, e1, e2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
            e0.record()
            views = forward(arm)
            e1.record()
            backward(views)
            e2.record()
            torch.cuda.synchronize()
            tf[arm].append(e0.elapsed_time(e1) / n_views)
            tb[arm].append(e1.elapsed_time(e2) / n_views)
    med = lambda v: sorted(v)[len(v) // 2]
    for name, t in (("forward", tf), ("backward", tb)):
        print(f"C2 per-view {name}, median of {reps} x {n_views} views: off {med(t[None]):.3f} ms, filter {med(t['f']):.3f} ms "
              f"({100 * (med(t['f']) / med(t[None]) - 1):+.2f} %); spread off {min(t[None]):.3f}-{max(t[None]):.3f}, "
              f"filter {min(t['f']):.3f}-{max(t['f']):.3f} ms")
    mp = {k: sum(v) / len(v) for k, v in pairs.items()}
    print(f"C2 pairs per view (mean of {n_views}): off {mp[None]:.0f}, filter {mp['f']:.0f} ({100 * (mp['f'] / mp[None] - 1):+.2f} %)")

    out = torch.empty_like(F)
    for n_cam in (24, 300, 1000):
        cam_set = _cameras(n_cam, (H, W), dev)
        for _ in range(3):
            scene.filter_3d_device(P["xyz"], *cam_set, out=out)
        torch.cuda.synchronize()
        ts = []
        for _ in range(reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            scene.filter_3d_device(P["xyz"], *cam_set, out=out)
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1))
        n_pts = P["xyz"].shape[-2] * P["xyz"].shape[-1]
        print(f"lgs_filter_3d, {n_pts} Gaussians x {n_cam} cameras: median {med(ts):.3f} ms of {reps} "
              f"({n_pts * n_cam / med(ts) / 1e6:.1f} G Gaussian-camera pairs/s), spread {min(ts):.3f}-{max(ts):.3f} ms")


if __name__ == "__main__":
    main()
