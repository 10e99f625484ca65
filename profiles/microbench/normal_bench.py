"""Cost of the normal mode at C2 (1M Gaussians, 1920x1080, SH degree 3, 8x16 tiles): the per-view forward (the whole
synchronising render_view_forward) and backward (raster + project backward, with a gradient for each rendered extra channel) of the
same views with normals off, depth only, normals only and both, the four arms alternated in one run, timed with CUDA events after
warm-up.  Prints the GPU's name and power limit beside the numbers."""
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import torch

from litegs_b200 import pipeline, scene

KEYS = ("xyz", "scale", "rot", "sh_0", "sh_rest", "opacity")
ARMS = {"off": (False, False), "depth": (True, False), "normal": (False, True), "both": (True, True)}


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
    A = [torch.from_numpy(p[k]).to(dev) for k in ("cluster_origin", "cluster_extend")]
    acc = {k: torch.zeros_like(P[k]) for k in KEYS}
    cams = [{k: torch.from_numpy(x).to(dev) for k, x in scene.make_camera(v, 64, W, H).items()} for v in range(n_views)]
    g = torch.Generator(device="cpu").manual_seed(0)
    d_imgs = [torch.randn((1, 3, H, W + (-W) % tile[1]), generator=g).to(dev) for _ in range(n_views)]
    d_depths = [torch.randn((1, 1, H, W), generator=g).to(dev) for _ in range(n_views)]
    d_normals = [torch.randn((1, 3, H, W), generator=g).to(dev) for _ in range(n_views)]

    def forward(arm):
        dep, nrm = ARMS[arm]
        out = []
        for cam in cams:
            img, st, _ = pipeline.render_view_forward(P, A[0], A[1], cam["frustumplane"], cam["view"], cam["proj"], 3, (H, W), tile,
                                                      clamp_zero=True, render_depth=dep, render_normal=nrm)
            out.append((img, st))
        return out

    def backward(views):
        for (img, st), d, dd, dn in zip(views, d_imgs, d_depths, d_normals):
            pipeline.render_view_backward(P, st, d[..., :img.shape[-2], :img.shape[-1]].contiguous(), accumulate_into=acc, clamped_img=img,
                                          d_depth=dd if st.depth is not None else None, d_normal=dn if st.normal is not None else None)

    names = list(ARMS)
    for _ in range(3):
        for arm in names:
            backward(forward(arm))
    torch.cuda.synchronize()
    tf, tb = {a: [] for a in names}, {a: [] for a in names}
    for r in range(reps):
        for arm in names[r % 4:] + names[:r % 4]:
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
        base = med(t["off"])
        print(f"C2 per-view {name}, median of {reps} x {n_views} views: " + ", ".join(
            f"{a} {med(t[a]):.3f} ms ({100 * (med(t[a]) / base - 1):+.2f} %, spread {min(t[a]):.3f}-{max(t[a]):.3f})" for a in names))


if __name__ == "__main__":
    main()
