"""Cost of the camera gradient in the per-view backward at C2 (1M Gaussians, 1920x1080, 8x16 tiles): the raster backward +
project backward of the same views with and without d_view / d_proj, the two arms alternated in one run, timed with CUDA events
after warm-up.  Prints the GPU's name and power limit beside the numbers."""
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import torch

from litegs_b200 import pipeline, scene

KEYS = ("xyz", "scale", "rot", "sh_0", "sh_rest", "opacity")


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
    views = []
    g = torch.Generator(device="cpu").manual_seed(0)
    for v in range(n_views):
        cam = {k: torch.from_numpy(x).to(dev) for k, x in scene.make_camera(v, 64, W, H).items()}
        img, st, _ = pipeline.render_view_forward(P, A[0], A[1], cam["frustumplane"], cam["view"], cam["proj"], 3, (H, W), tile, clamp_zero=True)
        views.append((st, torch.randn(img.shape, generator=g).to(dev), img))
    cg = torch.empty((2, 4, 4), device=dev)

    def run(cam_on):
        for st, d, img in views:
            pipeline.render_view_backward(P, st, d, accumulate_into=acc, clamped_img=img, camera_grad=cg if cam_on else None)

    for _ in range(3):
        run(False); run(True)
    torch.cuda.synchronize()
    times = {False: [], True: []}
    for r in range(reps):
        for cam_on in ((False, True) if r % 2 == 0 else (True, False)):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            run(cam_on)
            e1.record()
            torch.cuda.synchronize()
            times[cam_on].append(e0.elapsed_time(e1) / n_views)
    med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
    print(f"C2 per-view backward (raster + project), median of {reps} x {n_views} views: "
          f"without camera gradient {med[False]:.3f} ms, with {med[True]:.3f} ms, overhead {100 * (med[True] / med[False] - 1):+.2f} %")
    print(f"spread without: {min(times[False]):.3f}-{max(times[False]):.3f} ms, with: {min(times[True]):.3f}-{max(times[True]):.3f} ms")


if __name__ == "__main__":
    main()
