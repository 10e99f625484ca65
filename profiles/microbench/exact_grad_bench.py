"""Cost of the exact gradient mode at C2 (1M Gaussians, 1920x1080, SH degree 3, 8x16 tiles): the per-view backward (raster +
project) with the mode off and on, each without and with the camera gradient, and project_backward on its own (the same record
gradients fed to lgs_project_backward, dense-accumulate mode, as render_views runs it).  The arms are alternated in one run and
timed with CUDA events after warm-up; medians of 20 x 8 views.  Prints the GPU's name and power limit beside the numbers."""
import ctypes
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import torch

from litegs_b200 import _lib, pipeline, scene
from litegs_b200.fused import CONFIG, _ptr, _stream

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
    C, S = P["xyz"].shape[-2:]
    R = P["sh_rest"].shape[0]
    views = []
    g = torch.Generator(device="cpu").manual_seed(0)
    n_grad = []
    for v in range(n_views):
        cam = {k: torch.from_numpy(x).to(dev) for k, x in scene.make_camera(v, 64, W, H).items()}
        img, st, _ = pipeline.render_view_forward(P, A[0], A[1], cam["frustumplane"], cam["view"], cam["proj"], 3, (H, W), tile, clamp_zero=True)
        d = torch.randn(img.shape, generator=g).to(dev)
        _, pg = pipeline.render_view_backward(P, st, d, accumulate_into=acc, clamped_img=img)
        pg = pg.clone()
        n_grad.append(int((pg[0, :st.n_chunks_visible * S] != 0).any(dim=-1).sum()))
        views.append((st, d, img, pg))
    cg = torch.empty((2, 4, 4), device=dev)

    def backward(exact, cam_on):
        for st, d, img, _ in views:
            pipeline.render_view_backward(P, st, d, accumulate_into=acc, clamped_img=img, camera_grad=cg if cam_on else None,
                                          exact_grad=exact)

    def project(exact):
        st_ = _stream(dev)
        for st, _, _, pg in views:
            _lib.call("lgs_project_backward", 3, _ptr(st.chunk_ids), ctypes.c_void_p(st.counters.data_ptr()), _ptr(st.view), _ptr(st.proj),
                      _ptr(P["xyz"]), _ptr(P["scale"]), _ptr(P["rot"]), _ptr(P["opacity"]), C, S, st.n_chunks_visible, R, H, W,
                      int(CONFIG["true_sigmoid_grad"]), _ptr(pg), None, 2, *(_ptr(acc[k]) for k in KEYS), None, None, None, None, 0,
                      _ptr(P["sh_0"]), _ptr(P["sh_rest"]), int(exact), 0, None, st_)

    arms = {("backward", e, c): (lambda e=e, c=c: backward(e, c)) for e in (False, True) for c in (False, True)}
    arms.update({("project", e, False): (lambda e=e: project(e)) for e in (False, True)})
    keys = list(arms)
    for _ in range(3):
        for k in keys:
            arms[k]()
    torch.cuda.synchronize()
    times = {k: [] for k in keys}
    for r in range(reps):
        for k in (keys if r % 2 == 0 else keys[::-1]):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            arms[k]()
            e1.record()
            torch.cuda.synchronize()
            times[k].append(e0.elapsed_time(e1) / n_views)
    med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
    print(f"C2: {sum(n_grad) / n_views:.0f} Gaussians with a non-zero record gradient per view (mean of {n_views}); "
          f"the mode reads 15 * 3 * 4 = 180 B more of sh_rest for each")
    for what, cam_on in (("per-view backward (raster + project), no camera gradient", False),
                         ("per-view backward (raster + project), with the camera gradient", True),
                         ("project_backward alone (dense accumulate, no camera gradient)", False)):
        kind = "project" if what.startswith("project") else "backward"
        off, on = med[(kind, False, cam_on)], med[(kind, True, cam_on)]
        print(f"{what}, median of {reps} x {n_views} views: off {off:.4f} ms, exact {on:.4f} ms ({100 * (on / off - 1):+.2f} %); "
              f"spread off {min(times[(kind, False, cam_on)]):.4f}-{max(times[(kind, False, cam_on)]):.4f}, "
              f"exact {min(times[(kind, True, cam_on)]):.4f}-{max(times[(kind, True, cam_on)]):.4f} ms")


if __name__ == "__main__":
    main()
