"""One forward+backward view of the bench workload between cudaProfilerStart/Stop, for `ncu --profile-from-start off`:

    ncu --set full --clock-control none --import-source on --profile-from-start off -o prof_all python profiles/one_view.py [c2|c4]

Synchronising path, no CUDA graphs, one stream: every kernel of the view appears once, in order."""
import os
import sys

os.environ["LGS_GRAPHS"] = "0"
os.environ["LGS_SYNC_FREE"] = "0"
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import math  # noqa: E402

import torch  # noqa: E402

from litegs_b200 import pipeline, scene  # noqa: E402
from litegs_b200.dist import GradAccumulator, PARAM_ORDER  # noqa: E402

cfg = sys.argv[1] if len(sys.argv) > 1 else "c2"
n, W, H, rng = (1_000_000, 1920, 1080, (0.002, 0.02)) if cfg == "c2" else (5_000_000, 3840, 2160, (0.002 * math.exp(-0.5), 0.02 * math.exp(-0.5)))
dev = torch.device("cuda:0")
p = scene.make_scene(n, sh_degree=3, seed=0, log_scale_range=rng)
P = {k: torch.from_numpy(p[k]).to(dev) for k in PARAM_ORDER}
A = [torch.from_numpy(p[k]).to(dev) for k in ("cluster_origin", "cluster_extend")]
cam = {k: torch.from_numpy(v).to(dev) for k, v in scene.make_camera(0, 64, W, H).items()}
acc = GradAccumulator(P)
g = torch.randn((1, 3, H, W), device=dev)


def one():
    img, st, _ = pipeline.render_view_forward(P, A[0], A[1], cam["frustumplane"], cam["view"], cam["proj"], 3, (H, W), (8, 16), clamp_zero=True)
    d = torch.nn.functional.pad(g, (0, img.shape[-1] - W, 0, img.shape[-2] - H)) if img.shape[-2:] != g.shape[-2:] else g
    pipeline.render_view_backward(P, st, d, accumulate_into=acc.grads(), clamped_img=img)


for _ in range(2):
    one()
torch.cuda.synchronize()
torch.cuda.profiler.start()
one()
torch.cuda.synchronize()
torch.cuda.profiler.stop()
