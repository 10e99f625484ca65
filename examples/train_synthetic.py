"""A data-parallel training loop on the litegs_b200 stack, end to end on synthetic data (BASELINE.json config 5 in spirit:
no COLMAP files, the targets are renders of a hidden "true" scene).

    python examples/train_synthetic.py --iters 200                                   # one GPU
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 examples/train_synthetic.py

Per iteration and rank: render_views over this rank's views (fused pipeline, gradients accumulated densely and chunk marks
set by the backward kernel) with the fused L1+SSIM loss -> one NCCL all-reduce of the gradient buffer -> one fused Adam
launch (reference semantics: optimizer.py:9-44, trainer.py:119-160 without densification).  Every rank applies the same
reduced gradient, so the replicas stay identical without broadcasting parameters.
"""
import argparse
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from litegs_b200 import dist as lgs_dist, fused, optimizer, render, scene, ssim  # noqa: E402
from litegs_b200.arguments import PipelineParams  # noqa: E402
from litegs_b200.dist import PARAM_ORDER  # noqa: E402


def train(n_gaussians=50_000, hw=(270, 480), n_views=16, iters=100, seed=0, device=None, log=print, perturb=0.3, antialiased=False,
          exact_grad=False):
    """Returns the list of per-iteration mean losses (rank-local views)."""
    keep = fused.CONFIG["true_sigmoid_grad"]
    fused.CONFIG["true_sigmoid_grad"] = True               # our own loops train with the true sigmoid derivative (SURVEY Q15)
    try:
        return _train(n_gaussians, hw, n_views, iters, seed, device, log, perturb, antialiased, exact_grad)
    finally:
        fused.CONFIG["true_sigmoid_grad"] = keep


def _train(n_gaussians, hw, n_views, iters, seed, device, log, perturb, antialiased=False, exact_grad=False):
    import torch.distributed as dist
    world = dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1
    rank = dist.get_rank() if world > 1 else 0
    dev = device or torch.device("cuda", int(os.environ.get("LOCAL_RANK", 0)))
    torch.cuda.set_device(dev)
    H, W = hw
    pp = PipelineParams(tile_size=(8, 16), sparse_grad=True, antialiased=antialiased,     # targets and model in the same mode
                        exact_grad=exact_grad)
    truth = scene.make_scene(n_gaussians, sh_degree=3, seed=seed)
    T = {k: torch.from_numpy(truth[k]).to(dev) for k in PARAM_ORDER}
    A = [torch.from_numpy(truth[k]).to(dev) for k in ("cluster_origin", "cluster_extend")]
    cams = [{k: torch.from_numpy(v).to(dev) for k, v in scene.make_camera(j, n_views, W, H).items()} for j in range(n_views)]
    mine = lgs_dist.shard_views(n_views, rank, world)      # shards may differ by one view: the loss is the mean over ALL n_views
    with torch.no_grad():       # targets: renders of the true scene
        gts = {j: render.render_view(A[0], A[1], cams[j]["frustumplane"], cams[j]["view"], cams[j]["proj"], T["xyz"], T["scale"], T["rot"],
                                     T["sh_0"], T["sh_rest"], T["opacity"], 3, (H, W), pp)[0].contiguous() for j in mine}
    # the model: same positions/shapes (so the chunk AABBs stay valid), appearance perturbed; identical on every rank
    g = torch.Generator(device="cpu").manual_seed(seed + 1)
    P = {k: T[k].clone() for k in PARAM_ORDER}
    for k in ("sh_0", "sh_rest", "opacity"):
        P[k] += perturb * torch.randn(P[k].shape, generator=g).to(dev) * (1.0 if k != "sh_rest" else 0.3)
    P = {k: v.requires_grad_(True) for k, v in P.items()}
    acc = lgs_dist.GradAccumulator(P)
    opt, sched = optimizer.get_optimizer({k: P[k].data for k in PARAM_ORDER}, spatial_lr_scale=1.0)
    history = []
    t0 = time.perf_counter()
    for it in range(iters):
        losses = render.render_views(len(mine), lambda i: cams[mine[i]], None,
                                     A[0], A[1], P["xyz"], P["scale"], P["rot"], P["sh_0"], P["sh_rest"], P["opacity"], 3, (H, W), pp,
                                     acc.grads(),
                                     loss_and_grad_fn=lambda i, img: ssim.l1_ssim_loss_and_grad(img.contiguous(), gts[mine[i]], 0.2,
                                                                                              upstream=1.0 / n_views))
        acc.all_reduce()
        opt.step(acc)
        sched.step()
        history.append(torch.stack(losses).mean())          # stays on the device: no host synchronisation inside the loop
        if rank == 0 and (it % 50 == 0 or it == iters - 1):
            log(f"iter {it:4d}  loss {float(history[-1]):.5f}")
    torch.cuda.synchronize(dev)
    # GPU-driven sizing: each render_views call read the flags of the earlier batches that had landed; this reads the rest, so
    # together they say that no view of the run outgrew its workspace
    render.check_views()
    history = [float(h) for h in history]
    if rank == 0:
        dt = time.perf_counter() - t0
        log(f"{iters} iterations x {len(mine)} views x {world} ranks in {dt:.2f} s = {iters * len(mine) * world / dt:.1f} views/s (loss + optimizer included)")
    return history


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gaussians", type=int, default=200_000)
    ap.add_argument("--width", type=int, default=960)
    ap.add_argument("--height", type=int, default=540)
    ap.add_argument("--views", type=int, default=16)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--antialiased", action="store_true", help="render the targets and train in the antialiased mode")
    ap.add_argument("--exact-grad", action="store_true",
                    help="exact position gradients: also through the ray-space Jacobian and the SH view direction")
    args = ap.parse_args()
    import torch.distributed as dist
    if int(os.environ.get("WORLD_SIZE", "1")) > 1:
        dist.init_process_group("nccl")
    hist = train(args.gaussians, (args.height, args.width), args.views, args.iters, antialiased=args.antialiased,
                 exact_grad=args.exact_grad)
    if dist.is_initialized():
        dist.destroy_process_group()
    assert hist[-1] < hist[0], "the loss did not decrease"


if __name__ == "__main__":
    main()
