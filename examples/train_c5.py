"""BASELINE.json configs[4] ("C5"): `example_train.py` on the synthetic scene exported as a COLMAP directory, 7k iterations.

    python examples/train_c5.py --make /tmp/c5                                   # hidden scene -> COLMAP model + PNGs (needs a GPU)
    python examples/train_c5.py --data /tmp/c5 --trainer reference --iters 7000  # the reference's UNMODIFIED trainer on our kernels (1 GPU)
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 \
        examples/train_c5.py --data /tmp/c5 --trainer ours --iters 7000          # this repository's data-parallel loop (N GPUs)

--trainer reference imports the reference package (the LiteGS checkout, or the byte copy staged under oracle/_ref/py by
oracle/build_ref.py) and calls ``litegs.training.start`` exactly as ``example_train.py:26`` does, with ``litegs_fused`` /
``fused_ssim`` resolving to this repository and ``plyfile`` / ``torchmetrics`` / ``matplotlib`` / ``simple_knn`` to the stand-ins of
``litegs_b200/shims``.  The reference is single-GPU (SURVEY fact 3), so the multi-GPU half of C5 is --trainer ours: views of a
global batch of 8 sharded over the ranks, fused L1+SSIM loss, one NCCL all-reduce of the dense gradient buffer, one fused Adam
step per iteration (reference optimiser semantics, no densification: that policy is out of scope, SURVEY 2.1).

Both print one JSON line (iterations, seconds, Gaussians, PSNR over 8 training views)."""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "examples"))
import train_colmap  # noqa: E402
from litegs_b200 import colmap, dist as lgs_dist, fused, optimizer, ply as lgs_ply, render, scene, ssim  # noqa: E402
from litegs_b200.arguments import PipelineParams  # noqa: E402
from litegs_b200.dist import PARAM_ORDER  # noqa: E402


def psnr_of(P, frames, hw, dev, n=8):
    A = list(scene.cluster_aabb_torch(P["xyz"], P["scale"], P["rot"]))
    pp = PipelineParams(tile_size=(8, 16))
    mse = []
    with torch.no_grad():
        for cam, gt, _ in frames[:n]:
            img = render.render_view(A[0], A[1], cam["frustumplane"], cam["view"], cam["proj"], P["xyz"], P["scale"], P["rot"], P["sh_0"],
                                     P["sh_rest"], P["opacity"], 3, hw, pp)[0]
            mse.append(float(((img - gt) ** 2).mean()))
    return float(-10.0 * np.log10(np.mean(mse)))


def run_reference(data, iters, out_dir, target_primitives):
    from oracle import build_ref
    from litegs_b200 import shims
    path = build_ref.reference_python_path()
    if path is None:
        sys.exit("reference Python package not available (no LiteGS checkout found and none staged under oracle/_ref/py: see oracle/build_ref.py)")
    shims.install()
    sys.path.insert(1, path)
    import litegs
    import litegs.config
    dev = torch.device("cuda:0")
    lp, op, pp, dp = litegs.config.get_default_arg()
    lp.source_path, lp.model_path, lp.sh_degree, lp.resolution = data, out_dir, 3, 1
    op.iterations = iters
    op.position_lr_max_steps = iters
    dp.target_primitives = target_primitives
    torch.manual_seed(0)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    litegs.training.start(lp, op, pp, dp, [], [], [], None)              # example_train.py:26
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    g = lgs_ply.params_from_ply(os.path.join(out_dir, "point_cloud", "finish", "point_cloud.ply"), sh_degree=3)
    P = {k: torch.from_numpy(g[k]).to(dev) for k in PARAM_ORDER}
    frames, _, _ = train_colmap.load_dataset(data, dev=dev)
    H, W = frames[0][2]
    n_frames = len(frames)
    return {"trainer": "reference litegs.training.start (unmodified) on litegs_b200 kernels", "n_gpus": 1, "iterations": int(iters / n_frames) * n_frames,
            "views_per_iteration": 1, "seconds_incl_data_loading": dt, "gaussians": int(g["xyz"].shape[-2] * g["xyz"].shape[-1]),
            "resolution": [H, W], "psnr_train_8_views": psnr_of(P, frames, (H, W), dev)}


def run_ours(data, iters, global_batch):
    import torch.distributed as dist
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    dev = torch.device("cuda", int(os.environ.get("LOCAL_RANK", 0)))
    torch.cuda.set_device(dev)
    if world > 1:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        dist.init_process_group("nccl", device_id=dev)
    fused.CONFIG["true_sigmoid_grad"] = True          # our own loop trains with the true sigmoid derivative (the reference's cluster
    #                                                   path omits the (1 - sigma) factor, SURVEY Q15; kept only for parity runs)
    frames, xyz, rgb = train_colmap.load_dataset(data, dev=dev)
    H, W = frames[0][2]
    g = colmap.gaussians_from_points(xyz, rgb, sh_degree=3)
    P = {k: torch.from_numpy(g[k]).to(dev) for k in PARAM_ORDER}
    pp = PipelineParams(tile_size=(8, 16), sparse_grad=True)
    acc = lgs_dist.GradAccumulator(P)
    extent = float(np.linalg.norm(xyz.max(0) - xyz.min(0)) * 0.5)
    opt, sched = optimizer.get_optimizer(P, spatial_lr_scale=extent, position_lr_max_steps=iters)
    per_rank = max(1, global_batch // world)
    n_batch = per_rank * world
    A = list(scene.cluster_aabb_torch(P["xyz"], P["scale"], P["rot"]))
    if world > 1:
        dist.barrier()
    torch.cuda.synchronize(dev)
    t0 = time.perf_counter()
    redo = 0
    for it in range(iters):
        idx = [(it * n_batch + rank * per_rank + j) % len(frames) for j in range(per_rank)]
        if it % 100 == 0:       # positions and shapes move: refresh the chunk AABBs used for culling
            A = list(scene.cluster_aabb_torch(P["xyz"], P["scale"], P["rot"]))
        while True:
            try:
                render.render_views(per_rank, lambda i: frames[idx[i]][0], None, A[0], A[1], P["xyz"], P["scale"], P["rot"], P["sh_0"],
                                    P["sh_rest"], P["opacity"], 3, (H, W), pp, acc.grads(),
                                    loss_and_grad_fn=lambda i, img: ssim.l1_ssim_loss_and_grad(img.contiguous(), frames[idx[i]][1], 0.2,
                                                                                             upstream=1.0 / n_batch))
                break
            except Exception as e:      # pipeline.CapacityExceeded: the previous step outgrew its workspace -> measured again now
                if type(e).__name__ != "CapacityExceeded":
                    raise
                redo += 1
                acc.zero_()
        acc.all_reduce()
        opt.step(acc)
        sched.step()
    torch.cuda.synchronize(dev)
    if world > 1:
        dist.barrier()
    dt = time.perf_counter() - t0
    out = None
    if rank == 0:
        out = {"trainer": "litegs_b200 data-parallel loop (render_views + fused L1+SSIM + NCCL all-reduce + fused Adam)", "n_gpus": world,
               "iterations": iters, "views_per_iteration": n_batch, "seconds": dt, "views_per_s": iters * n_batch / dt,
               "gaussians": int(xyz.shape[0]), "resolution": [H, W], "workspace_regrowths": redo,
               "psnr_train_8_views": psnr_of(P, frames, (H, W), dev)}
    if world > 1:
        dist.destroy_process_group()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--make", default=None)
    ap.add_argument("--data", default=None)
    ap.add_argument("--trainer", default="ours", choices=["ours", "reference"])
    ap.add_argument("--iters", type=int, default=7000)
    ap.add_argument("--global-batch", type=int, default=8)
    ap.add_argument("--gaussians", type=int, default=1_000_000, help="--make: Gaussians of the hidden scene (the C2 scene)")
    ap.add_argument("--points", type=int, default=150_000, help="--make: SfM points handed to the trainers")
    ap.add_argument("--views", type=int, default=64)
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--height", type=int, default=1080)
    ap.add_argument("--target-primitives", type=int, default=1_000_000)
    ap.add_argument("--out", default="/tmp/c5_out")
    a = ap.parse_args()
    if a.make:
        # the C2 synthetic scene (1M Gaussians, seed 0, BASELINE.md log-scale range) as the hidden truth
        train_colmap.make_dataset(a.make, n_gaussians=a.gaussians, n_views=a.views, hw=(a.height, a.width), n_points=a.points,
                                  log_scale_range=(0.002, 0.02) if a.gaussians >= 500_000 else (0.01, 0.04))
        print(f"dataset written to {a.make}")
        if a.data is None:
            return
    if a.data is None:
        ap.error("give --data (and/or --make)")
    res = run_reference(a.data, a.iters, a.out, a.target_primitives) if a.trainer == "reference" else run_ours(a.data, a.iters, a.global_batch)
    if res is not None:
        print("C5_RESULT " + json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
