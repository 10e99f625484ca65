"""Timing of the SURVEY 8(f) "next" rows beside the unmodified reference kernels where they exist:

  * fused L1+SSIM loss forward+backward at 1920x1080x3 (what trainer.py:145 runs per iteration): ours through the
    reference-shaped autograd surface, ours through l1_ssim_loss_and_grad (no loss map), the reference's fused_ssim_cuda
    (oracle/_ref/fused_ssim_cuda_ref.so) through its own Python layer;
  * the optimizer step at 1M Gaussians: one lgs_adam_step_dense launch vs six adamUpdate launches (ours and the
    reference's litegs_fused.adamUpdate).

Prints one JSON object; CUDA events, 5 warm-up + 50 timed repetitions, inputs (25-236 MB) streamed from HBM each time.
usage: python profiles/microbench/next_rows_bench.py > next_rows.json"""
import json
import sys

import torch

sys.path.insert(0, ".")
from litegs_b200 import dist as lgs_dist, fused, optimizer, scene, ssim  # noqa: E402
from litegs_b200.dist import PARAM_ORDER  # noqa: E402


def timeit(fn, reps=50, warm=5):
    for _ in range(warm):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    dev = torch.device("cuda:0")
    out = {}
    peak = 6650.0
    try:
        peak = float(json.load(open("MEASURED_PEAKS.json")).get("hbm_gbs", peak))
    except Exception:
        pass
    # ---- L1 + SSIM ----------------------------------------------------------------------------------------------------
    g = torch.Generator().manual_seed(0)
    H, W = 1080, 1920
    img = torch.rand((1, 3, H, W), generator=g).to(dev)
    gt = torch.rand((1, 3, H, W), generator=g).to(dev)
    n = img.numel()

    def ours_autograd():
        x = img.detach().requires_grad_(True)
        ssim.fused_l1_ssim_loss(x, gt).backward()

    def ours_fused():
        ssim.l1_ssim_loss_and_grad(img, gt, 0.2)

    C1, C2 = 0.01 ** 2, 0.03 ** 2

    def ours_kernels_only():
        _, d0, d1, d2, _ = ssim._forward(1, 0.2, C1, C2, img, gt, True, want_map=False, want_sums=True)
        ssim._backward(1, 0.2, img, gt, None, 1.0 / n, d0, d1, d2)

    res = {"shape": [1, 3, H, W], "ours_autograd_ms": timeit(ours_autograd), "ours_loss_and_grad_ms": timeit(ours_fused),
           "ours_two_kernels_ms": timeit(ours_kernels_only)}
    # algorithmic bytes: fwd reads 2 images, writes 3 partial maps; bwd reads 3 maps + 2 images, writes the gradient
    alg = n * 4 * (2 + 3 + 3 + 2 + 1)
    res["alg_bytes"] = alg
    res["ours_two_kernels_gbs"] = alg / (res["ours_two_kernels_ms"] * 1e-3) / 1e9
    res["hbm_frac"] = res["ours_two_kernels_gbs"] / peak
    from oracle import build_ref
    ref = build_ref.load_ssim()
    if ref is not None:
        class RefMap(torch.autograd.Function):           # the reference's FusedL1SSIMLossMap (fused_ssim/__init__.py:53-80) on its kernels
            @staticmethod
            def forward(ctx, x, y):
                m, a, b, c = ref.fusedl1ssim_loss(0.2, C1, C2, x, y, True)
                ctx.save_for_backward(x.detach(), y, a, b, c)
                return m

            @staticmethod
            def backward(ctx, gr):
                x, y, a, b, c = ctx.saved_tensors
                return ref.fusedl1ssim_loss_backward(0.2, C1, C2, x, y, gr, a, b, c), None

        def ref_autograd():
            x = img.detach().requires_grad_(True)
            RefMap.apply(x, gt).mean().backward()

        res["reference_autograd_ms"] = timeit(ref_autograd)
    out["l1_ssim_1080p_fwd_bwd"] = res
    # ---- optimizer step -------------------------------------------------------------------------------------------------
    sc = scene.make_scene(1_000_000, sh_degree=3, seed=0)
    P = {k: torch.from_numpy(sc[k]).to(dev) for k in PARAM_ORDER}
    C, S = P["xyz"].shape[-2:]
    acc = lgs_dist.GradAccumulator(P)
    acc.buf.normal_()
    opt = optimizer.FusedAdam(P, {k: 1e-4 for k in PARAM_ORDER})
    ids = torch.arange(C, dtype=torch.int64, device=dev)
    cnt = torch.tensor([C], dtype=torch.int32, device=dev)

    def fused_step():
        acc.mark(ids, cnt)
        opt.step(acc, clear_grad=False)

    def six_calls(mod):
        def f():
            for k in PARAM_ORDER:
                R = P[k].numel() // (C * S)
                m, v = opt.state_for(k)
                mod.adamUpdate(P[k].view(R, C, S), acc.buf[acc.rows[k]], m.view(R, C, S), v.view(R, C, S), ids, cnt, 1e-4, 0.9, 0.999, 1e-15)
        return f

    elems = acc.buf.numel()
    ares = {"gaussians": C * S, "elements": elems, "fused_one_launch_ms": timeit(fused_step), "ours_six_adamUpdate_ms": timeit(six_calls(fused))}
    ares["alg_bytes"] = elems * 28
    ares["fused_gbs"] = ares["alg_bytes"] / (ares["fused_one_launch_ms"] * 1e-3) / 1e9
    ares["hbm_frac"] = ares["fused_gbs"] / peak
    refgr = build_ref.load()
    if refgr is not None:
        ares["reference_six_adamUpdate_ms"] = timeit(six_calls(refgr))
    out["adam_step_1M"] = ares
    out["hbm_peak_gbs"] = peak
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
