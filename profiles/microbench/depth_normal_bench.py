"""Cost of the depth-normal consistency term at C2 (1M Gaussians, 1920x1080, SH degree 3, 8x16 tiles, depth and normals on).

On D, T and N of one rendered C2 view:
  * the fused kernel (csrc/geometry.cu) alone, loss + three gradients, without and with the n_d map: 100 launches captured in a
    CUDA graph, the graph replayed and timed with CUDA events; achieved bytes/s against the kernel's algorithmic bytes (each
    input read once, each output written once: 40 B per pixel, 52 B with the map);
  * the public call geometry.depth_normal_loss_and_grad (kernel, block-sum reduction, allocations, host overhead) and the same math
    as a torch composition with autograd (forward + backward), the two alternated in one loop;
then the per-view render_views step (the GPU-driven path, 8 views per batch, L1+SSIM colour loss) with depth and normals off,
rendered without a depth or normal loss, rendered with precomputed zero gradients for D, T and N (the raster backward's extra
channels without the term), and rendered with the term, the four arms alternated.  Medians after warm-up; the GPU's name and
power limit are printed beside the numbers."""
import ctypes
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import torch

from litegs_b200 import _lib, geometry, pipeline, render, scene, ssim
from litegs_b200.arguments import PipelineParams
from litegs_b200.dist import GradAccumulator
from litegs_b200.fused import _ptr, _stream

KEYS = ("xyz", "scale", "rot", "sh_0", "sh_rest", "opacity")


def torch_composition(depth, trans, normal, proj, weight, alpha_min=0.5):
    """The loss of DESIGN.md section 1, "Depth-normal consistency", written with torch operations (autograd gives its gradient)."""
    H, W = depth.shape[-2:]
    P = proj.reshape(4, 4)
    fx, fy = P[0, 0] * W * 0.5, P[1, 1] * H * 0.5
    dev = depth.device
    rx = ((torch.arange(W, device=dev, dtype=torch.float32) + 0.5) - 0.5 * W) / fx
    ry = ((torch.arange(H, device=dev, dtype=torch.float32) + 0.5) - 0.5 * H) / fy
    alpha = 1 - trans[0, 0]
    valid = alpha > alpha_min
    E = torch.where(valid, depth[0, 0] / torch.where(valid, alpha, torch.ones_like(alpha)), torch.zeros_like(alpha))
    eL, eR, eT, eB = E[1:-1, :-2], E[1:-1, 2:], E[:-2, 1:-1], E[2:, 1:-1]
    m = valid[1:-1, 1:-1] & valid[1:-1, :-2] & valid[1:-1, 2:] & valid[:-2, 1:-1] & valid[2:, 1:-1]
    dx, dy = eR - eL, eB - eT
    a = torch.stack([dx * rx[None, :-2] + eR * (2 / fx), dx * ry[1:-1, None], dx])
    b = torch.stack([dy * rx[None, 1:-1], dy * ry[:-2, None] + eB * (2 / fy), dy])
    c = torch.linalg.cross(b, a, dim=0)
    cn = c.norm(dim=0)
    q = normal[0, :, 1:-1, 1:-1]
    qn = q.norm(dim=0)
    lm = m & (cn > 0) & (qn > 1e-6)
    one = torch.ones_like(cn)
    cs = ((c / torch.where(lm, cn, one)) * (q / torch.where(lm, qn, one))).sum(0)
    return weight * torch.where(lm, 1 - cs, torch.zeros_like(cs)).sum() / (H * W)


def _med(v):
    return sorted(v)[len(v) // 2]


def main(reps=30, n_views=8):
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
    cams = [{k: torch.from_numpy(x).to(dev) for k, x in scene.make_camera(v, 64, W, H).items()} for v in range(n_views)]
    cam = cams[0]
    _, st, _ = pipeline.render_view_forward(P, A[0], A[1], cam["frustumplane"], cam["view"], cam["proj"], 3, (H, W), tile, clamp_zero=True,
                                            render_depth=True, render_normal=True)
    D, T, N = st.depth[..., :H, :W], st.T[..., :H, :W], st.normal[..., :H, :W]       # the strided views render_views hands out
    proj = cam["proj"]
    weight = 0.1
    cover = float(((1 - T) > 0.5).float().mean())
    nd, mask = geometry.depth_normal(D, T, proj)
    print(f"C2 view: {100 * cover:.1f} % of the pixels have alpha > 0.5, n_d defined on {100 * float(mask.float().mean()):.1f} %")

    # the kernel alone, 100 launches per graph
    nb = ctypes.c_int(0)
    _lib.call("lgs_depth_normal_num_block_sums", H, W, ctypes.byref(nb))
    sums = torch.empty(nb.value, device=dev)
    gD, gT, gN, ndm = torch.empty((1, 1, H, W), device=dev), torch.empty((1, 1, H, W), device=dev), torch.empty((1, 3, H, W), device=dev), \
        torch.empty((1, 3, H, W), device=dev)
    Pc = proj.contiguous()

    def launch(with_map):
        _lib.call("lgs_depth_normal", _ptr(D), D.stride(-2), _ptr(T), T.stride(-2), _ptr(N), N.stride(-2), N.stride(1), _ptr(Pc), H, W, 0.5,
                  weight / (H * W), _ptr(ndm) if with_map else None, _ptr(gD), _ptr(gT), _ptr(gN), _ptr(sums), _stream(dev))

    graphs = {}
    side = torch.cuda.Stream(dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
        for with_map in (False, True):
            launch(with_map)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=side):
                for _ in range(100):
                    launch(with_map)
            graphs[with_map] = g
    torch.cuda.current_stream(dev).wait_stream(side)
    tk = {False: [], True: []}
    for r in range(reps + 3):
        for with_map in ((False, True) if r % 2 == 0 else (True, False)):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            graphs[with_map].replay()
            e1.record()
            torch.cuda.synchronize()
            if r >= 3:
                tk[with_map].append(e0.elapsed_time(e1) / 100 * 1e3)          # us per launch
    for with_map in (False, True):
        byts = H * W * (40 + (12 if with_map else 0))
        t = _med(tk[with_map])
        print(f"fused kernel, loss + gradients{' + n_d map' if with_map else ''}: {t:.1f} us per launch (median of {reps} graphs of 100, "
              f"spread {min(tk[with_map]):.1f}-{max(tk[with_map]):.1f}); {byts / 1e6:.1f} MB algorithmic -> {byts / t / 1e6:.2f} TB/s")

    # the public call against the torch composition (forward + backward), alternated
    Dl, Tl, Nl = (x.detach().clone().requires_grad_(True) for x in (D, T, N))

    def fused_call():
        return geometry.depth_normal_loss_and_grad(D, T, N, proj, weight)

    def torch_call():
        for x in (Dl, Tl, Nl):
            x.grad = None
        loss = torch_composition(Dl, Tl, Nl, proj, weight)
        loss.backward()
        return loss

    lf, dDf, dTf, dNf = fused_call()
    lt = torch_call().detach()
    rel = lambda a, b: float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))
    print(f"fused vs torch composition: loss {float(lf):.7e} vs {float(lt):.7e}, gradients (max |diff| / max): D {rel(dDf, Dl.grad):.1e}, "
          f"T {rel(dTf, Tl.grad):.1e}, N {rel(dNf, Nl.grad):.1e}")
    tc = {"fused call": [], "torch composition": []}
    calls = {"fused call": fused_call, "torch composition": torch_call}
    for r in range(reps + 3):
        for name in (list(calls) if r % 2 == 0 else list(calls)[::-1]):
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(10):
                calls[name]()
            e1.record()
            torch.cuda.synchronize()
            if r >= 3:
                tc[name].append(e0.elapsed_time(e1) / 10 * 1e3)
    base = _med(tc["torch composition"])
    for name, t in tc.items():
        print(f"{name} (loss + gradients): {_med(t):.1f} us per call (median of {reps} x 10, spread {min(t):.1f}-{max(t):.1f}; "
              f"{base / _med(t):.1f}x the torch composition's speed)")

    # render_views step time per view: off, depth + normals rendered without the term, with the term
    gts = [torch.rand((1, 3, H, W), device=dev) for _ in range(n_views)]
    acc = GradAccumulator(P)
    arms = {"off": PipelineParams(tile_size=tile), "rendered": PipelineParams(tile_size=tile, render_depth=True, render_normal=True),
            "gradients": PipelineParams(tile_size=tile, render_depth=True, render_normal=True),
            "term": PipelineParams(tile_size=tile, render_depth=True, render_normal=True)}
    zD, zN = torch.zeros((1, 1, H, W), device=dev), torch.zeros((1, 3, H, W), device=dev)

    def colour(i, img):
        return ssim.l1_ssim_loss_and_grad(img.contiguous(), gts[i], 0.2, upstream=1.0 / n_views)

    def rendered(i, img, depth, trans, normal):
        return (*colour(i, img), None, None, None)

    def zero_gradients(i, img, depth, trans, normal):
        return (*colour(i, img), zD, zD, zN)

    def with_term(i, img, depth, trans, normal):
        loss, d_img = colour(i, img)
        ln, dD, dT, dN = geometry.depth_normal_loss_and_grad(depth, trans, normal, cams[i]["proj"], weight, upstream=1.0 / n_views)
        return loss + ln, d_img, dD, dT, dN

    fns = {"off": colour, "rendered": rendered, "gradients": zero_gradients, "term": with_term}

    def step(arm):
        acc.zero_()
        render.render_views(n_views, lambda i: cams[i], None, A[0], A[1], P["xyz"], P["scale"], P["rot"], P["sh_0"], P["sh_rest"],
                            P["opacity"], 3, (H, W), arms[arm], acc.grads(), loss_and_grad_fn=fns[arm])

    for _ in range(3):
        for arm in arms:
            step(arm)
    torch.cuda.synchronize()
    render.check_views()
    ts = {a: [] for a in arms}
    names = list(arms)
    for r in range(reps):
        for arm in names[r % len(names):] + names[:r % len(names)]:
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            step(arm)
            e1.record()
            torch.cuda.synchronize()
            ts[arm].append(e0.elapsed_time(e1) / n_views)
    render.check_views()
    base = _med(ts["off"])
    print(f"render_views per view (GPU-driven path, {n_views} views per batch, L1+SSIM), median of {reps}: " + ", ".join(
        f"{a} {_med(ts[a]):.3f} ms ({100 * (_med(ts[a]) / base - 1):+.2f} %, spread {min(ts[a]):.3f}-{max(ts[a]):.3f})" for a in names))


if __name__ == "__main__":
    main()
