"""Cost of mesh extraction (csrc/mesh.cu through litegs_b200.mesh) at the sizes of a real capture.

  * integration: 64 views at 1920x1080 (analytic expected depth of a unit sphere seen from a radius-3 Fibonacci lattice, alpha 1 on
    the sphere, colour on) into a 512^3 volume over [-1.3, 1.3]^3, in 4 launches of 16 views, timed with CUDA events; achieved
    bytes/s against the algorithmic bytes: 20 B (tsdf, weight, colour) read and 20 B written per lattice point per launch, plus
    the pixels gathered (T for every (point, view) pair that projects into the image, D and rgb for those with alpha > 0.5),
    counted here with torch;
  * extraction of the resulting mesh (count kernel, two int64 scans, the read-back of the totals, emit kernels), host clock
    around a synchronised call.
Medians after warm-up; the GPU's name and power limit are printed beside the numbers."""
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import time

import torch

from litegs_b200 import mesh, scene

HBM = 3.35e12          # H100 SXM data-sheet bandwidth, B/s


def sphere_batch(n_views, hw, rho=1.0, radius=3.0, dev="cuda"):
    """D, T, rgb f32[V,*,H,W] and views, projs f32[V,4,4] of a unit sphere along lgs_depth_normal's pixel rays."""
    H, W = hw
    D, T, C, Vs, Ps = [], [], [], [], []
    for i in range(n_views):
        cam = scene.make_camera(i, n_views, W, H, radius=radius)
        Vm = torch.from_numpy(cam["view"][0]).double().to(dev)
        Pm = torch.from_numpy(cam["proj"][0]).double().to(dev)
        fx, fy = Pm[0, 0] * W * 0.5, Pm[1, 1] * H * 0.5
        v, u = torch.meshgrid(torch.arange(H, device=dev, dtype=torch.float64) + 0.5, torch.arange(W, device=dev, dtype=torch.float64) + 0.5,
                              indexing="ij")
        r = torch.stack([(u - W / 2) / fx, (v - H / 2) / fy, torch.ones_like(u)], -1)
        Rinv = torch.linalg.inv(Vm[:3, :3])
        c = -Vm[3, :3] @ Rinv
        d = r @ Rinv
        a, b, cc = (d * d).sum(-1), 2 * d @ c, c @ c - rho * rho
        disc = b * b - 4 * a * cc
        hit = disc > 0
        z = torch.where(hit, (-b - torch.sqrt(disc.clamp_min(0))) / (2 * a), torch.zeros_like(a))
        alpha = hit.double()
        D.append((alpha * z)[None]); T.append((1 - alpha)[None])
        C.append(alpha[None] * torch.stack([0.5 + 0.4 * torch.sin(3 * u / W), 0.5 + 0.4 * torch.cos(2 * v / H), torch.full_like(u, 0.3)]))
        Vs.append(Vm); Ps.append(Pm)
    return tuple(torch.stack(x).float().contiguous() for x in (D, T, C, Vs, Ps))


def gathered_pairs(vol, views, projs, T, alpha_min=0.5):
    """(pairs that read T, pairs that also read D and rgb) over all lattice points and views, by the kernel's rules (fp32)."""
    nx, ny, nz = vol.dims
    dev = vol.device
    o, h = vol.origin, vol.voxel_size
    xs = torch.arange(nx, device=dev, dtype=torch.float32) * h + o[0]
    ys = torch.arange(ny, device=dev, dtype=torch.float32) * h + o[1]
    H, W = T.shape[-2:]
    n_t = n_d = 0
    for k in range(nz):
        zk = float(torch.tensor(k, dtype=torch.float32) * h + o[2])
        X, Y = xs[None, :].expand(ny, nx), ys[:, None].expand(ny, nx)
        for v in range(views.shape[0]):
            M, P = views[v], projs[v]
            x = X * M[0, 0] + Y * M[1, 0] + zk * M[2, 0] + M[3, 0]
            y = X * M[0, 1] + Y * M[1, 1] + zk * M[2, 1] + M[3, 1]
            z = X * M[0, 2] + Y * M[1, 2] + zk * M[2, 2] + M[3, 2]
            u = x / z * (P[0, 0] * W * 0.5) + W * 0.5
            w = y / z * (P[1, 1] * H * 0.5) + H * 0.5
            m = (z > 0.01) & (u >= 0) & (u < W) & (w >= 0) & (w < H)
            n_t += int(m.sum())
            a = 1 - T[v, 0][w.clamp(0, H - 1).long()[m], u.clamp(0, W - 1).long()[m]]
            n_d += int((a > alpha_min).sum())
    return n_t, n_d


def _med(v):
    return sorted(v)[len(v) // 2]


def main(reps=10):
    dev = torch.device("cuda:0")
    try:
        plim = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    except OSError:
        plim = "unknown"
    print(f"GPU: {torch.cuda.get_device_name(0)}, power limit {plim}")
    hw, n_views, batch, res = (1080, 1920), 64, 16, 512
    D, T, C, V, P = sphere_batch(n_views, hw)
    vol = mesh.bounding_volume(None, bounds=(-1.3, -1.3, -1.3, 1.3, 1.3, 1.3), resolution=res)
    N = vol.tsdf.numel()

    def integrate_all():
        for b in range(0, n_views, batch):
            vol.integrate(D[b:b + batch], T[b:b + batch], V[b:b + batch], P[b:b + batch], rgb=C[b:b + batch])

    def reset():
        vol.tsdf.fill_(1.0); vol.weight.zero_(); vol.color.zero_()

    times = []
    for r in range(reps + 2):
        reset()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        integrate_all()
        e1.record()
        torch.cuda.synchronize()
        if r >= 2:
            times.append(e0.elapsed_time(e1) * 1e-3)
    t_int = _med(times)
    n_t, n_d = gathered_pairs(vol, V, P, T)
    launches = n_views // batch
    vol_bytes = 40 * N * launches
    gather_bytes = 4 * n_t + 16 * n_d
    print(f"integration, {n_views} views {hw[1]}x{hw[0]} into {res}^3 with colour, {launches} launches of {batch}: "
          f"{t_int * 1e3:.2f} ms (median of {reps}, spread {min(times) * 1e3:.2f}-{max(times) * 1e3:.2f}); "
          f"{(t_int / n_views) * 1e3:.3f} ms per view")
    print(f"  algorithmic bytes: volume {vol_bytes / 1e9:.2f} GB (40 B per point per launch) + gathers {gather_bytes / 1e9:.2f} GB "
          f"({n_t / 1e9:.2f} G (point, view) pairs in the image, {n_d / 1e9:.2f} G with alpha > 0.5) = "
          f"{(vol_bytes + gather_bytes) / t_int / 1e12:.2f} TB/s, {100 * (vol_bytes + gather_bytes) / t_int / HBM:.0f} % of 3.35 TB/s; "
          f"volume traffic alone {vol_bytes / t_int / 1e12:.2f} TB/s ({100 * vol_bytes / t_int / HBM:.0f} %)")
    ext = []
    for r in range(reps // 2 + 2):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        v, f, c = vol.extract()
        torch.cuda.synchronize()
        if r >= 2:
            ext.append(time.perf_counter() - t0)
        del v, f, c
    v, f, c = vol.extract()
    print(f"extraction: {_med(ext) * 1e3:.2f} ms (median of {len(ext)}, spread {min(ext) * 1e3:.2f}-{max(ext) * 1e3:.2f}) for "
          f"{len(v)} vertices, {len(f)} faces from {N / 1e6:.1f} M lattice points")


if __name__ == "__main__":
    main()
