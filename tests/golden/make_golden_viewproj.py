"""Generates tests/golden/viewproj.npz: the reference's own create_viewproj kernels (GR/compact.cu:17-316, in
oracle/_ref/litegs_fused_ref*.so, built by oracle/build_ref.py for sm_90a) run on an H100 over seeded inputs:

    python tests/golden/make_golden_viewproj.py OUTDIR        # then copy OUTDIR/viewproj.npz into tests/golden/

1920x1080 (integer aspect quotient 1, not 16/9), non-unit quaternions, V = 5 views.  grad_recp is stored from a V = 1 call
only: for V > 1 the reference's += on one word races across the views.  The inputs are stored with the outputs (a few KB).
tests/test_oracle_camera.py compares the CPU restatement against it, tests/test_gpu_camera.py our kernels.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

VIEWPROJ = dict(n_views=5, hw=(1080, 1920), z_near=0.01, z_far=5000.0, seed=21)


def viewproj_inputs():
    c = VIEWPROJ
    rng = np.random.default_rng(c["seed"])
    V = c["n_views"]
    q = rng.normal(size=(V, 4))
    q *= (rng.uniform(0.6, 1.5, size=(V, 1)) / np.linalg.norm(q, axis=1, keepdims=True))       # |q| in [0.6, 1.5)
    t = rng.normal(size=(V, 3)) * 2.0
    g = lambda: rng.normal(size=(V, 4, 4)).astype(np.float32)
    return dict(view_params=np.concatenate([q, t], axis=1).astype(np.float32), recp=np.array([1.0 / np.tan(np.radians(30.0))], np.float32),
                g_view=g(), g_proj=g(), g_viewproj=g())


def run_viewproj(mod, torch, dev):
    """create_viewproj forward (V = 5), backward (V = 5) and backward of the first view alone on backend `mod`."""
    c = VIEWPROJ
    H, W = c["hw"]
    x = viewproj_inputs()
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    view, proj, viewproj, planes = mod.create_viewproj_forward(T(x["view_params"]), T(x["recp"]), H, W, c["z_near"], c["z_far"])
    gp, _ = mod.create_viewproj_backward(T(x["g_view"]), T(x["g_proj"]), T(x["g_viewproj"]), T(x["view_params"]), T(x["recp"]), H, W,
                                         c["z_near"], c["z_far"])
    _, gr1 = mod.create_viewproj_backward(T(x["g_view"][:1]), T(x["g_proj"][:1]), T(x["g_viewproj"][:1]), T(x["view_params"][:1]),
                                          T(x["recp"]), H, W, c["z_near"], c["z_far"])
    n = lambda a: a.detach().cpu().numpy()
    return dict(x, view=n(view), proj=n(proj), viewproj=n(viewproj), frustumplane=n(planes), grad_view_params=n(gp), grad_recp_v1=n(gr1))


def main():
    import torch
    from oracle import build_ref
    outdir = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden")
    os.makedirs(outdir, exist_ok=True)
    ref = build_ref.load()
    if ref is None:
        sys.exit("oracle/_ref is not built: see oracle/build_ref.py")
    out = run_viewproj(ref, torch, torch.device("cuda:0"))
    torch.cuda.synchronize()
    path = os.path.join(outdir, "viewproj.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
