"""Generates the golden fixtures that pin the CPU oracle and our kernels to the REFERENCE ITSELF.

Runs the unmodified reference kernels (oracle/_ref/litegs_fused_ref*.so, built by oracle/build_ref.py with the
reference's own flags, for sm_90a) on an H100 over a small seeded scene and stores every output of the hot path that
the tests compare as float32/int32 arrays:

    python tests/golden/make_golden.py OUTDIR        # then copy OUTDIR/*.npz into tests/golden/

Inputs are NOT stored: tests regenerate them from the seed with litegs_b200.scene (numpy PCG64 streams are
stable), plus the seeded upstream gradients below.  Arrays of more than SAMPLE_ABOVE elements are stored as the values at
seeded flat positions (``<name>`` + ``<name>__index``), which keeps every fixture under 1 MB.  tests/test_golden.py
compares the oracle (CPU) against these fixtures, tests/test_gpu_vs_reference.py our kernels (GPU).
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

CASES = {
    # name: (n_gaussians, (H, W), (tile_h, tile_w), sh_degree, seed, view)
    "c_small_16x16": (2000, (96, 128), (16, 16), 3, 0, 0),
    "c_small_8x16": (2000, (96, 128), (8, 16), 2, 1, 3),
}
PARAM_KEYS = ("xyz", "scale", "rot", "sh_0", "sh_rest", "opacity")
SAMPLE_ABOVE = 65536
NOT_STORED = ("left_up", "right_down", "final_T")          # outputs no test compares


def matched(ref, got, k):
    """(stored reference values, ours at the same positions) for output k."""
    got = np.asarray(got[k])
    if f"{k}__index" in ref:
        return ref[k], got.reshape(-1)[ref[f"{k}__index"]]
    return ref[k], got


def case_inputs(name):
    from litegs_b200 import scene
    n, hw, tile, deg, seed, view = CASES[name]
    p = scene.make_scene(n, sh_degree=3, seed=seed, log_scale_range=(0.02, 0.08))
    cam = scene.make_camera(view, 8, hw[1], hw[0])
    rng = np.random.default_rng(seed + 1000)
    C, S = p["xyz"].shape[-2:]
    N = C * S
    up = dict(
        d_img=rng.normal(size=(1, 3, hw[0], hw[1])).astype(np.float32),
        g_inv=rng.normal(size=(1, 2, 2, N)).astype(np.float32),
        g_cov=rng.normal(size=(1, 2, 2, N)).astype(np.float32),
        g_T=rng.normal(size=(3, 3, N)).astype(np.float32),
        g_ndc=rng.normal(size=(1, 4, N)).astype(np.float32),
        g_view=rng.normal(size=(1, 4, N)).astype(np.float32),
        g_act=[rng.normal(size=s).astype(np.float32) for s in ((4, C, S), (3, C, S), (4, C, S), (1, 3, C, S), (1, C, S))],
    )
    up["g_inv"][:, 1, 0] = up["g_inv"][:, 0, 1]
    up["g_cov"][:, 1, 0] = up["g_cov"][:, 0, 1]
    return p, cam, hw, tile, deg, up


def run_backend(mod, name, torch, dev):
    """Runs the whole op chain on backend `mod` (an object with the litegs_fused surface); returns dict of numpy."""
    p, cam, hw, tile, deg, up = case_inputs(name)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    out = {}
    P = {k: T(p[k]) for k in PARAM_KEYS}
    view, proj, fp = T(cam["view"]), T(cam["proj"]), T(cam["frustumplane"])
    vis, num, ids = mod.frustum_culling_aabb(T(p["cluster_origin"]), T(p["cluster_extend"]), fp, None, None)
    nvis = int(num.item())
    ids_sorted = torch.sort(ids[:nvis])[0].contiguous()
    out["cull_vis"] = vis.detach().cpu().numpy(); out["cull_ids"] = ids_sorted.detach().cpu().numpy()
    act = mod.cull_compact_activate(deg, ids_sorted, num, view, P["xyz"], P["scale"], P["rot"], P["sh_0"], P["sh_rest"], P["opacity"])
    for k, a in zip(("act_pos", "act_scale", "act_rot", "act_color", "act_opacity"), act):
        out[k] = a.detach().cpu().numpy()
    xyz, scale, rot, color, opacity = [a.reshape(*a.shape[:-2], -1).contiguous() for a in act]
    vp, ndc = mod.mvp_transform_forward(xyz, view, proj, None)
    Tm = mod.createTransformMatrix_forward(rot, scale, None)
    J = mod.jacobianRayspace(vp, proj, hw[0], hw[1], None)
    cov = mod.createCov2dDirectly_forward(J, view, Tm, None)
    val, vec, inv = mod.eigh_and_inv_2x2matrix_forward(cov, None)
    out.update(view_pos=vp.detach().cpu().numpy(), ndc=ndc.detach().cpu().numpy(), T=Tm.detach().cpu().numpy(), J=J.detach().cpu().numpy(), cov2d=cov.detach().cpu().numpy(),
               eig_val=val.detach().cpu().numpy(), inv_cov2d=inv.detach().cpu().numpy())
    N = xyz.shape[1]
    sl = lambda a: T(a[..., :N])
    out["bw_inv"] = mod.inv_2x2matrix_backward(inv, sl(up["g_inv"]), None).detach().cpu().numpy()
    out["bw_cov"] = mod.createCov2dDirectly_backward(sl(up["g_cov"]), J, view, Tm, None).detach().cpu().numpy()
    gq, gs = mod.createTransformMatrix_backward(sl(up["g_T"]), rot, scale, None)
    out["bw_T_q"] = gq.detach().cpu().numpy(); out["bw_T_s"] = gs.detach().cpu().numpy()
    out["bw_mvp"] = mod.mvp_transform_backward(sl(up["g_ndc"]), sl(up["g_view"]), view, proj, vp, None).detach().cpu().numpy()
    # binning (wrapper.py:718-763 glue)
    vz = vp[:, 2].contiguous()
    lu, rd, alloc = mod.get_allocate_size(ndc, vz, inv, opacity, hw[0], hw[1], tile[0], tile[1], None)
    out["alloc"] = alloc.detach().cpu().numpy(); out["left_up"] = lu.detach().cpu().numpy(); out["right_down"] = rd.detach().cpu().numpy()
    _, order = vz.sort(dim=-1, descending=False, stable=True)
    prefix = torch.gather(alloc, 1, order).cumsum(1, dtype=torch.int32)
    keys, vals = mod.create_table(ndc, inv, opacity, prefix, order, None, None, hw[0], hw[1], tile[0], tile[1])
    gx, gy = -(-hw[1] // tile[1]), -(-hw[0] // tile[0])
    ranges = mod.tileRange(keys, gx * gy)
    out["table_keys"] = keys.detach().cpu().numpy(); out["table_vals"] = vals.detach().cpu().numpy(); out["tile_range"] = ranges.detach().cpu().numpy()
    # raster
    r = mod.rasterize_forward(vals, ranges, ndc, inv, color, opacity, None, hw[0], hw[1], tile[0], tile[1], False, False, False)
    img, Tr, _, last, packed = r[0], r[1], r[2], r[3], r[4]
    out["img"] = img.detach().cpu().numpy(); out["final_T"] = Tr.detach().cpu().numpy(); out["last"] = last.detach().cpu().numpy()
    Hp, Wp = img.shape[-2:]
    d_img = torch.zeros((1, 3, Hp, Wp), device=dev)
    d_img[..., : hw[0], : hw[1]] = T(up["d_img"])
    gmax = d_img.abs().max()
    b = mod.rasterize_backward(vals, ranges, packed, None, Tr, last, d_img / gmax, None, None, gmax.reshape(1), hw[0], hw[1], tile[0], tile[1],
                               False)
    for k, a in zip(("d_ndc", "d_cov2d_inv", "d_color", "d_opacity"), b[:4]):
        out[k] = a.detach().cpu().numpy()
    C, S = p["xyz"].shape[-2:]
    A = ids_sorted.shape[0]
    ga = [T(g[..., :A, :]) for g in up["g_act"]]
    ab = mod.activate_backward(deg, ids_sorted, num, view, P["xyz"], P["scale"], P["rot"], P["sh_0"], P["sh_rest"], P["opacity"], *ga)
    for k, a in zip(("ab_pos", "ab_scale", "ab_rot", "ab_sh0", "ab_shr", "ab_opacity"), ab):
        out[k] = a.detach().cpu().numpy()
    return out


def main():
    import torch
    from oracle import build_ref
    outdir = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden")
    os.makedirs(outdir, exist_ok=True)
    ref = build_ref.load()
    if ref is None:
        sys.exit("oracle/_ref is not built: see oracle/build_ref.py")
    dev = torch.device("cuda:0")
    for name in CASES:
        out = run_backend(ref, name, torch, dev)
        torch.cuda.synchronize()
        store = {}
        rng = np.random.default_rng(11)
        for k, v in out.items():
            if k in NOT_STORED:
                continue
            if v.size > SAMPLE_ABOVE:
                idx = np.sort(rng.choice(v.size, SAMPLE_ABOVE // 2, replace=False))
                store[k], store[f"{k}__index"] = v.reshape(-1)[idx], idx
            else:
                store[k] = v
        path = os.path.join(outdir, f"{name}.npz")
        np.savez_compressed(path, **store)
        print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
