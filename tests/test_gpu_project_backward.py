"""project_backward_kernel against the fp64 per-Gaussian reference (tests/project_grad_oracle.py) on constructed edge cases.

Every family in HELD of tests/project_grad_oracle.constructed_cases() runs through lgs_project_backward alone on a hand-made record
gradient (the raw-moment slots, a depth slot and a normal row, with all-zero, depth-only and normal-only rows among them), with
every mode flag on and off against every other flag and all on, at SH degrees 0 and 3, under both opacity-logit conventions.
Every component of every Gaussian, and the camera gradient, must meet

    |kernel - ref| <= 1e-4 |ref| + 1e-6 (|J|^T |g|) + 2^-20 chain

with |J|^T |g| the magnitude of the component through the record map and chain the absolute terms of the kernel's own backward
stages (project_grad_oracle.chain_magnitude; scale, rotation, and position in exact mode).  The second term bounds fp32 noise where
the record map is well conditioned; the third where the backward's terms cancel (rotation gradients of splats symmetric about an
axis, the long-axis scale of screen-sized needles).  The families in CONDITIONED (screen-sized needles, rho down to 1e-3, the
rotated camera's needles) add 2^-22 (kappa_c + kappa_aa) (|J|^T |g|): the kernel evaluates the conic and the antialiasing factor in
fp32, and entries of M^T M rounded to a few ulps move the determinants by a few ulps of kappa_c = (|c00 c11| + c01^2) / |det| and
kappa_aa = (a00 a11 + a01^2) / det(M^T M).  Gaussians whose branch decisions are within rounding of flipping (project_grad_oracle.
fragile) are masked, taken out of the camera gradient, and counted.  Then the output forms, capacity-sized launches and
camera_grad_sum_kernel.
"""
import zlib

import numpy as np
import pytest
import torch

from litegs_b200 import _lib, pipeline
from tests import project_grad_oracle as pg

pytestmark = pytest.mark.gpu

S = 32
R = 15                                        # sh_rest rows: more than degree 0..2 use
FLAGS = ("cam", "aa", "f3d", "exact", "depth", "normal")
# all off, each alone, all on, each off from all on: every pair of flags takes all four values
MODES = ([{f: False for f in FLAGS}] + [{f: f == g for f in FLAGS} for g in FLAGS] + [{f: True for f in FLAGS}] +
         [{f: f != g for f in FLAGS} for g in FLAGS])
CASES = pg.constructed_cases()
# The families held to the bar on the device: all but the needles (see DESIGN.md section 2, "Projection gradient coverage").
HELD = tuple(f for f in CASES if f != "needles_sizes")
# Families whose conic or antialiasing factor is ill-conditioned (kappa up to 1e6): their bar carries the conditioning term.
CONDITIONED = ("det1", "antialias", "rotated_camera")
CHAIN = 2.0 ** -20                 # 16 ulps of the backward's own absolute terms (project_grad_oracle.chain_magnitude)


def _pad(x, n):
    """Pad the last axis to n with copies of its first entry."""
    k = n - x.shape[-1]
    return x if k == 0 else np.concatenate([x, np.repeat(x[..., :1], k, -1)], -1)


def _record_grad(N, rng, depth_only=(), normal_only=(), zero=()):
    m = rng.normal(size=(N, 12))
    m[:, 9] = 0.0
    m[:, 11] = 0.0
    gn = np.concatenate([rng.normal(size=(N, 3)), np.zeros((N, 1))], 1)
    for i in depth_only:
        m[i, :] = 0.0
        m[i, 10] = rng.normal()
        gn[i] = 0.0
    for i in normal_only:
        m[i, :] = 0.0
        gn[i, :3] = rng.normal(size=3)
    for i in zero:
        m[i] = 0.0
        gn[i] = 0.0
    return m.astype(np.float32), gn.astype(np.float32)


class Scene:
    """One family on the device: C chunks of S Gaussians in a permuted chunk order (chunk_ids non-contiguous)."""

    def __init__(self, cuda, case, seed=0, chunk=S):
        self.S = S = chunk
        p = case["params"]
        N0 = p["xyz"].shape[1]
        self.N0 = N0
        self.C = -(-N0 // S)
        self.N = self.C * S
        self.p = {k: _pad(np.asarray(v), self.N) for k, v in p.items()}
        self.view, self.proj = case["cam"]
        self.hw = case["hw"]
        rng = np.random.default_rng(seed)
        self.perm = rng.permutation(self.C)
        self.cuda = cuda
        P = self.p
        t = lambda a, *shape: torch.from_numpy(np.ascontiguousarray(a, np.float32).reshape(*shape)).to(cuda)
        C = self.C
        self.dev = dict(xyz=t(P["xyz"], 3, C, S), scale=t(P["scale"], 3, C, S), rot=t(P["rot"], 4, C, S),
                        sh_0=t(P["sh"][:1], 1, 3, C, S), sh_rest=t(P["sh"][1:1 + R], R, 3, C, S), opacity=t(P["opacity"], 1, C, S),
                        filt=t(P["filt"], 1, C, S), view=t(self.view, 4, 4), proj=t(self.proj, 4, 4))

    def launch(self, deg, mode, m, gn, *, ts=1, form=0, chunk_ids=None, nvis=None, A=None, out=None, touched=None,
               partials=None, sc=None):
        """lgs_project_backward.  m [A*S,12] and gn [A*S,4] in compacted (dst) order.  -> (outs, d_cam or None, partials)."""
        d, cuda, S = self.dev, self.cuda, self.S
        ids = self.perm if chunk_ids is None else chunk_ids
        A = len(ids) if A is None else A
        nvis = len(ids) if nvis is None else nvis
        ids_t = torch.zeros(A, dtype=torch.int64, device=cuda)
        ids_t[:len(ids)] = torch.as_tensor(np.asarray(ids), dtype=torch.int64)
        cnt = torch.tensor([nvis, 0, 0, 0], dtype=torch.int32, device=cuda)
        pgr = torch.zeros((A * S, 12), device=cuda)
        pgr[: m.shape[0]] = torch.from_numpy(m).to(cuda)
        gnt = torch.zeros((A * S, 4), device=cuda)
        gnt[: gn.shape[0]] = torch.from_numpy(gn).to(cuda)
        if out is None:
            rows = self.C if form == 2 else A
            out = [torch.full(s, float("nan"), device=cuda) for s in ((3, rows, S), (3, rows, S), (4, rows, S), (1, 3, rows, S),
                                                                         (R, 3, rows, S), (1, rows, S))]
        cam = torch.full((2, 4, 4), float("nan"), device=cuda) if mode["cam"] else None
        if mode["cam"] and partials is None:
            partials = torch.full((A, 32), float("nan"), device=cuda)
        p = pipeline._ptr
        _lib.call("lgs_project_backward", deg, p(ids_t), p(cnt), p(d["view"]), p(d["proj"]), p(d["xyz"]), p(d["scale"]), p(d["rot"]),
                  p(d["opacity"]), self.C, S, A, R, *self.hw, ts, p(pgr), p(sc), form, *(p(o) for o in out), p(touched),
                  p(partials) if mode["cam"] else None, p(cam), p(d["filt"]) if mode["f3d"] else None, int(mode["aa"]), p(d["sh_0"]),
                  p(d["sh_rest"]), int(mode["exact"]), int(mode["depth"]), p(gnt) if mode["normal"] else None,
                  pipeline._stream(cuda))
        torch.cuda.synchronize()
        return [o.cpu().numpy().astype(np.float64) for o in out], None if cam is None else cam.cpu().numpy().astype(np.float64), partials

    def src_order(self, x):
        """Per-Gaussian array [..., N] in source order -> compacted (dst) order of the default chunk permutation."""
        return x.reshape(*x.shape[:-1], self.C, self.S)[..., self.perm, :].reshape(*x.shape[:-1], -1)

    def reference(self, deg, mode, m_src, gn_src, ts=1):
        K = (deg + 1) ** 2
        P = dict(self.p, sh=self.p["sh"][:K])
        return pg.backward(P, self.view, self.proj, self.hw, deg, m_src, gn=gn_src if mode["normal"] else None,
                           filt=self.p["filt"] if mode["f3d"] else None, aa=mode["aa"], exact=mode["exact"], depth=mode["depth"],
                           true_sigmoid=bool(ts))


def _kappas(ref, aa):
    it = ref["it"]
    c00, c01, c11 = it["c00"], it["c01"], it["c11"]
    det = c00 * c11 - c01 * c01
    kc = (np.abs(c00 * c11) + c01 * c01) / np.abs(det)
    ka = np.zeros_like(kc)
    if aa:
        a00, a11 = c00 - 0.3, c11 - 0.3
        do = a00 * a11 - c01 * c01
        ka = np.where(do > 0, (np.abs(a00 * a11) + c01 * c01) / np.where(do > 0, do, 1.0), 0.0)
    return kc, ka


def _compare(kern, ref, bar, mask):
    """Largest err / bar over the unmasked Gaussians (last axis) and the failing indices; all arrays the same shape."""
    err = np.abs(kern - ref)
    r = np.where(mask, err / np.maximum(bar, 1e-30), 0.0)
    return (float(r.max()) if r.size else 0.0), np.argwhere((err > bar) & mask)


def _check_against_reference(sc, deg, mode, m_src, gn_src, ts, kern_out, d_cam, conditioned=False, masked_have_no_gradient=False):
    """Compare one launch with the reference -> (failures, largest err/bar, fragile Gaussians among the family's own)."""
    ref = sc.reference(deg, mode, m_src, gn_src, ts)
    K = (deg + 1) ** 2
    kc, ka = _kappas(ref, mode["aa"])
    cond = 2.0 ** -22 * (kc + ka) if conditioned else np.zeros_like(kc)
    chain = pg.chain_magnitude(ref, sc.view, sc.hw, aa=mode["aa"], filt=sc.p["filt"] if mode["f3d"] else None, normal=mode["normal"],
                               exact=mode["exact"])
    fr = pg.fragile(ref, sc.view, exact=mode["exact"], aa=mode["aa"])
    mask = ~fr
    n_fragile = int(fr[:sc.N0].sum())                     # the padding repeats the family's first Gaussian
    d = lambda x: sc.src_order(x)
    outs = dict(xyz=kern_out[0], scale=kern_out[1], rot=kern_out[2], opacity=kern_out[5][0])
    fails, worst = [], 0.0
    md = d(mask)

    def bar(k):
        b = 1e-4 * np.abs(ref["grads"][k]) + (1e-6 + cond) * ref["mag"][k]
        return d(b + CHAIN * chain[k] if k in chain else b)
    for k in ("xyz", "scale", "rot", "opacity"):
        kv = outs[k].reshape(*outs[k].shape[:-2], -1)
        w, bad = _compare(kv, d(ref["grads"][k]), bar(k), md)
        worst = max(worst, w)
        if len(bad):
            fails.append((k, bad[:4].tolist(), w))
    shk = np.concatenate([kern_out[3], kern_out[4][:K - 1]]).reshape(K, 3, -1)
    w, bad = _compare(shk, d(ref["grads"]["sh"]), bar("sh"), md)
    worst = max(worst, w)
    if len(bad):
        fails.append(("sh", bad[:4].tolist(), w))
    if d_cam is not None and (masked_have_no_gradient or not fr.any()):
        # with masked Gaussians the caller checks the camera on a launch that gives them no record gradient
        keep = mask[:, None, None, None]
        got = d_cam
        cref = (ref["cam_each"] * keep).sum(0)
        cbar = 1e-4 * np.abs(cref) + ((1e-6 + cond)[:, None, None, None] * ref["mag_cam_each"] * keep).sum(0)
        w, bad = _compare(got.reshape(-1), cref.reshape(-1), cbar.reshape(-1), np.ones(32, bool))
        worst = max(worst, w)
        if len(bad):
            fails.append(("cam", bad[:4].tolist(), w))
    return fails, worst, n_fragile, fr


@pytest.mark.parametrize("family", HELD)
def test_family_matches_fp64_reference(cuda, family):
    """Every mode pair at SH degrees 0 and 3 and both opacity conventions: each component of each Gaussian within the bar."""
    sc = Scene(cuda, CASES[family])
    conditioned = family in CONDITIONED
    rng = np.random.default_rng(zlib.crc32(family.encode()))
    N = sc.N
    m_src, gn_src = _record_grad(N, rng, depth_only=(1,), normal_only=(2,), zero=(3,))
    m_dst, gn_dst = sc.src_order(m_src.T).T.copy(), sc.src_order(gn_src.T).T.copy()
    fails, worst, nfrag = [], 0.0, 0
    for deg in (0, 3):
        for mi, mode in enumerate(MODES):
            for ts in (0, 1):
                kern, d_cam, _ = sc.launch(deg, mode, m_dst, gn_dst, ts=ts)
                f, w, nf, fr = _check_against_reference(sc, deg, mode, m_src, gn_src, ts, kern, d_cam, conditioned)
                if d_cam is not None and fr.any():
                    # the camera gradient without the masked Gaussians: their record gradient zeroed
                    m2, g2 = m_src.copy(), gn_src.copy()
                    m2[fr], g2[fr] = 0.0, 0.0
                    kern2, d_cam2, _ = sc.launch(deg, mode, sc.src_order(m2.T).T.copy(), sc.src_order(g2.T).T.copy(), ts=ts)
                    f2, w2, _, _ = _check_against_reference(sc, deg, mode, m2, g2, ts, kern2, d_cam2, conditioned, True)
                    f += [x for x in f2 if x[0] == "cam"]
                    w = max(w, w2)
                worst, nfrag = max(worst, w), max(nfrag, nf)
                fails += [(deg, mi, ts) + tuple(x) for x in f]
    print(f"\n[project_backward] {family}: largest err/bar {worst:.3g}, fragile Gaussians masked {nfrag}")
    assert nfrag <= 2, nfrag
    assert not fails, fails[:12]


def test_sh_degrees_1_and_2_and_rows_above_the_degree(cuda):
    """Degrees 1 and 2, every mode on: the active rows match the reference; form 1 leaves the rows above the degree zero."""
    sc = Scene(cuda, CASES["quaternions"])
    rng = np.random.default_rng(5)
    m_src, gn_src = _record_grad(sc.N, rng)
    m_dst, gn_dst = sc.src_order(m_src.T).T.copy(), sc.src_order(gn_src.T).T.copy()
    mode = {f: True for f in FLAGS}
    for deg in (1, 2):
        K = (deg + 1) ** 2
        kern, d_cam, _ = sc.launch(deg, mode, m_dst, gn_dst, form=1)
        fails, _, _, _ = _check_against_reference(sc, deg, mode, m_src, gn_src, 1, kern, d_cam)
        assert not fails, (deg, fails[:8])
        assert np.all(kern[4][K - 1:] == 0.0)
        kern0, _, _ = sc.launch(deg, mode, m_dst, gn_dst, form=0)
        assert np.all(np.isnan(kern0[4][K - 1:])), "form 0 writes no sh_rest row above the degree"


def test_skipped_and_unskipped_rows(cuda):
    """All-zero record gradients (and o_rec = 0 records, which the raster gives zero) are skipped: zero in forms 0 and 1; a depth
    slot alone (depth mode) and a normal row alone (normal mode) are not."""
    case = CASES["opacity"]
    p = {k: v.copy() for k, v in case["params"].items()}
    p["opacity"][0] = -200.0                                   # sigma underflows: o_rec = 0, record gradient zero
    sc = Scene(cuda, dict(case, params=p))
    rng = np.random.default_rng(9)
    m_src, gn_src = _record_grad(sc.N, rng, depth_only=(4, 5), normal_only=(6, 7), zero=(0, 8, 9))
    m_dst, gn_dst = sc.src_order(m_src.T).T.copy(), sc.src_order(gn_src.T).T.copy()
    pos = lambda i: int(np.flatnonzero(sc.src_order(np.arange(sc.N)) == i)[0])
    for form in (0, 1):
        for mode in ({f: True for f in FLAGS}, {f: False for f in FLAGS}):
            kern, _, _ = sc.launch(3, mode, m_dst, gn_dst, form=form)
            flat = [o.reshape(-1, sc.N) for o in kern[:4]] + [kern[4][:15].reshape(-1, sc.N), kern[5].reshape(-1, sc.N)]
            for i in (0, 8, 9):
                assert all(np.all(f[:, pos(i)] == 0.0) for f in flat), (form, mode, i)
            for i in (4, 5):
                xyz = kern[0].reshape(3, -1)[:, pos(i)]
                assert np.any(xyz != 0.0) == mode["depth"], (form, i)
            for i in (6, 7):
                rot = kern[2].reshape(4, -1)[:, pos(i)]
                assert np.any(rot != 0.0) == mode["normal"], (form, i)


def test_form1_clears_rows_past_the_visible_count(cuda):
    sc = Scene(cuda, CASES["rotated_camera"])
    rng = np.random.default_rng(3)
    mode = {f: True for f in FLAGS}
    A = sc.C + 2
    m, gn = _record_grad(A * S, rng)
    kern, _, _ = sc.launch(3, mode, m, gn, form=1, A=A, nvis=sc.C)
    for o in kern:
        assert np.all(o[..., sc.C:, :] == 0.0)
        assert np.all(np.isfinite(o))


def test_form2_accumulates_at_the_source_chunk(cuda):
    """Form 2 on dense buffers with random contents: visible chunks (non-contiguous ids) gain the form-0 result at their source
    chunk, bit for bit (the SH rows within an fma's rounding), untouched Gaussians and chunks keep their bits, and ``touched``
    marks exactly the visible chunks.  Three views accumulated equal the fp64 sum of the references within the bar."""
    case = CASES["quaternions"]
    p = {k: np.concatenate([v] * 20, -1) for k, v in case["params"].items()}
    sc = Scene(cuda, dict(case, params=p))
    assert sc.C >= 5
    rng = np.random.default_rng(11)
    ids = np.array([sc.C - 1, 1, sc.C - 3])
    mode = {f: True for f in FLAGS}
    m, gn = _record_grad(len(ids) * S, rng, zero=(0, 5))
    f0, cam0, _ = sc.launch(3, mode, m, gn, form=0, chunk_ids=ids)
    prev = [rng.normal(size=o.shape[:-2] + (sc.C, S)).astype(np.float32) for o in f0]
    out = [torch.from_numpy(x.copy()).to(cuda) for x in prev]
    touched = torch.zeros(sc.C, device=cuda)
    f2, cam2, _ = sc.launch(3, mode, m, gn, form=2, chunk_ids=ids, out=out, touched=touched)
    assert np.array_equal(cam0, cam2)
    assert np.array_equal(touched.cpu().numpy(), np.isin(np.arange(sc.C), ids).astype(np.float32))
    K = 16
    for j, (a, b, c) in enumerate(zip(prev, f0, f2)):
        want = a.astype(np.float64).copy()
        skip = np.zeros(want.shape[-2:], bool)
        for r, cid in enumerate(ids):
            add = b[..., r, :]
            if j == 4:
                add = np.where(np.isnan(add), 0.0, add)[:K - 1]
                want[:K - 1, ..., cid, :] = (a[:K - 1, ..., cid, :] + add).astype(np.float32)
            else:
                want[..., cid, :] = (a[..., cid, :] + add).astype(np.float32)
            skip[cid] = True
        zero_rows = np.zeros_like(skip)
        for r, cid in enumerate(ids):
            zero_rows[cid] = np.all(m[r * S:(r + 1) * S] == 0, 1) & np.all(gn[r * S:(r + 1) * S] == 0, 1)
        assert np.array_equal(c[..., ~skip], a[..., ~skip]), j                 # untouched chunks keep their bits
        assert np.array_equal(c[..., zero_rows], a[..., zero_rows]), j         # skipped Gaussians keep their bits
        if j in (3, 4):
            tol = 2.0 ** -23 * (np.abs(a) + np.abs(want - a))
            assert np.all(np.abs(c - want) <= tol), j
        else:
            assert np.array_equal(c, want.astype(np.float32)), j
    # three views accumulate to the fp64 sum
    out = [torch.zeros(x.shape, device=cuda) for x in prev]
    acc = {k: 0.0 for k in ("xyz", "scale", "rot", "opacity", "sh")}
    bars = {k: 0.0 for k in acc}
    for v in range(3):
        m, gn = _record_grad(len(ids) * S, rng)
        sc.launch(3, mode, m, gn, form=2, chunk_ids=ids, out=out, touched=touched)
        msrc = np.zeros((sc.N, 12), np.float32)
        gsrc = np.zeros((sc.N, 4), np.float32)
        for r, cid in enumerate(ids):
            msrc[cid * S:(cid + 1) * S] = m[r * S:(r + 1) * S]
            gsrc[cid * S:(cid + 1) * S] = gn[r * S:(r + 1) * S]
        ref = sc.reference(3, mode, msrc, gsrc)
        chain = pg.chain_magnitude(ref, sc.view, sc.hw, aa=True, filt=sc.p["filt"], normal=True, exact=True)
        for k in acc:
            acc[k] = acc[k] + ref["grads"][k]
            bars[k] = bars[k] + 1e-4 * np.abs(ref["grads"][k]) + 1e-6 * ref["mag"][k] + CHAIN * chain.get(k, 0.0)
    got = dict(xyz=out[0].cpu().numpy().reshape(3, -1), scale=out[1].cpu().numpy().reshape(3, -1),
               rot=out[2].cpu().numpy().reshape(4, -1), opacity=out[5].cpu().numpy().reshape(-1),
               sh=np.concatenate([out[3].cpu().numpy(), out[4].cpu().numpy()]).reshape(16, 3, -1))
    for k in acc:
        assert np.all(np.abs(got[k] - acc[k]) <= bars[k]), k
    # at degree 1 the dense sh_rest rows above the degree keep their bits
    buf = [torch.from_numpy(x.copy()).to(cuda) for x in prev]
    m, gn = _record_grad(len(ids) * S, rng)
    sc.launch(1, mode, m, gn, form=2, chunk_ids=ids, out=buf, touched=touched)
    assert np.array_equal(buf[4].cpu().numpy()[3:], prev[4][3:])
    assert not np.array_equal(buf[4].cpu().numpy()[:3], prev[4][:3])


def test_capacity_sized_launch(cuda):
    """A > visible count, as ViewWorkspace launches: the camera partials past the visible count are zero, d_cam is bit-identical to
    the exact-size launch, and the visible rows are the exact launch's."""
    sc = Scene(cuda, CASES["needles_sizes"])
    rng = np.random.default_rng(2)
    m, gn = _record_grad(sc.C * S, rng)
    for mode in ({f: True for f in FLAGS}, dict({f: False for f in FLAGS}, cam=True)):
        exact, cam_e, part_e = sc.launch(3, mode, m, gn, form=0)
        A = sc.C + 37
        mc = np.concatenate([m, rng.normal(size=(37 * S, 12)).astype(np.float32)])
        gc = np.concatenate([gn, rng.normal(size=(37 * S, 4)).astype(np.float32)])
        cap, cam_c, part_c = sc.launch(3, mode, mc, gc, form=0, A=A, nvis=sc.C,
                                       chunk_ids=np.concatenate([sc.perm, np.zeros(37, np.int64)]))
        part_c = part_c.cpu().numpy()
        assert np.all(part_c[sc.C:] == 0.0)
        assert np.array_equal(part_c[:sc.C], part_e.cpu().numpy())
        assert np.array_equal(cam_c, cam_e)
        for a, b in zip(exact, cap):
            assert np.array_equal(a[..., :sc.C, :], b[..., :sc.C, :], equal_nan=True)


@pytest.mark.parametrize("S_", [32, 128, 1024])
def test_camera_grad_sum(cuda, S_):
    """camera_grad_sum_kernel over A = 1 .. 4097 chunks: d_cam against the fp64 sum of the per-Gaussian camera terms.  The chunks
    repeat 7 source chunks, so the reference is 7 chunks' worth of Gaussians."""
    rng = np.random.default_rng(S_)
    n = 7 * S_
    Vi = np.linalg.inv(CASES["rotated_camera"]["cam"][0].astype(np.float64))
    vs = np.stack([rng.uniform(-1, 1, n), rng.uniform(-0.7, 0.7, n), rng.uniform(1.5, 5, n), np.ones(n)], 1)
    params = pg._gaussians((vs @ Vi)[:, :3], np.exp(rng.uniform(-5, -2, (n, 3))), rng.normal(size=(n, 4)), rng.uniform(-3, 5, n), rng)
    sc = Scene(cuda, dict(CASES["rotated_camera"], params=params), chunk=S_)
    mode = dict({f: False for f in FLAGS}, cam=True)
    m_src, _ = _record_grad(n, rng)
    ref = sc.reference(0, mode, m_src, None)
    chunk_cam = ref["cam_each"].reshape(7, S_, 2, 4, 4).sum(1)
    chunk_mag = ref["mag_cam_each"].reshape(7, S_, 2, 4, 4).sum(1)
    for A in (1, 31, 32, 33, 1023, 1024, 1025, 4097):
        if A * S_ > 5_000_000:
            continue
        ids = np.arange(A) % 7
        m = np.concatenate([m_src.reshape(7, S_, 12)[i] for i in ids])
        try:
            _, d_cam, _ = sc.launch(0, mode, m, np.zeros((A * S_, 4), np.float32), chunk_ids=ids)
        except _lib.LiteGSB200Error as e:
            # the camera instantiation has no launch bounds: where it cannot run S threads the launch itself fails
            if A == 1 and "resources" in str(e):
                pytest.skip(f"the camera instantiation does not launch at S = {S_}: {e}")
            raise
        want = chunk_cam[ids].sum(0)
        mag = chunk_mag[ids].sum(0)
        bar = 1e-4 * np.abs(want) + 1e-6 * mag
        assert np.all(np.abs(d_cam - want) <= bar), (A, np.abs(d_cam - want).max(), bar.min())
