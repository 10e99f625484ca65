"""project_forward_kernel against the fp64 record map (tests/project_grad_oracle.record) on constructed edge cases.

Every family of project_grad_oracle.constructed_cases(), and a family of forward-only edges (depth at the 0.2 cull and one ulp
either side of it, below 1e-2 and behind the camera; ndc just inside and just outside +-1.3 on both axes; record opacities on
the logit ulps that straddle the 1/255 floor after the antialiasing and 3D-filter factors; a Gaussian at the camera centre), runs
through lgs_project_forward alone in all 128 instantiations (SH degree 0..3 x tile 8x16, 12x16, 16x16, 8x8 x antialiasing x 3D
filter x normals), spread over at least three different chunks in an order that moves every chunk (no record is read from its own
slot), into outputs filled with NaN and sentinel integers.

Values, per Gaussian and component, where the view-space z is at least 1e-2 (J's clamp decisions made in fp32, as the kernel
makes them; the colour everywhere, since it does not depend on z):
  px, py, ndc   16 ulps of the absolute terms of v = w.Vm and h = v.P, carried through ndc = h / h_w (and to pixels);
  A, B, C       (2^-20 + 2^-19 kappa_c) max(|A|, |C|), kappa_c = (|c00 c11| + c01^2) / |det| of the conic;
  o             2^-20 |o|, plus 2^-22 (kappa_aa + kappa_c) |o| in the antialiased mode (DESIGN.md section 2);
  r, g, b       2^-20 (sum_k |b_k c_k| + 0.5), plus the colour's fp64 sensitivity to the direction times
                2^-21 (|p| + |cc|) / |p - cc|, the fp32 direction's error;
  z             4 ulps of sum_k |w_k Vm[k][2]|;
  normal        within 2^-20 of the fp32 frame's normal (tests/normal_oracle.normal_frame: a wrong axis or sign is off by O(1))
                with the frame's facing sign exactly, and within 2^-20 of the fp64 normal with that sign; slot 3 zero.  Where the
                fp64 facing dot product is within rounding of 0 the normal is not compared; those Gaussians are counted.
Gaussians whose rho is within rounding of 0 (project_grad_oracle.fragile) have their antialiased opacity masked, and are counted.

Structure, bit for bit: tile_count is oracle.get_allocate_size (the exact tile bound) on the kernel's own record, and above 0
exactly where test_gpu_tile_cover.live_mask accepts it; depth_key is the bits of the record's z where the count is above 0 and
all ones elsewhere; iota[dst] = dst; totals = (sum of counts, ~min key, max key) over the splats with pairs, zeros when there
are none.  Capacity-sized launches leave zero records, normal rows and counts and all-ones keys in the tail chunks.  Chunks of
1024 (896 with normals) with visible splats only in warps 16 and above exercise the block reduction of the totals.
"""
import numpy as np
import pytest
import torch

import oracle
from litegs_b200 import _lib, pipeline
from tests import normal_oracle as no
from tests import project_grad_oracle as pg
from tests.test_gpu_project_backward import Scene, _kappas
from tests.test_gpu_tile_cover import live_mask

pytestmark = pytest.mark.gpu

TILES = ((8, 16), (12, 16), (16, 16), (8, 8))
CASES = pg.constructed_cases()
FAMILIES = tuple(CASES) + ("forward_edges",)
QUANTITIES = ("px", "py", "ndc", "conic", "o", "rgb", "z", "normal")
FLOOR = np.float32(1.0) / np.float32(255.0)          # lgs_splat_setup's opacity floor, __fdiv_rn(1, 255)
U = 2.0 ** -24
KEY_SENTINEL, IOTA_SENTINEL, COUNT_SENTINEL = 0x5A5A5A5A, 0xA5A5A5A5, -7


# ----------------------------------------------------------------------------------------------------------------------------
# the launch
# ----------------------------------------------------------------------------------------------------------------------------

def to_src(sc, x):
    """[..., >= C*S] in dst order of sc's chunk permutation (the visible chunks) -> [..., N] in source order."""
    C, S = sc.C, sc.S
    y = np.asarray(x)[..., :C * S].reshape(*np.shape(x)[:-1], C, S)
    out = np.empty_like(y)
    out[..., sc.perm, :] = y
    return out.reshape(*np.shape(x)[:-1], -1)


def moved_scene(cuda, case, chunk=32, chunks=3):
    """Scene of a family spread over at least `chunks` chunks of `chunk`, each chunk a different cyclic run of the family (chunk 0
    the family in order) unless the family fills its chunks, in a chunk order that moves every chunk, so that no record is read from the slot it is written to.
    sc.n_family is the family's own size."""
    p = case["params"]
    n = p["xyz"].shape[1]
    N = max(chunks * chunk, -(-n // chunk) * chunk)
    j = np.arange(N)
    idx = j if N == n else (j + j // chunk) % n              # a family that fills its chunks is kept as it is
    params = {k: np.asarray(v)[..., idx] for k, v in p.items()}
    C = N // chunk
    seed = next(s for s in range(1000) if np.all(np.random.default_rng(s).permutation(C) != np.arange(C)))
    sc = Scene(cuda, dict(case, params=params), seed=seed, chunk=chunk)
    sc.n_family = n
    return sc


def launch(sc, deg, tile, aa, f3d, normal, *, chunk_ids=None, A=None, nvis=None):
    """lgs_project_forward on Scene sc into NaN / sentinel-filled outputs -> dict of numpy arrays in dst order."""
    cuda, d, S = sc.cuda, sc.dev, sc.S
    assert sc.C > 1 and np.all(sc.perm != np.arange(sc.C)), "every chunk must be read from another slot than it is written to"
    ids = sc.perm if chunk_ids is None else np.asarray(chunk_ids)
    A = len(ids) if A is None else A
    nvis = len(ids) if nvis is None else nvis
    ids_t = torch.zeros(A, dtype=torch.int64, device=cuda)
    ids_t[:len(ids)] = torch.as_tensor(ids, dtype=torch.int64)
    cnt = torch.tensor([nvis], dtype=torch.int32, device=cuda)
    n = A * S
    rec = torch.full((n, 12), float("nan"), device=cuda)
    nrm = torch.full((n, 4), float("nan"), device=cuda) if normal else None
    key = torch.full((n,), KEY_SENTINEL, dtype=torch.int32, device=cuda)
    iota = torch.full((n,), IOTA_SENTINEL - 2 ** 32, dtype=torch.int32, device=cuda)
    tcount = torch.full((n,), COUNT_SENTINEL, dtype=torch.int32, device=cuda)
    totals = torch.full((3,), -3, dtype=torch.int32, device=cuda)
    p = pipeline._ptr
    _lib.call("lgs_project_forward", deg, p(ids_t), p(cnt), p(d["view"]), p(d["proj"]), p(d["xyz"]), p(d["scale"]), p(d["rot"]),
              p(d["sh_0"]), p(d["sh_rest"]), p(d["opacity"]), sc.C, S, A, *sc.hw, *tile, p(rec), p(key), p(iota), p(tcount), p(totals),
              p(d["filt"]) if f3d else None, int(aa), p(nrm), pipeline._stream(cuda))
    torch.cuda.synchronize()
    u32 = lambda t: t.cpu().numpy().view(np.uint32)
    return dict(rec=rec.cpu().numpy(), normal=None if nrm is None else nrm.cpu().numpy(), key=u32(key), iota=u32(iota),
                count=tcount.cpu().numpy(), totals=u32(totals))


# ----------------------------------------------------------------------------------------------------------------------------
# the fp64 reference and its bars, per (family, degree, antialiasing, 3D filter)
# ----------------------------------------------------------------------------------------------------------------------------

class Reference:
    """fp64 records and bars of every Gaussian of sc (source order), for one degree and mode."""

    def __init__(self, sc, deg, aa, f3d):
        K = (deg + 1) ** 2
        P = dict(sc.p, sh=sc.p["sh"][:K])
        th, Vm, Pm = pg.leaves(P, sc.view, sc.proj)
        th = {k: v.detach() for k, v in th.items()}
        Vm, Pm = Vm.detach(), Pm.detach()
        hw = sc.hw
        H, W = hw
        filt = torch.as_tensor(sc.p["filt"], dtype=pg.F64) if f3d else None
        with torch.no_grad():
            v0 = pg.record(th, Vm, Pm, hw, deg)[1]["v"].numpy()
            pred = pg.clamp_decisions_fp32(v0, Pm.numpy())
            rec, it = pg.record(th, Vm, Pm, hw, deg, filt=filt, aa=aa, pred=pred)
        rec = rec.numpy()
        it = {k: v.numpy() for k, v in it.items()}
        self.rec, self.it = rec, it
        V = np.asarray(sc.view, np.float64)
        Pn = np.asarray(sc.proj, np.float64)
        xyz = np.asarray(sc.p["xyz"], np.float64)
        w = np.concatenate([xyz, np.ones_like(xyz[:1])])
        v = it["v"]
        h = np.einsum("in,ik->kn", v, Pn)
        self.v, self.h = v, h
        with np.errstate(divide="ignore", invalid="ignore"):         # h_w = 0 at the camera centre, which is not compared
            self.ndc = h[:2] / h[3]
        self.near = v[2] >= 1e-2                                   # where the values are compared
        # px, py, ndc: 16 ulps of the absolute terms of v and h, through ndc = h / h_w
        va = np.einsum("in,ik->kn", np.abs(w), np.abs(V))
        ha = np.einsum("kn,kj->jn", va, np.abs(Pn))
        e = 16 * U
        hw_abs = np.abs(h[3])
        dndc = e * (ha[:2] + np.abs(self.ndc) * ha[3]) / np.where(hw_abs > 0, hw_abs, 1.0)
        self.bar_ndc = dndc + e * np.abs(self.ndc)
        self.bar_pix = np.stack([self.bar_ndc[0] * W * 0.5 + e * (np.abs(rec[0]) + W),
                                 self.bar_ndc[1] * H * 0.5 + e * (np.abs(rec[1]) + H)])
        # conic
        ref_like = dict(it=it, proj=Pn)
        self.kc, self.ka = _kappas(ref_like, aa)
        mx = np.maximum(np.abs(rec[2]), np.abs(rec[4]))
        self.bar_conic = (2.0 ** -20 + 2.0 ** -19 * self.kc) * mx
        # opacity (the antialiasing factor's determinants carry kappa_aa, its denominator kappa_c)
        self.bar_o = 2.0 ** -20 * np.abs(rec[5])
        if aa:
            self.bar_o = self.bar_o + 2.0 ** -22 * (self.ka + self.kc) * np.abs(rec[5])
        self.fragile = pg.fragile(ref_like, sc.view, aa=True) if aa else np.zeros(rec.shape[1], bool)
        # colour: the sum's absolute terms, and the direction's fp32 error through the colour's sensitivity to it
        cc = -np.einsum("k,mk->m", V[3, :3], V[:3, :3])
        dv = xyz - cc[:, None]
        dist = np.sqrt((dv * dv).sum(0))
        rel = np.where(dist > 0, 2.0 ** -21 * (np.linalg.norm(xyz, axis=0) + np.linalg.norm(cc)) / np.where(dist > 0, dist, 1.0), 0.0)
        dirn = torch.as_tensor(it["dirn"]).clone().requires_grad_()
        sh = torch.as_tensor(np.asarray(P["sh"], np.float64))
        terms = pg.sh_basis(deg, dirn)[:, None, :] * sh                       # [K,3,N]
        col = terms.sum(0)
        sens = np.zeros((3, rec.shape[1]))
        if deg > 0:
            for c in range(3):
                g, = torch.autograd.grad(col[c].sum(), dirn, retain_graph=True)
                sens[c] = g.abs().sum(0).numpy()
        self.bar_rgb = 2.0 ** -20 * (terms.detach().abs().sum(0).numpy() + 0.5) + sens * rel
        # z
        self.bar_z = 4 * U * va[2]
        # normal: the fp32 frame decides axis and sign; the fp64 normal with that sign
        q32 = np.asarray(sc.p["rot"], np.float32)
        s32 = np.asarray(sc.p["scale"], np.float32)
        v32 = self._view_pos32(sc)
        self.frame32 = no.normal_frame(s32, q32, np.asarray(sc.view, np.float32), v32)
        ax = self.frame32["a"]
        nc64 = np.einsum("nk,kj->jn", it["R"][np.arange(ax.shape[0]), ax], V[:3, :3])
        self.n64 = self.frame32["sg"].astype(np.float64) * nc64
        dot = (nc64 * v[:3]).sum(0)
        # the facing sign is compared where the fp64 dot product is clear of rounding; the others are counted
        self.sign_clear = np.abs(dot) > 2.0 ** -16 * (np.abs(nc64) * np.abs(v[:3])).sum(0)
        self.n_sign_unclear = int((~self.sign_clear[:sc.n_family]).sum())

    @staticmethod
    def _view_pos32(sc):
        """The view position in fp32 as lgs_mvp_view sums it (exactly the kernel's under the axis camera)."""
        f = np.float32
        x = np.asarray(sc.p["xyz"], f)
        V = np.asarray(sc.view, f)
        return np.stack([((x[0] * V[0, k] + x[1] * V[1, k]) + x[2] * V[2, k]) + V[3, k] for k in range(3)]).astype(f)


_REFS = {}


def reference(key, sc, deg, aa, f3d):
    k = (key, deg, aa, f3d)
    if k not in _REFS:
        _REFS[k] = Reference(sc, deg, aa, f3d)
    return _REFS[k]


# ----------------------------------------------------------------------------------------------------------------------------
# the checks
# ----------------------------------------------------------------------------------------------------------------------------

def _ratio(got, want, bar, mask):
    err = np.abs(got.astype(np.float64) - want)
    r = np.where(mask, err / np.maximum(bar, 1e-30), 0.0)
    r = np.where(mask & ~np.isfinite(got), np.inf, r)
    return float(r.max()) if r.size else 0.0


def check_values(sc, out, ref, normal, worst):
    """Compare the visible chunks' records with the reference -> list of failures; worst[q] keeps the largest err / bar."""
    rec = to_src(sc, out["rec"].T)                        # [12, N] in source order
    fails = []
    near = ref.near

    def q(name, got, want, bar, mask):
        r = _ratio(got, want, bar, mask)
        worst[name] = max(worst.get(name, 0.0), r)
        if not r <= 1.0:
            bad = np.argwhere(np.broadcast_to(mask, got.shape) & ~(np.abs(got - want) <= bar)).tolist()[:4]
            fails.append((name, r, bad))
    q("px", rec[0], ref.rec[0], ref.bar_pix[0], near)
    q("py", rec[1], ref.rec[1], ref.bar_pix[1], near)
    q("ndc", rec[10:12], ref.ndc, ref.bar_ndc, near[None])
    q("conic", rec[2:5], ref.rec[2:5], ref.bar_conic[None], near[None])
    q("o", rec[5], ref.rec[5], ref.bar_o, near & ~ref.fragile)
    q("rgb", rec[6:9], ref.rec[6:9], ref.bar_rgb, np.ones((1, rec.shape[1]), bool))
    q("z", rec[9], ref.rec[9], ref.bar_z, near)
    if normal:
        nr = to_src(sc, out["normal"].T)
        if not np.all(nr[3] == 0.0):
            fails.append(("normal slot 3", None, np.flatnonzero(nr[3] != 0.0)[:4].tolist()))
        # axis and sign: the kernel's normal is the fp32 frame's within rounding (a wrong axis or sign is off by O(1)), and its
        # facing sign is the fp32 frame's exactly
        n32 = ref.frame32["n"].astype(np.float64)
        clear = ref.sign_clear[None]
        q("normal", nr[:3], ref.n64, np.full(nr[:3].shape, 2.0 ** -20), clear)
        sg = np.where((nr[:3] * ref.frame32["nc"]).sum(0) < 0, -1.0, 1.0)
        axis_sign = (np.all(np.abs(nr[:3] - n32) <= 2.0 ** -20, 0) & (sg == ref.frame32["sg"])) | ~ref.sign_clear
        if not axis_sign.all():
            fails.append(("normal axis / sign", None, np.flatnonzero(~axis_sign)[:4].tolist()))
    return fails


def check_structure(sc, out, tile, normal, A, nvis):
    """The bit-exact outputs of one launch of A chunks (nvis visible) -> list of failures."""
    S = sc.S
    H, W = sc.hw
    th, tw = tile
    fails = []
    N = A * S
    rec, cnt, key = out["rec"], out["count"], out["key"]
    if not np.array_equal(out["iota"], np.arange(N, dtype=np.uint32)):
        fails.append("iota")
    vis = np.arange(N) < nvis * S
    # the kernel's own fp32 record through the oracle's allocate size (the exact tile bound)
    r = rec[vis]
    n = r.shape[0]
    ndc = np.zeros((1, 4, n), np.float32)
    ndc[0, 0], ndc[0, 1], ndc[0, 2], ndc[0, 3] = r[:, 10], r[:, 11], 0.5, 1.0
    inv = np.zeros((1, 2, 2, n), np.float32)
    inv[0, 0, 0], inv[0, 0, 1], inv[0, 1, 0], inv[0, 1, 1] = r[:, 2], r[:, 3], r[:, 3], r[:, 4]
    _, _, alloc = oracle.get_allocate_size(ndc, np.ascontiguousarray(r[:, 9][None]), inv, np.ascontiguousarray(r[:, 5][None]),
                                           H, W, th, tw)
    if not np.array_equal(cnt[vis], alloc[0]):
        fails.append(("tile_count", np.flatnonzero(cnt[vis] != alloc[0])[:4].tolist()))
    live = live_mask(r[:, :6], r[:, 10:12], r[:, 9])
    if not np.array_equal(cnt[vis] > 0, live):
        fails.append(("count > 0 vs live", np.flatnonzero((cnt[vis] > 0) != live)[:4].tolist()))
    want_key = np.where(cnt[vis] > 0, r[:, 9].view(np.uint32), np.uint32(0xFFFFFFFF))
    if not np.array_equal(key[vis], want_key):
        fails.append(("depth_key", np.flatnonzero(key[vis] != want_key)[:4].tolist()))
    # the tail chunks: invisible records
    tail = ~vis
    if tail.any():
        if not (np.all(rec[tail] == 0.0) and np.all(cnt[tail] == 0) and np.all(key[tail] == 0xFFFFFFFF)):
            fails.append("tail chunks")
        if normal and not np.all(out["normal"][tail] == 0.0):
            fails.append("tail normal rows")
    has = cnt > 0
    want_tot = np.array([cnt.sum(), ~key[has].min(), key[has].max()] if has.any() else [0, 0, 0], np.int64).astype(np.uint32)
    if not np.array_equal(out["totals"], want_tot):
        fails.append(("totals", out["totals"].tolist(), want_tot.tolist()))
    return fails


def instantiations():
    for deg in range(4):
        for tile in TILES:
            for aa in (False, True):
                for f3d in (False, True):
                    for normal in (False, True):
                        yield deg, tile, aa, f3d, normal


# ----------------------------------------------------------------------------------------------------------------------------
# the forward-only edges
# ----------------------------------------------------------------------------------------------------------------------------

def _floor_gaussian(rng, n):
    z = 4.0
    u = pg._px(pg._cams()["axis"], z)
    return pg._gaussians(np.tile([[0.1, -0.05, z]], (n, 1)), np.tile([[4 * u, 3 * u, 2 * u]], (n, 1)), np.tile([[0.9, 0.1, 0.2, -0.3]], (n, 1)),
                         np.zeros(n), rng)


def _edge_params(rng):
    """The forward-only edges; the last three Gaussians are the opacity-floor ones, their logits set by land_floor."""
    ax = pg._cams()["axis"]
    xyz, s = [], []
    z02 = np.float32(0.2)
    for z in (z02, np.nextafter(z02, np.float32(1)), np.nextafter(z02, np.float32(0)), np.float32(5e-3), np.float32(-1.0)):
        u = pg._px(ax, 0.2)
        xyz.append([0.01, -0.008, float(z)])
        s.append([4 * u, 3 * u, 2.5 * u])
    z = 4.0
    u = pg._px(ax, z)
    for k, p in ((0, ax[1][0, 0]), (1, ax[1][1, 1])):
        for sign in (1.0, -1.0):
            for f in (1 - 1e-5, 1 + 1e-5):
                c = [0.03, -0.02, z]
                c[k] = sign * 1.3 * f * z / float(p)
                xyz.append(c)
                s.append([25 * u, 20 * u, 15 * u])              # reaches the image from 0.15 of its width outside
    xyz.append([0.0, 0.0, 0.0])                                 # at the camera centre: the direction guard
    s.append([2 * u, 2 * u, 2 * u])
    n = len(xyz)
    p = pg._gaussians(xyz, s, rng.normal(size=(n, 4)), np.full(n, 0.5), rng)
    fl = _floor_gaussian(rng, 3)
    return {k: np.concatenate([p[k], fl[k]], -1) for k in p}


def land_floor(cuda, aa, f3d):
    """Logits of the floor Gaussian whose record opacities (after the antialiasing and 3D-filter factors) straddle 1/255: the
    last logit ulp below it, the first at or above it and the next.  One launch over 128 consecutive fp32 logits around the fp64
    estimate."""
    rng = np.random.default_rng(1)
    p = _floor_gaussian(rng, 128)
    sc0 = moved_scene(cuda, dict(params=p, cam=pg._cams()["axis"], hw=pg.HW))
    ref = Reference(sc0, 0, aa, f3d)
    fac = ref.rec[5, 0] / (1.0 / (1.0 + np.exp(-0.0)))          # rho rho3 of the geometry (logit 0: sigma = 1/2)
    x0 = np.float32(-np.log(fac / float(FLOOR) - 1.0))
    xs = (np.array([x0]).view(np.int32) + np.arange(-64, 64, dtype=np.int32)).view(np.float32)
    xs = np.sort(xs)
    p["opacity"] = xs.copy()
    sc = moved_scene(cuda, dict(params=p, cam=pg._cams()["axis"], hw=pg.HW))
    out = launch(sc, 0, TILES[0], aa, f3d, False)
    o = to_src(sc, out["rec"][:, 5][None])[0]
    assert np.all(np.diff(o) >= 0), "record opacity not monotone in the logit"
    i = int(np.searchsorted(o, FLOOR, side="left"))
    assert 0 < i < 127, (aa, f3d, o[0], o[-1])
    assert o[i - 1] < FLOOR <= o[i]
    return xs[i - 1:i + 2]


def edge_scene(cuda, aa, f3d):
    p = _edge_params(np.random.default_rng(3))
    p["opacity"][-3:] = land_floor(cuda, aa, f3d)
    return moved_scene(cuda, dict(params=p, cam=pg._cams()["axis"], hw=pg.HW))


# ----------------------------------------------------------------------------------------------------------------------------
# the tests
# ----------------------------------------------------------------------------------------------------------------------------

def _report(family, worst, nfrag, nsign):
    print(f"\n[project_forward] {family}: largest err/bar " + ", ".join(f"{k} {worst.get(k, 0.0):.3g}" for k in QUANTITIES) +
          f"; fragile Gaussians masked {nfrag}, normal signs within rounding of a flip {nsign}")


@pytest.mark.parametrize("family", FAMILIES)
def test_family_matches_fp64_reference(cuda, family):
    """All 128 instantiations: each record component of each Gaussian within its bar, every structural output bit for bit."""
    scenes = {}
    worst, fails, nfrag, nsign = {}, [], 0, 0
    for deg, tile, aa, f3d, normal in instantiations():
        if family == "forward_edges":
            if (aa, f3d) not in scenes:
                scenes[(aa, f3d)] = edge_scene(cuda, aa, f3d)
            sc, key = scenes[(aa, f3d)], (family, aa, f3d)
        else:
            if None not in scenes:
                scenes[None] = moved_scene(cuda, CASES[family])
            sc, key = scenes[None], family
        ref = reference(key, sc, deg, aa, f3d)
        out = launch(sc, deg, tile, aa, f3d, normal)
        f = check_values(sc, out, ref, normal, worst)
        f += check_structure(sc, out, tile, normal, sc.C, sc.C)
        nfrag = max(nfrag, int(ref.fragile[:sc.n_family].sum()))
        nsign = max(nsign, ref.n_sign_unclear)
        fails += [(deg, tile, aa, f3d, normal, x) for x in f]
    _report(family, worst, nfrag, nsign)
    assert nfrag <= 2 and nsign <= 2, (nfrag, nsign)
    assert not fails, fails[:12]


def test_forward_edges_reach_their_conditions(cuda):
    """The forward-only edges land where they were built: the cull at z = 0.2 keeps only the ulp above, ndc just inside +-1.3 is
    live and reaches the image while just outside is not, and the floor Gaussians straddle 1/255 in every mode."""
    for aa in (False, True):
        for f3d in (False, True):
            sc = edge_scene(cuda, aa, f3d)
            out = launch(sc, 0, (16, 16), aa, f3d, False)
            cnt = to_src(sc, out["count"][None])[0]
            o = to_src(sc, out["rec"][:, 5][None])[0]
            assert cnt[0] == 0 and cnt[1] > 0 and cnt[2] == 0 and cnt[3] == 0 and cnt[4] == 0, cnt[:5]
            assert np.array_equal(cnt[5:13] > 0, [True, False] * 4), cnt[5:13]
            assert cnt[13] == 0
            n = sc.n_family
            assert o[n - 3] < FLOOR <= o[n - 2] <= o[n - 1] and o[n - 2] < o[n - 1], o[n - 3:n]
            assert cnt[n - 3] == 0 and cnt[n - 2] > 0 and cnt[n - 1] > 0


def test_capacity_sized_launch(cuda):
    """A > visible count, as ViewWorkspace launches: the visible chunks are the exact launch's bit for bit, the tail chunks are
    invisible records (zero record, normal row and count, all-ones key) and iota is dst everywhere."""
    sc = moved_scene(cuda, CASES["rotated_camera"])
    fails = []
    for deg, tile, aa, f3d, normal in instantiations():
        exact = launch(sc, deg, tile, aa, f3d, normal)
        A = sc.C + 3
        ids = np.concatenate([sc.perm, np.zeros(3, np.int64)])
        cap = launch(sc, deg, tile, aa, f3d, normal, chunk_ids=ids, A=A, nvis=sc.C)
        n = sc.C * sc.S
        same = all(np.array_equal(exact[k][:n], cap[k][:n], equal_nan=True) for k in ("rec", "key", "count")) and \
            (not normal or np.array_equal(exact["normal"], cap["normal"][:n]))
        if not same or not np.array_equal(exact["totals"], cap["totals"]):
            fails.append((deg, tile, aa, f3d, normal, "visible part differs"))
        fails += [(deg, tile, aa, f3d, normal, x) for x in check_structure(sc, cap, tile, normal, A, sc.C)]
    assert not fails, fails[:12]


def _wide_chunks(S):
    """Three chunks of S: chunk 0 holds the rotated-camera family in warps 16 and above only (its nearest and farthest splats
    among them), chunk 1 a few of its middle-depth splats in warp 0 and warp 20, chunk 2 nothing visible.  The rest are
    copies of the first Gaussian below the opacity floor."""
    case = CASES["rotated_camera"]
    p = case["params"]
    n = p["xyz"].shape[1]
    N = 3 * S
    slots = np.full(N, -1)
    slots[16 * 32:16 * 32 + n] = np.arange(n)
    vz = (np.concatenate([p["xyz"].astype(np.float64), np.ones((1, n))]).T @ case["cam"][0].astype(np.float64))[:, 2]
    mid = np.argsort(vz)[n // 2 - 2:n // 2 + 2]
    slots[S + np.array([0, 5, 20 * 32, 20 * 32 + 31])] = mid
    out = {}
    for k, v in p.items():
        fill = np.repeat(v[..., :1], N, -1)
        fill[..., slots >= 0] = v[..., slots[slots >= 0]]
        out[k] = fill
    out["opacity"][slots < 0] = -30.0
    return dict(case, params=out)


@pytest.mark.parametrize("normal", [False, True], ids=["S1024", "S896-normal"])
def test_wide_chunks_block_reduction(cuda, normal):
    """Chunks of 1024 threads (896, the limit of the heaviest normal instantiation, with normals), with the splats that carry the
    pairs and the extreme depth keys in warps 16 and above: every value and structural check, and the totals."""
    S = 896 if normal else 1024
    sc = moved_scene(cuda, _wide_chunks(S), chunk=S)
    worst, fails = {}, []
    for deg in range(4):
        for tile in TILES:
            for aa in (False, True):
                for f3d in (False, True):
                    ref = reference(("wide", S), sc, deg, aa, f3d)
                    out = launch(sc, deg, tile, aa, f3d, normal)
                    f = check_values(sc, out, ref, normal, worst)
                    f += check_structure(sc, out, tile, normal, sc.C, sc.C)
                    assert out["totals"][0] > 0
                    fails += [(deg, tile, aa, f3d, x) for x in f]
    _report(f"wide chunks S={S}", worst, 0, 0)
    assert not fails, fails[:12]
