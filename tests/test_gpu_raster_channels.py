"""The raster kernels with depth and normals against the fp64 oracle on constructed edge cases, at every compiled variant.

test_gpu_raster_edges.py holds the colour-only kernels to the oracle on hand-built records and tile lists.  This module runs the
same cases (imported from there: chunks, saturation, clamp, views, padded, needles and the screen-sized splat) through the
instantiations that render depth and normals, plus one case built for the clamp mask:
  * clampmask:  black splats (colour exactly 0) and splats with negative channels, rendered with clamp_zero: the colour upstream
                is masked where a channel composites to <= 0, while the depth and normal upstreams still flow.
Every record carries a view-space z in ndc[:, 2] (pack_kernel copies it into the record's depth slot), log-uniform over
[0.2, 1000] with exact ties and neighbours an ulp apart, and a unit normal in the side row nrec f32[V, N, 4] (components exactly
0 and +-1 among them, w = 0, different per view).

The fp64 reference is the oracle's colour composite on three colours (tests/depth_oracle.py, tests/normal_oracle.py): the
colour itself, (z / zs, 0, 0) with zs a power of two, so that D = zs x its red channel, and n / 2, so that N = 2 x it.  The
backward reference is the sum of the three passes run on the same T and last: the colour pass with the (masked) image gradient
and d_trans, the depth pass with g_z zs in channel 0 and the normal pass with 2 g_N.  The depth pass's d_color[0] / zs is the
record gradient's slot 10 (LGS_GRAD_DEPTH), the normal pass's d_color / 2 is grad_normal; the same passes run on |g| give
sum_px w |g| per splat, the scale of their bars.

Template arguments reached (D = depth, N = normal; {D, N, DN} below means depth only, normal only, both):
  raster_forward_kernel<TH, TW, STAT, false, false, D, N>  -- ch x stat x tile: 3 x 2 x 4 = 24, at 1, 2 and 4 warps per block;
  raster_backward_v2_kernel<TH, TW, STAT, TRANS, DET, D, N> -- ch x the STAT/TRANS/DET loop x tile: 3 x 8 x 4 = 96;
  the colour-only TRANS set: v2 and v2 deterministic (STAT x tile) and raster_backward_kernel<.., STAT, true, BULK, DEFER> for
  the deferred, butterfly and bulk forms, all with clamped_img."""
import functools
import itertools
import math

import numpy as np
import pytest
import torch

import oracle
from litegs_b200 import _lib, fused
from tests import test_gpu_raster_edges as edges
from tests.depth_oracle import depth_colour
from tests.normal_oracle import normal_colour
from tests.test_gpu_raster_edges import switch  # noqa: F401  (fixture)
from tests.util import scaled_err

pytestmark = pytest.mark.gpu
TOL = edges.TOL
TILES, TILE_IDS = edges.TILES, edges.TILE_IDS
GRAD_NAMES = edges.GRAD_NAMES
CHANNELS = {"depth": (True, False), "normal": (False, True), "both": (True, True)}
# Absolute part of the bar of slot 10 and grad_normal, per splat, as a fraction of sum_px w |g|.  The backward rebuilds each
# pixel's T front to back by dividing the final T by (1 - a), one rcp.approx and one multiply per list position, so w = a T carries a
# relative error that grows along the list: on the 1000-long lists of "chunks" and the saturated stacks it reaches ~1.1e-6.  The
# colour sums sum_px w g have the same error (test_backward_channel_layout_identities: with g_z = g_img[0] slot 10 is slot 5 to
# the bit), which the max-normalised record bar hides.
CH_ABS = 2e-6
FLAGS = list(itertools.product((False, True), repeat=3))     # (STAT, TRANS, DET)
P, f64, f32 = fused._ptr, edges.f64, np.float32

# largest error / bar seen per check family, printed when the module ends
RATIOS = {}


def note(family, err, bar):
    r = float(np.max(np.asarray(err, np.float64) / np.maximum(np.asarray(bar, np.float64), 1e-300))) if np.size(err) else 0.0
    RATIOS[family] = max(RATIOS.get(family, 0.0), r)
    return r


@pytest.fixture(scope="module", autouse=True)
def _report_ratios():
    yield
    for k, v in sorted(RATIOS.items()):
        print(f"[raster channels] largest error / bar, {k}: {v:.3g}")


# ---------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------

def case_clampmask(tile):
    """One view of random splats where every third is black and every third has negative channels (60 % of its channels)."""
    sc = edges._random_views(tile, 48, 64, 1, 160, 17)
    N = sc["ndc"].shape[2]
    rng = np.random.default_rng(18)
    col = rng.uniform(0.05, 0.95, (1, 3, N))
    col[:, :, 0::3] = 0.0
    neg = np.where(rng.random((1, 3, N)) < 0.6, rng.uniform(-0.9, -0.05, (1, 3, N)), col)
    col[:, :, 1::3] = neg[:, :, 1::3]
    return dict(sc, col=col.astype(f32))


CASES = {**edges.CASES, "clampmask": case_clampmask}
CLAMP_ZERO = {"clampmask"}                                   # cases whose forward writes clamp(c, 0, 1)
SPECIAL_N = np.array([(1, 0, 0), (-1, 0, 0), (0, 1, 0), (0, -1, 0), (0, 0, 1), (0, 0, -1),
                      (math.sqrt(0.5), -math.sqrt(0.5), 0), (0, math.sqrt(0.5), math.sqrt(0.5))])


def with_channels(sc, seed):
    """The scene plus z (in ndc[:, 2]) and normals, and the oracle's depth and normal colours (fp64, [V, 3, N])."""
    V, N = sc["ndc"].shape[0], sc["ndc"].shape[2]
    rng = np.random.default_rng(seed)
    z = np.exp(rng.uniform(math.log(0.2), math.log(1000.0), (V, N))).astype(f32)
    z[:, 1:N:7] = z[:, 0:N - 1:7]                                                  # exact ties with the record before
    z[:, 4:N:11] = np.nextafter(z[:, 3:N - 1:11], np.float32(np.inf))              # one ulp above it
    z[:, 9:N:13] = np.nextafter(z[:, 8:N - 1:13], np.float32(0))                   # one ulp below it
    if N > 6:
        z[:, 5], z[:, 6] = 0.2, 1000.0                                             # the ends of the range
    n = rng.normal(size=(V, N, 3))
    n /= np.linalg.norm(n, axis=-1, keepdims=True)
    for b in range(V):                                                             # axis and in-plane normals, per view
        sel = np.arange((2 + 3 * b) % 5, N, 5)
        n[b, sel] = SPECIAL_N[(np.arange(len(sel)) + b) % len(SPECIAL_N)]
    nrec = np.zeros((V, N, 4), f32)
    nrec[..., :3] = n
    ndc = sc["ndc"].copy()
    ndc[:, 2] = z
    dz = [depth_colour(z[b].astype(np.float64), np.float64) for b in range(V)]
    dcol = np.concatenate([c for c, _ in dz])
    zs = np.array([s for _, s in dz])
    ncol = np.concatenate([normal_colour(nrec[b, :, :3].T.astype(np.float64), np.float64) for b in range(V)])
    return dict(sc, ndc=ndc, z=z, zs=zs, nrec=nrec, dcol=dcol, ncol=ncol)


@functools.lru_cache(maxsize=None)
def scene(case, tile):
    return with_channels(CASES[case](tile), 100 + list(CASES).index(case))


@functools.lru_cache(maxsize=None)
def oracle_forward(case, tile):
    """img, T, last, fragment statistics and fragile mask of the colour, and D and N, from the fp64 oracle."""
    sc = scene(case, tile)

    def run(col, stat=False):
        return oracle.rasterize_forward(sc["pid"], sc["ranges"], f64(sc["ndc"]), f64(sc["inv"]), col, f64(sc["op"]), None, sc["H"],
                                        sc["W"], tile[0], tile[1], enable_statistic=stat, fragile_eps=edges.FRAGILE_EPS)
    img, T, last, fc, fw, frag = run(f64(sc["col"]), True)
    return dict(img=img, T=T, last=last, fc=fc, fw=fw, frag=frag, D=run(sc["dcol"])[0][:, 0] * sc["zs"][:, None, None],
                N=run(sc["ncol"])[0] * 2)


@functools.lru_cache(maxsize=None)
def upstreams(case, tile):
    """(d_img, d_depth, d_normal, d_trans) f32, random and zero on the oracle's fragile pixels; d_depth is scaled by 1 / zs so
    that its term z g_z of dalpha is of the order of the colour term."""
    sc = scene(case, tile)
    frag = oracle_forward(case, tile)["frag"]
    V, Hp, Wp = frag.shape
    rng = np.random.default_rng(7)
    g = rng.normal(size=(V, 3, Hp, Wp)).astype(f32)
    gz = (rng.normal(size=(V, 1, Hp, Wp)) / sc["zs"][:, None, None, None]).astype(f32)
    gn = rng.normal(size=(V, 3, Hp, Wp)).astype(f32)
    gt = rng.normal(size=(V, 1, Hp, Wp)).astype(f32)
    for a in (g, gz, gn, gt):
        a[np.broadcast_to(frag[:, None], a.shape)] = 0.0
    return g, gz, gn, gt


# ---------------------------------------------------------------------------------------------------
# launches through the C entry points (the host mirrors in fused.py take neither depth nor normals)
# ---------------------------------------------------------------------------------------------------

def dev(a, cuda):
    return None if a is None else (a if isinstance(a, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(a)).to(cuda))


def pack(cuda, sc):
    V, N = sc["ndc"].shape[0], sc["ndc"].shape[2]
    ndc, inv, col, op = (dev(sc[k], cuda) for k in ("ndc", "inv", "col", "op"))
    packed = torch.empty((V, N, 12), dtype=torch.float32, device=cuda)
    _lib.call("lgs_pack_params", P(ndc), P(inv), P(col), P(op), V, N, sc["H"], sc["W"], P(packed), fused._stream(cuda))
    return packed


def forward(cuda, sc, tile, stat=False, depth=False, normal=False, clamp_zero=False, nrec=None):
    """-> dict(img, T, last, fc, fw, D, N, packed) of the forward kernel under the current switches."""
    V, N = sc["ndc"].shape[0], sc["ndc"].shape[2]
    Hp, Wp = sc["Hp"], sc["Wp"]
    packed = pack(cuda, sc)
    pid, rg = dev(sc["pid"], cuda), dev(sc["ranges"], cuda)
    e = functools.partial(torch.empty, dtype=torch.float32, device=cuda)
    img, T, last = e((V, 3, Hp, Wp)), e((V, 1, Hp, Wp)), torch.empty((V, 1, Hp, Wp), dtype=torch.int16, device=cuda)
    fc = torch.zeros((V, 1, N), dtype=torch.int32, device=cuda) if stat else None
    fw = torch.zeros((V, 1, N), dtype=torch.float32, device=cuda) if stat else None
    D = e((V, 1, Hp, Wp)) if depth else None
    Nimg = e((V, 3, Hp, Wp)) if normal else None
    nr = dev(sc["nrec"] if nrec is None else nrec, cuda) if normal else None
    _lib.call("lgs_rasterize_forward_packed", P(pid), P(rg), P(packed), None, 0, V, N, pid.shape[1], sc["H"], sc["W"], tile[0], tile[1],
              int(stat), int(clamp_zero), P(img), P(T), P(last), P(fc), P(fw), None, P(D), P(nr), P(Nimg), fused._stream(cuda))
    return dict(img=img, T=T, last=last, fc=fc, fw=fw, D=D, N=Nimg, packed=packed)


def backward(cuda, sc, tile, packed, T, last, g, gt=None, clamped=None, gz=None, gn=None, stat=False):
    """-> dict(pg = packed_grad [V, N, 12], the four unpacked record gradients, gn = grad_normal [V, N, 4] or None)."""
    V, N = sc["ndc"].shape[0], sc["ndc"].shape[2]
    pid, rg = dev(sc["pid"], cuda), dev(sc["ranges"], cuda)
    T, last, g, gt, clamped, gz, gn = (dev(a, cuda) for a in (T, last, g, gt, clamped, gz, gn))
    e = functools.partial(torch.empty, dtype=torch.float32, device=cuda)
    pg, d_ndc, d_cov, d_col, d_op = e((V, N, 12)), e((V, 4, N)), e((V, 2, 2, N)), e((V, 3, N)), e((1, N))
    e1, e2 = e((V, 1, N)), e((V, 1, N))
    nr = dev(sc["nrec"], cuda) if gn is not None else None
    grad_n = e((V, N, 4)) if gn is not None else None
    _lib.call("lgs_rasterize_backward", P(pid), P(rg), P(packed), None, 0, P(T), P(last), P(g), P(gt), P(clamped), None, V, N,
              pid.shape[1], sc["H"], sc["W"], tile[0], tile[1], int(stat), P(pg), P(d_ndc), P(d_cov), P(d_col), P(d_op), P(e1), P(e2),
              P(gz), P(nr), P(gn), P(grad_n), fused._stream(cuda))
    return dict(pg=pg, d_ndc=d_ndc, d_cov2d_inv=d_cov, d_color=d_col, d_opacity=d_op, gn=grad_n)


@functools.lru_cache(maxsize=None)
def forward_state(cuda, case, tile, state):
    """(T, last, clamped image) for the backward.  state "oracle": the oracle's T and last; "kernel": the default forward's own.
    The clamped image is the default forward's clamp_zero output in either state (an input of the backward, like d_img)."""
    sc = scene(case, tile)
    edges._set(edges.DEFAULTS)
    k = forward(cuda, sc, tile, clamp_zero=True)
    clamped = k["img"].cpu().numpy()
    if state == "oracle":
        o = oracle_forward(case, tile)
        return o["T"].astype(f32), o["last"], clamped
    return k["T"].cpu().numpy(), k["last"].cpu().numpy(), clamped


def _oracle_backward(sc, tile, col, T, last, g, gt=None):
    return oracle.rasterize_backward(sc["pid"], sc["ranges"], f64(sc["ndc"]), f64(sc["inv"]), col, f64(sc["op"]), None, f64(T), last,
                                     f64(g), None if gt is None else f64(gt), 1.0, sc["H"], sc["W"], tile[0], tile[1])[:4]


@functools.lru_cache(maxsize=None)
def reference(cuda, case, tile, state, part):
    """One oracle pass on the backward's forward state -> (four record gradients, channel gradient, its bar).
    part "colour" / "colour_trans": the colour with d_img masked by the clamped image (and d_trans); no channel gradient.
    part "depth": colour (z / zs, 0, 0), upstream g_z zs -> slot 10 = d_color[0] / zs [V, N], bar sum w |g_z|.
    part "normal": colour n / 2, upstream 2 g_N -> grad_normal = d_color / 2 [V, 3, N], bar sum w |g_N|."""
    sc = scene(case, tile)
    T, last, clamped = forward_state(cuda, case, tile, state)
    g, gz, gn, gt = upstreams(case, tile)
    if part.startswith("colour"):
        return _oracle_backward(sc, tile, f64(sc["col"]), T, last, np.where(clamped > 0, g, 0.0),
                                gt if part == "colour_trans" else None), None, None
    if part == "depth":
        zs = sc["zs"][:, None, None, None]
        up = np.zeros(g.shape)
        up[:, :1] = f64(gz) * zs
        r = _oracle_backward(sc, tile, sc["dcol"], T, last, up)
        up[:, :1] = np.abs(f64(gz)) * zs
        bar = _oracle_backward(sc, tile, sc["dcol"], T, last, up)[2][:, 0] / sc["zs"][:, None]
        return r, r[2][:, 0] / sc["zs"][:, None], bar
    r = _oracle_backward(sc, tile, sc["ncol"], T, last, 2.0 * f64(gn))
    bar = _oracle_backward(sc, tile, sc["ncol"], T, last, 2.0 * np.abs(f64(gn)))[2] / 2
    return r, r[2] / 2, bar


# ---------------------------------------------------------------------------------------------------
# needles: the fp32 power's conditioning (test_gpu_raster_edges.py, COND) with depth and normals as colours
# ---------------------------------------------------------------------------------------------------

@functools.lru_cache(maxsize=None)
def needle_image_bounds(tile):
    """Per-pixel bounds on D [Hp, Wp] and N [3, Hp, Wp]: 2^-20 Q alpha |z| and 2^-20 Q alpha |n_k| summed over the needles."""
    sc = scene("needles", tile)
    bD, bN = np.zeros((sc["Hp"], sc["Wp"])), np.zeros((3, sc["Hp"], sc["Wp"]))
    for i in range(sc["ndc"].shape[2]):
        a, _, _, Q = edges._needle_fields(sc, i)
        t = edges.COND * Q * np.where(a >= 0.5 / 256, a, 0.0)
        bD += t * abs(float(sc["z"][0, i]))
        bN += t[None] * np.abs(sc["nrec"][0, i, :3].astype(np.float64))[:, None, None]
    return bD, bN


@functools.lru_cache(maxsize=None)
def needle_gradient_bounds(tile, trans, depth, normal):
    """test_gpu_raster_edges.needle_gradient_bounds with the whole dL/dpower of an isolated splat on black,
    alpha (c . g + z g_z + n . g_N - g_T), and the conditioning of slot 10 and grad_normal, 2^-20 sum alpha |g| Q.  For d_ndc, S
    sums the absolute value of each of these terms (the colour, depth, normal and transmittance terms of a pixel may cancel), and
    each pixel's term carries the conditioning 2^-20 Q on top of 1e-5: with d_trans the far ends of the 100:1 needles, where Q is
    largest, weigh more in the position gradient than with a colour loss alone, and every backward form differs from the oracle
    there by the same ~1.2e-5 S.
    -> (d_ndc, d_cov2d_inv, d_color, d_opacity, slot 10 [1, N], grad_normal [1, 3, N])."""
    sc = scene("needles", tile)
    g, gz, gn, gt = (f64(a[0]) for a in upstreams("needles", tile))
    N = sc["ndc"].shape[2]
    b_ndc, b_cov, b_col, b_op = np.zeros((1, 4, N)), np.zeros((1, 2, 2, N)), np.zeros((1, 3, N)), np.zeros((1, N))
    b_z, b_n = np.zeros((1, N)), np.zeros((1, 3, N))
    for i in range(N):
        a, dx, dy, Q = edges._needle_fields(sc, i)
        on = np.where(a >= 1.0 / 256, a, 0.0)
        terms = [float(sc["col"][0, c, i]) * g[c] for c in range(3)]
        if depth:
            terms.append(float(sc["z"][0, i]) * gz[0])
        if normal:
            terms += [float(sc["nrec"][0, i, k]) * gn[k] for k in range(3)]
        if trans:
            terms.append(-gt[0])
        dpw = on * sum(terms)
        adpw = on * sum(np.abs(t) for t in terms)        # the absolute per-pixel terms, one per upstream channel
        A, B, C = sc["A"][0, i], sc["B"][0, i], sc["C"][0, i]
        b_ndc[0, 0, i] = 0.5 * sc["W"] * (np.abs(adpw * (A * dx + B * dy)) * (1e-5 + edges.COND * Q)).sum()
        b_ndc[0, 1, i] = 0.5 * sc["H"] * (np.abs(adpw * (B * dx + C * dy)) * (1e-5 + edges.COND * Q)).sum()
        b_cov[0, 0, 0, i] = edges.COND * (np.abs(0.5 * dx * dx * dpw) * Q).sum()
        b_cov[0, 0, 1, i] = b_cov[0, 1, 0, i] = edges.COND * (np.abs(0.5 * dx * dy * dpw) * Q).sum()
        b_cov[0, 1, 1, i] = edges.COND * (np.abs(0.5 * dy * dy * dpw) * Q).sum()
        for c in range(3):
            b_col[0, c, i] = edges.COND * (np.abs(on * g[c]) * Q).sum()
            b_n[0, c, i] = edges.COND * (np.abs(on * gn[c]) * Q).sum()
        b_op[0, i] = edges.COND * (np.abs(dpw / float(sc["op"][0, i])) * Q).sum()
        b_z[0, i] = edges.COND * (np.abs(on * gz[0]) * Q).sum()
    return b_ndc, b_cov, b_col, b_op, b_z, b_n


# ---------------------------------------------------------------------------------------------------
# forward
# ---------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("tile", TILES, ids=TILE_IDS)
@pytest.mark.parametrize("stat", [False, True], ids=["nostat", "stat"])
@pytest.mark.parametrize("ch", list(CHANNELS))
@pytest.mark.parametrize("case", list(CASES))
def test_forward_channels_match_fp64_oracle(cuda, switch, case, ch, stat, tile):
    """img, T, last and the fragment counts bit-identical to the colour-only forward, the fragment weights to fp32 atomic order;
    per non-fragile pixel |D - D_ref| <= 1e-4 D_ref + 1e-7 zs (z > 0, so D_ref = sum w |z|) and |N - N_ref| <= 1e-4 max(1, |N_ref|),
    plus the needles' conditioning; at 1 and 2 warps per block bit-identical to 4; and with n_0 = z / zs, D = zs N_0 bit for bit."""
    sc, o = scene(case, tile), oracle_forward(case, tile)
    depth, normal = CHANNELS[ch]
    cz = case in CLAMP_ZERO
    switch()
    plain = forward(cuda, sc, tile, stat, clamp_zero=cz)
    got = forward(cuda, sc, tile, stat, depth, normal, cz)
    for name in ("img", "T", "last") + (("fc",) if stat else ()):
        assert torch.equal(got[name], plain[name]), name
    if stat:
        fw, fw0 = got["fw"].cpu().numpy().astype(np.float64), plain["fw"].cpu().numpy().astype(np.float64)
        assert (np.abs(fw - fw0) <= 1e-5 * np.abs(fw0)).all()
    for wpb in (1, 2):
        switch(warps_per_block=wpb)
        other = forward(cuda, sc, tile, stat, depth, normal, cz)
        for name in ("img", "T", "last", "D", "N") + (("fc",) if stat else ()):
            if got[name] is not None:
                assert torch.equal(other[name], got[name]), (wpb, name)
    switch()
    ok = ~o["frag"]
    assert np.array_equal(got["last"].cpu().numpy().astype(np.uint16)[:, 0][ok], o["last"].astype(np.uint16)[:, 0][ok])
    bD, bN = needle_image_bounds(tile) if case == "needles" else (0.0, 0.0)
    if depth:
        Dk = got["D"].cpu().numpy()[:, 0].astype(np.float64)
        bar = 1e-4 * np.abs(o["D"]) + 1e-7 * sc["zs"][:, None, None] + bD
        err = np.abs(Dk - o["D"])
        assert (err[ok] <= bar[ok]).all(), note("forward D", err[ok], bar[ok])
        note("forward D", err[ok], bar[ok])
    if normal:
        Nk = got["N"].cpu().numpy().astype(np.float64)
        bar = 1e-4 * np.maximum(1.0, np.abs(o["N"])) + bN
        err = np.abs(Nk - o["N"])
        m3 = np.broadcast_to(ok[:, None], err.shape)
        assert (err[m3] <= bar[m3]).all(), note("forward N", err[m3], bar[m3])
        note("forward N", err[m3], bar[m3])
    nx = sc["nrec"].copy()
    nx[..., 0] = sc["z"] / sc["zs"][:, None].astype(f32)
    x = forward(cuda, sc, tile, stat, True, True, cz, nrec=nx)
    zs = torch.tensor(sc["zs"], dtype=torch.float32, device=cuda).view(-1, 1, 1)
    assert torch.equal(x["D"][:, 0], zs * x["N"][:, 0])
    if depth:
        assert torch.equal(x["D"], got["D"])


# ---------------------------------------------------------------------------------------------------
# backward
# ---------------------------------------------------------------------------------------------------

def check_backward(out, case, tile, ch, trans, refs, family):
    """The four record gradients against the sum of the oracle passes -- max-normalised 1e-4, the needles per splat -- and slot 10
    and grad_normal per splat to |err| <= 1e-4 |ref| + CH_ABS sum_px w |g| (+ the needles' conditioning)."""
    depth, normal = CHANNELS[ch] if ch else (False, False)
    ref = [sum(r[0][k] for r in refs) if k != 2 else refs[0][0][2] for k in range(4)]     # d_color: the colour pass's alone
    got = [out[k].cpu().numpy().astype(np.float64) for k in GRAD_NAMES]
    nb = needle_gradient_bounds(tile, trans, depth, normal) if case == "needles" else None
    for k, name in enumerate(GRAD_NAMES):
        if case == "needles":
            err, bar = np.abs(got[k] - ref[k]), TOL * np.abs(ref[k]) + nb[k]
            w = np.unravel_index(np.argmax(err - bar), err.shape)
            assert (err <= bar).all(), (family, name, note(family + " record", err, bar), w, err[w], bar[w], ref[k][w], got[k][w])
            note(family + " record", err, bar)
        else:
            e = scaled_err(got[k], ref[k])
            assert e < TOL, (family, name, e)
            note(family + " record", e, TOL)
    pg = out["pg"].cpu().numpy().astype(np.float64)
    if depth:
        _, rz, bz = refs[-2] if normal else refs[-1]
        err, bar = np.abs(pg[..., 10] - rz), TOL * np.abs(rz) + CH_ABS * bz + (nb[4] if nb else 0.0)
        assert (err <= bar).all(), (family, "slot 10", note(family + " slot 10", err, bar))
        note(family + " slot 10", err, bar)
    else:
        assert (pg[..., 10] == 0).all(), (family, "slot 10 written without depth")
    if normal:
        _, rn, bn = refs[-1]
        gn = out["gn"].cpu().numpy().astype(np.float64)
        assert (gn[..., 3] == 0).all()
        err, bar = np.abs(gn[..., :3].transpose(0, 2, 1) - rn), TOL * np.abs(rn) + CH_ABS * bn + (nb[5] if nb else 0.0)
        assert (err <= bar).all(), (family, "grad_normal", note(family + " grad_normal", err, bar))
        note(family + " grad_normal", err, bar)


@pytest.mark.parametrize("state", ["oracle", "kernel"])
@pytest.mark.parametrize("tile", TILES, ids=TILE_IDS)
@pytest.mark.parametrize("ch", list(CHANNELS))
@pytest.mark.parametrize("case", list(CASES))
def test_backward_channels_match_fp64_oracle(cuda, switch, case, ch, tile, state):
    """The v2 backward with depth and/or normals, for every (STAT, TRANS, DET), against the oracle passes run on the same forward
    state (the oracle's, or the kernel's own), with the clamp mask; with all three flags on, 1 and 2 warps per block bit-identical
    to 4 (deterministic mode)."""
    sc = scene(case, tile)
    depth, normal = CHANNELS[ch]
    T, last, clamped = forward_state(cuda, case, tile, state)
    g, gz, gn, gt = upstreams(case, tile)
    switch()
    packed = pack(cuda, sc)
    extra = ([reference(cuda, case, tile, state, "depth")] if depth else []) + \
            ([reference(cuda, case, tile, state, "normal")] if normal else [])
    args = dict(clamped=clamped, gz=gz if depth else None, gn=gn if normal else None)
    all_on = None
    for stat, trans, det in FLAGS:
        switch(deterministic=int(det))
        out = backward(cuda, sc, tile, packed, T, last, g, gt if trans else None, stat=stat, **args)
        refs = [reference(cuda, case, tile, state, "colour_trans" if trans else "colour")] + extra
        check_backward(out, case, tile, ch, trans, refs, f"v2{' det' if det else ''} {ch}"
                       f"{' stat' if stat else ''}{' trans' if trans else ''}")
        if stat and trans and det:
            all_on = out
    for wpb in (1, 2):
        switch(deterministic=1, warps_per_block=wpb)
        out = backward(cuda, sc, tile, packed, T, last, g, gt, stat=True, **args)
        for name in ("pg",) + GRAD_NAMES + (("gn",) if normal else ()):
            assert torch.equal(out[name], all_on[name]), (wpb, name)


@pytest.mark.parametrize("tile", TILES, ids=TILE_IDS)
@pytest.mark.parametrize("ch", list(CHANNELS))
@pytest.mark.parametrize("case", ["saturation", "views", "clampmask"])
def test_backward_channel_layout_identities(cuda, switch, case, ch, tile):
    """Deterministic mode, bit for bit, with and without STAT and TRANS: g_z = g_N = 0 leaves every slot of the colour-only run
    (and writes zeros to slot 10 and grad_normal); g_z = g_img[0] makes slot 10 the red colour slot (5), g_N = g_img the normal
    rows the colour slots (5, 6, 7); STAT on leaves every other slot; two runs are identical."""
    sc = scene(case, tile)
    depth, normal = CHANNELS[ch]
    T, last, clamped = forward_state(cuda, case, tile, "kernel")
    g, gz, gn, gt = upstreams(case, tile)
    switch(deterministic=1)
    packed = pack(cuda, sc)
    names = ("pg",) + GRAD_NAMES
    nostat = {}
    for trans, stat in itertools.product((False, True), repeat=2):
        t = gt if trans else None
        what = (trans, stat)
        off = backward(cuda, sc, tile, packed, T, last, g, t, clamped, stat=stat)
        zero = backward(cuda, sc, tile, packed, T, last, g, t, clamped, np.zeros_like(gz) if depth else None,
                        np.zeros_like(gn) if normal else None, stat)
        for name in names:
            assert torch.equal(zero[name], off[name]), (what, "zero upstream", name)
        if normal:
            assert not zero["gn"].any(), what
        same = backward(cuda, sc, tile, packed, T, last, g, t, None, g[:, :1] if depth else None, g if normal else None, stat)
        if depth:
            assert torch.equal(same["pg"][..., 10], same["pg"][..., 5]), what
        if normal:
            assert torch.equal(same["gn"][..., :3], same["pg"][..., 5:8]), what
        full = backward(cuda, sc, tile, packed, T, last, g, t, clamped, gz if depth else None, gn if normal else None, stat)
        again = backward(cuda, sc, tile, packed, T, last, g, t, clamped, gz if depth else None, gn if normal else None, stat)
        for name in names + (("gn",) if normal else ()):
            assert torch.equal(full[name], again[name]), (what, "second run", name)
        if not stat:
            nostat[trans] = full
        else:
            keep = [s for s in range(12) if s != 9]
            assert torch.equal(full["pg"][..., keep], nostat[trans]["pg"][..., keep]), (what, "statistics")
            if normal:
                assert torch.equal(full["gn"], nostat[trans]["gn"]), (what, "statistics")


@pytest.mark.parametrize("det", [False, True], ids=["fp32", "det"])
@pytest.mark.parametrize("tile", TILES, ids=TILE_IDS)
def test_views_in_one_launch_equal_single_view_launches_with_channels(cuda, switch, tile, det):
    """V = 3 with depth and normals in one launch against three V = 1 launches (per-view offsets of the records, nrec, d_depth,
    d_normal and grad_normal): forward bit for bit; the record gradients, slot 10 and grad_normal bit for bit in deterministic
    mode, max-normalised 1e-5 otherwise; d_opacity is view 0's."""
    sc = scene("views", tile)
    T, last, clamped = forward_state(cuda, "views", tile, "oracle")
    g, gz, gn, gt = upstreams("views", tile)
    switch(deterministic=int(det))
    full = forward(cuda, sc, tile, False, True, True)
    fb = backward(cuda, sc, tile, full["packed"], T, last, g, gt, clamped, gz, gn, stat=True)
    for b in range(3):
        v = slice(b, b + 1)
        one = dict(sc, ndc=sc["ndc"][v], inv=sc["inv"][v], col=sc["col"][v], pid=sc["pid"][v], ranges=sc["ranges"][v], nrec=sc["nrec"][v])
        f1 = forward(cuda, one, tile, False, True, True)
        for name in ("img", "T", "last", "D", "N", "packed"):
            assert torch.equal(full[name][v], f1[name]), (b, name)
        b1 = backward(cuda, one, tile, f1["packed"], T[v], last[v], g[v], gt[v], clamped[v], gz[v], gn[v], stat=True)
        pairs = [(fb[k][v], b1[k], k) for k in GRAD_NAMES[:3]] + [(fb["pg"][v][..., 10], b1["pg"][..., 10], "slot 10"),
                                                                   (fb["gn"][v], b1["gn"], "grad_normal")]
        if b == 0:
            pairs.append((fb["d_opacity"], b1["d_opacity"], "d_opacity"))
        for a, c, name in pairs:
            if det:
                assert torch.equal(a, c), (b, name)
            else:
                assert scaled_err(a.cpu().numpy(), c.cpu().numpy()) < 1e-5, (b, name)


@pytest.mark.parametrize("det", [False, True], ids=["v2", "v2_det"])
@pytest.mark.parametrize("size", list(edges.BIG))
def test_screen_sized_splat_with_depth_loss(cuda, switch, size, det):
    """The screen-sized splat of test_gpu_raster_edges.py at z ~ 1000 under a depth loss g_z = 1: z g_z dominates dalpha, so the
    raw moments grow ~370-fold past the colour-only ones (slot 2 passes 1e15 at 3840x2160), inside the deterministic accumulator's
    range.  Every record gradient and slot 10 within 1e-4 relative of the fp64 oracle."""
    sc, T, last, g, ref, _ = edges.big_case(size)
    tile = edges.BIG[size]["tile"]
    z = np.full((1, 1), 999.7, f32)
    sc = dict(sc, ndc=sc["ndc"].copy())
    sc["ndc"][:, 2] = z
    dcol, zs = depth_colour(z[0].astype(np.float64), np.float64)
    gz = g[:, :1].copy()                                          # 1, zero on the fragile pixels as d_img
    up = np.zeros(g.shape)
    up[:, :1] = f64(gz) * zs
    rd = _oracle_backward(sc, tile, dcol, T, last, up)
    want = [ref[k] + (rd[k] if k != 2 else 0.0) for k in range(4)] + [rd[2][:, 0] / zs]
    switch()
    packed = pack(cuda, sc)
    switch(deterministic=int(det))
    out = backward(cuda, sc, tile, packed, T, last, g, gz=gz)
    got = [out[k] for k in GRAD_NAMES] + [out["pg"][..., 10]]
    for a, b, name in zip(got, want, GRAD_NAMES + ("slot 10",)):
        a, b = a.cpu().numpy().astype(np.float64).reshape(-1), np.asarray(b).reshape(-1)
        live = np.abs(b) > 0
        assert np.array_equal(np.abs(a) > 0, live), name
        err = np.abs(a[live] - b[live]) / np.abs(b[live])
        assert err.max() < TOL, (name, err.max(), a[live], b[live])
        note("screen-sized splat, depth loss", err, TOL)


# ---------------------------------------------------------------------------------------------------
# colour only: d_trans and the clamp mask in every backward form
# ---------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("tile", TILES, ids=TILE_IDS)
@pytest.mark.parametrize("bwd", list(edges.BWD))
@pytest.mark.parametrize("case", list(CASES))
def test_colour_backward_with_trans_and_clamp_mask(cuda, switch, case, bwd, tile):
    """Every backward form of test_gpu_raster_edges.py with d_trans and clamped_img, with and without STAT, against the oracle
    with d_img masked where the clamped image is <= 0 and d_trans: the four record gradients to the same bars."""
    sc = scene(case, tile)
    T, last, clamped = forward_state(cuda, case, tile, "oracle")
    g, _, _, gt = upstreams(case, tile)
    switch()
    packed = pack(cuda, sc)
    refs = [reference(cuda, case, tile, "oracle", "colour_trans")]
    for stat in (False, True):
        switch(**edges.BWD[bwd])
        out = backward(cuda, sc, tile, packed, T, last, g, gt, clamped, stat=stat)
        check_backward(out, case, tile, None, True, refs, f"colour {bwd} trans clamp{' stat' if stat else ''}")
