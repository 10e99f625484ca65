"""Numpy restatement of mesh extraction (DESIGN.md section 1, "Mesh extraction"; csrc/mesh.cu): TSDF integration in the fp32
operation order the kernel uses, and marching tetrahedra on the Freudenthal subdivision in the canonical output order, so that
the kernels' arrays can be compared with these exactly.  Plus the mesh checks the tests share (closedness, orientation, Euler
characteristic, signed volume)."""
import numpy as np

F32 = np.float32
# edge directions 0..6 as (dx, dy, dz): x, y, z, x+y, x+z, y+z, x+y+z
DIRS = np.array([(1, 0, 0), (0, 1, 0), (0, 0, 1), (1, 1, 0), (1, 0, 1), (0, 1, 1), (1, 1, 1)], np.int64)
# the 6 tetrahedra 0 -> e_p1 -> e_p1 + e_p2 -> (1,1,1), permutations p in lexicographic order, as cube corners (bit 0 = +x,
# bit 1 = +y, bit 2 = +z), and the signs of the permutations
TETS = [(0, 1, 3, 7), (0, 1, 5, 7), (0, 2, 3, 7), (0, 2, 6, 7), (0, 4, 5, 7), (0, 4, 6, 7)]
TET_SIGN = [1, -1, -1, 1, 1, -1]
MASK_DIR = {1: 0, 2: 1, 4: 2, 3: 3, 5: 4, 6: 5, 7: 6}


def corner_offset(c):
    return np.array([c & 1, (c >> 1) & 1, (c >> 2) & 1], np.int64)


def lattice_points(origin, h, dims):
    """f32[nz,ny,nx] x, y, z of the lattice points: origin + index * h, each a rounded fp32 product and sum."""
    nx, ny, nz = dims
    o = [F32(v) for v in origin]
    h = F32(h)
    i, j, k = (np.arange(n, dtype=np.int64).astype(F32) for n in (nx, ny, nz))
    px, py, pz = o[0] + i * h, o[1] + j * h, o[2] + k * h
    return np.broadcast_to(px[None, None, :], (nz, ny, nx)), np.broadcast_to(py[None, :, None], (nz, ny, nx)), np.broadcast_to(pz[:, None, None], (nz, ny, nx))


def project(p0, p1, p2, view, proj, H, W):
    """The kernel's steps 1-2: view-space (x, y, z) = p~ V, then u = (x / z) fx + W/2, v = (y / z) fy + H/2 -> (z, u, v), fp32."""
    Vm = np.asarray(view, F32).reshape(4, 4)
    Pm = np.asarray(proj, F32).reshape(4, 4)
    p0, p1, p2 = (np.asarray(a, F32) for a in (p0, p1, p2))
    x, y, z = (((p0 * Vm[0, c] + p1 * Vm[1, c]) + p2 * Vm[2, c]) + Vm[3, c] for c in range(3))
    fx = (Pm[0, 0] * F32(W)) * F32(0.5)
    fy = (Pm[1, 1] * F32(H)) * F32(0.5)
    with np.errstate(divide="ignore", invalid="ignore"):
        u = (x / z) * fx + F32(W) * F32(0.5)
        v = (y / z) * fy + F32(H) * F32(0.5)
    return z, u, v


def unproject(u, v, ed, view, proj, H, W):
    """World points (fp64 [N,3]) that lgs_depth_normal's ray ((u + 0.5 - W/2) / fx, (v + 0.5 - H/2) / fy, 1) at expected depth ed
    reaches from pixel (u, v)."""
    Vm = np.asarray(view, np.float64).reshape(4, 4)
    Pm = np.asarray(proj, np.float64).reshape(4, 4)
    fx, fy = Pm[0, 0] * W * 0.5, Pm[1, 1] * H * 0.5
    X = np.stack([(u + 0.5 - W / 2) / fx * ed, (v + 0.5 - H / 2) / fy * ed, ed, np.ones_like(ed)], -1)
    return (X @ np.linalg.inv(Vm))[:, :3]


def integrate(vol, origin, h, trunc, depth, trans, views, projs, rgb=None, alpha_min=0.5, depth_far=np.inf):
    """vol = dict(tsdf, weight[, color]) numpy f32 arrays, updated in place with the views of the batch in index order."""
    tsdf, weight = vol["tsdf"], vol["weight"]
    color = vol.get("color")
    nz, ny, nx = tsdf.shape
    p0, p1, p2 = lattice_points(origin, h, (nx, ny, nz))
    trunc, alpha_min, depth_far = F32(trunc), F32(alpha_min), F32(depth_far)
    V, _, H, W = depth.shape
    for v in range(V):
        z, u, w = project(p0, p1, p2, views[v], projs[v], H, W)
        with np.errstate(invalid="ignore"):
            m = (z > F32(0.01)) & (u >= 0) & (u < F32(W)) & (w >= 0) & (w < F32(H))
        iu, iw = np.floor(np.where(m, u, 0)).astype(np.int64), np.floor(np.where(m, w, 0)).astype(np.int64)
        a = F32(1) - trans[v, 0][iw, iu]
        m &= a > alpha_min
        with np.errstate(divide="ignore", invalid="ignore"):
            ed = depth[v, 0][iw, iu] / a
            m &= ~(ed > depth_far)
            sdf = ed - z
            m &= ~(sdf < -trunc)
            t = np.minimum(F32(1), sdf / trunc)
        w0 = weight[m]
        w1 = w0 + F32(1)
        tsdf[m] = (tsdf[m] * w0 + t[m]) / w1
        if color is not None:
            for ch in range(3):
                with np.errstate(divide="ignore", invalid="ignore"):
                    e = np.minimum(F32(1), np.maximum(F32(0), rgb[v, ch][iw, iu] / a))
                color[ch][m] = (color[ch][m] * w0 + e[m]) / w1
        weight[m] = w1
    return vol


def new_volume(dims, color=True):
    nx, ny, nz = dims
    vol = dict(tsdf=np.ones((nz, ny, nx), F32), weight=np.zeros((nz, ny, nx), F32))
    if color:
        vol["color"] = np.zeros((3, nz, ny, nx), F32)
    return vol


def _shift(a, d):
    """a[k + dz, j + dy, i + dx] over the index range where it exists (the rest: False / 0)."""
    dx, dy, dz = (int(x) for x in d)
    out = np.zeros_like(a)
    nz, ny, nx = a.shape
    out[: nz - dz, : ny - dy, : nx - dx] = a[dz:, dy:, dx:]
    return out


def extract(tsdf, weight, origin, h, color=None, weight_min=1.0):
    """Marching tetrahedra -> (vertices f32[M,3], faces i32[F,3], colors u8[M,3] or None) in the canonical order."""
    nz, ny, nx = tsdf.shape
    N = tsdf.size
    ok = weight >= F32(weight_min)
    inside = tsdf < 0
    # cell with lower corner a valid: all 8 corners in the lattice and ok
    cell = np.zeros_like(ok)
    cell[: nz - 1, : ny - 1, : nx - 1] = True
    for c in range(8):
        cell &= _shift(ok, corner_offset(c))
    # edge a -> a + d in some valid cell: cells with lower corner a - o, o = 0 on the axes of d and 0 or 1 elsewhere
    has = np.zeros((7, nz, ny, nx), bool)
    for d in range(7):
        dd = DIRS[d]
        owner = np.zeros_like(ok)
        free = [ax for ax in range(3) if dd[ax] == 0]
        for bits in range(1 << len(free)):
            o = np.zeros(3, np.int64)
            for n, ax in enumerate(free):
                o[ax] = (bits >> n) & 1
            # owner(a) |= cell[a - o]
            src = cell
            ox, oy, oz = o
            sh = np.zeros_like(cell)
            sh[oz:, oy:, ox:] = src[: nz - oz, : ny - oy, : nx - ox]
            owner |= sh
        has[d] = owner & (inside != _shift(inside, dd)) & _valid_end(dd, (nz, ny, nx))
    hasf = has.reshape(7, N).T                                      # [N, 7]: canonical order is row-major
    vid = np.full(N * 7, -1, np.int64)
    flat = hasf.reshape(-1)
    vid[flat] = np.arange(int(flat.sum()))
    pl, dl = np.nonzero(hasf)
    kk, rem = np.divmod(pl, nx * ny)
    jj, ii = np.divmod(rem, nx)
    o = [F32(v) for v in origin]
    hh = F32(h)
    t = tsdf.reshape(-1)
    q = pl + DIRS[dl, 0] + DIRS[dl, 1] * nx + DIRS[dl, 2] * nx * ny
    ta, tb = t[pl], t[q]
    s = ta / (ta - tb)
    verts = np.empty((len(pl), 3), F32)
    for ax, idx in enumerate((ii, jj, kk)):
        pa = o[ax] + idx.astype(F32) * hh
        pb = o[ax] + (idx + DIRS[dl, ax]).astype(F32) * hh
        verts[:, ax] = pa + s * (pb - pa)
    cols = None
    if color is not None:
        cols = np.empty((len(pl), 3), np.uint8)
        for ch in range(3):
            c = color[ch].reshape(-1)
            cv = c[pl] + s * (c[q] - c[pl])
            cols[:, ch] = np.clip(np.rint(cv * F32(255)), 0, 255).astype(np.uint8)
    # faces
    cells = np.nonzero(cell.reshape(-1))[0]
    ins = np.stack([inside.reshape(-1)[cells + corner_offset(c) @ np.array([1, nx, nx * ny])] for c in range(8)], 1)
    recs = []                                                       # (cell, tet, tri, v0, v1, v2)

    def E(ci, t_, x, y):
        a, b = TETS[t_][x], TETS[t_][y]
        if (a & b) != a:
            a, b = b, a
        qq = ci + corner_offset(a) @ np.array([1, nx, nx * ny])
        return vid[qq * 7 + MASK_DIR[a ^ b]]

    for t_ in range(6):
        tc = TETS[t_]
        s_ = sum(ins[:, tc[v]].astype(np.int64) << v for v in range(4))
        for case in range(1, 15):
            sel = cells[s_ == case]
            if not len(sel):
                continue
            inn = [v for v in range(4) if (case >> v) & 1]
            out = [v for v in range(4) if not (case >> v) & 1]
            tris = []
            if len(inn) in (1, 3):
                a = inn[0] if len(inn) == 1 else out[0]
                b, c, d = [v for v in range(4) if v != a]
                pos = (TET_SIGN[t_] * (-1) ** a > 0) == (len(inn) == 1)
                tris = [(a, b, a, c, a, d)] if pos else [(a, b, a, d, a, c)]
            else:
                a, b = inn
                c, d = out
                odd = case in (5, 10)
                if TET_SIGN[t_] * (-1 if odd else 1) > 0:
                    tris = [(a, c, a, d, b, d), (a, c, b, d, b, c)]
                else:
                    tris = [(a, c, b, d, a, d), (a, c, b, c, b, d)]
            for r, tr in enumerate(tris):
                vs = [E(sel, t_, tr[2 * n], tr[2 * n + 1]) for n in range(3)]
                recs.append(np.stack([sel, np.full_like(sel, t_), np.full_like(sel, r), *vs], 1))
    if recs:
        R = np.concatenate(recs)
        R = R[np.lexsort((R[:, 2], R[:, 1], R[:, 0]))]
        faces = R[:, 3:].astype(np.int32)
    else:
        faces = np.zeros((0, 3), np.int32)
    assert (faces >= 0).all()
    return verts, faces, cols


def _valid_end(d, shape):
    nz, ny, nx = shape
    m = np.zeros(shape, bool)
    m[: nz - d[2], : ny - d[1], : nx - d[0]] = True
    return m


# ---- mesh checks ----------------------------------------------------------------------------------------------------------

def edge_counts(faces):
    """(undirected edge -> number of faces, directed edge -> number of faces) as (keys, counts) pairs."""
    f = np.asarray(faces, np.int64)
    a = np.concatenate([f[:, 0], f[:, 1], f[:, 2]])
    b = np.concatenate([f[:, 1], f[:, 2], f[:, 0]])
    M = int(f.max()) + 1 if f.size else 1
    und = np.unique(np.minimum(a, b) * M + np.maximum(a, b), return_counts=True)
    dire = np.unique(a * M + b, return_counts=True)
    return und, dire, M


def closed_and_oriented(faces):
    """Every edge in exactly two faces, traversed once in each direction."""
    (uk, uc), (dk, dc), M = edge_counts(faces)
    if not (uc == 2).all() or not (dc == 1).all():
        return False
    rev = (dk % M) * M + dk // M
    return bool(np.isin(rev, dk).all())


def euler(vertices, faces):
    (uk, _), _, _ = edge_counts(faces)
    used = np.unique(np.asarray(faces).reshape(-1)).size
    return used - uk.size + len(faces), used == len(vertices)


def signed_volume(vertices, faces):
    v = np.asarray(vertices, np.float64)[np.asarray(faces, np.int64)]
    return float(np.einsum("ij,ij->i", v[:, 0], np.cross(v[:, 1], v[:, 2])).sum() / 6.0)
