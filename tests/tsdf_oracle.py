"""fp64 numpy restatement of TSDF fusion and marching-cubes extraction (include/r3dg_b200.h, r3dg_tsdf_*), the
marching-cubes table parsed from the repository's header (csrc/mc_table.cuh), mesh-topology checks, and the analytic
sphere views the tests fuse."""
import math
import os
import re

import numpy as np

from helpers import ROOT

TABLE = os.path.join(ROOT, "relightable3dgaussian_b200", "csrc", "mc_table.cuh")


def parse_table(path=TABLE):
    """(edges [12,2], count [256], tris [256, max, 3] with -1 for unused) from the header."""
    src = open(path).read()
    body = lambda name: re.search(name + r"\[[^=]*=\s*\{(.*?)\};", src, re.S).group(1)
    nums = lambda s: [int(x) for x in re.findall(r"\d+", s)]
    edges = np.array(nums(body("kMcEdge")), dtype=np.int64).reshape(12, 2)
    count = np.array(nums(body("kMcCount")), dtype=np.int64)
    mx = int(re.search(r"kMcMaxTris = (\d+);", src).group(1))
    tris = np.array(nums(body("kMcTris")), dtype=np.int64).reshape(256, mx, 3)
    tris[tris == 255] = -1
    return edges, count, tris


def cam_rows(settings):
    """[(view [4,4] float64 of the fp32 matrix, fx, fy, cx, cy, W, H)] of GaussianRasterizationSettings or cameras."""
    out = []
    for s in settings:
        W, H = s.image_width, s.image_height
        vm = np.asarray(s.viewmatrix.detach().cpu().numpy(), dtype=np.float64)
        out.append((vm, W / (2.0 * s.tanfovx), H / (2.0 * s.tanfovy), float(s.cx), float(s.cy), W, H))
    return out


def grid_points(origin, voxel_size, dims):
    i, j, k = np.meshgrid(*[np.arange(n, dtype=np.float64) for n in dims], indexing="ij")
    o = np.asarray(origin, dtype=np.float64)
    return np.stack([o[0] + voxel_size * i, o[1] + voxel_size * j, o[2] + voxel_size * k], axis=-1)


def integrate(tsdf, weight, color, origin, voxel_size, sdf_trunc, depth, rgb, cams, depth_trunc=math.inf):
    """Fuse views in order into float64 copies of (tsdf, weight, color or None).  depth [V,H,W], rgb [V,3,H,W] or None,
    cams from cam_rows.  Returns (tsdf, weight, color, near) where `near` marks grid points some view decided within
    1e-4 px of a rounding boundary or 1e-6 (relative) of a cut-off: fp32 may decide those differently."""
    t, w = tsdf.astype(np.float64).copy(), weight.astype(np.float64).copy()
    c = None if color is None else color.astype(np.float64).copy()
    pts = grid_points(origin, voxel_size, t.shape).reshape(-1, 3)
    tf, wf = t.reshape(-1), w.reshape(-1)
    cf = None if c is None else c.reshape(-1, 3)
    near = np.zeros(tf.shape, dtype=bool)
    for v, (vm, fx, fy, cx, cy, W, H) in enumerate(cams):
        p = pts @ vm[:3, :3] + vm[3, :3]
        X, Y, Z = p[:, 0], p[:, 1], p[:, 2]
        near |= np.abs(Z) < 1e-6
        ok = Z > 0
        Zs = np.where(ok, Z, 1.0)
        u, vv = fx * X / Zs + cx + 0.5, fy * Y / Zs + cy + 0.5
        for q in (u, vv):
            near |= ok & (np.abs(q - np.round(q)) < 1e-4)
        pu, pv = np.floor(u), np.floor(vv)
        ok &= (pu >= 0) & (pu < W) & (pv >= 0) & (pv < H)
        iu, iv = np.where(ok, pu, 0).astype(np.int64), np.where(ok, pv, 0).astype(np.int64)
        D = depth[v].astype(np.float64)[iv, iu]
        near |= ok & np.isfinite(D) & (np.abs(D - depth_trunc) <= 1e-6 * np.abs(D))
        ok &= np.isfinite(D) & (D > 0) & (D <= depth_trunc)
        sdf = D - Z
        near |= ok & (np.abs(sdf + sdf_trunc) <= 1e-6 * np.maximum(np.abs(D), 1.0))
        ok &= sdf >= -sdf_trunc
        obs = np.minimum(1.0, sdf / sdf_trunc)
        w1 = wf + 1.0
        tf[:] = np.where(ok, (tf * wf + obs) / w1, tf)
        if cf is not None:
            col = rgb[v].astype(np.float64)[:, iv, iu].T
            cf[:] = np.where(ok[:, None], (cf * wf[:, None] + col) / w1[:, None], cf)
        wf[:] = np.where(ok, w1, wf)
    return t, w, c, near.reshape(t.shape)


def marching_cubes(tsdf, weight, color, origin, voxel_size, table=None):
    """(verts [N,3], faces [F,3], colors [N,3] or None) in the definition's order, in float64."""
    edges, count, tris = table if table is not None else parse_table()
    NX, NY, NZ = tsdf.shape
    t = tsdf.astype(np.float64)
    inside, obs = tsdf < 0, weight > 0
    cv = np.ones((NX - 1, NY - 1, NZ - 1), dtype=bool)
    for c in range(8):
        a, b, d = c & 1, (c >> 1) & 1, (c >> 2) & 1
        cv &= obs[a:NX - 1 + a, b:NY - 1 + b, d:NZ - 1 + d]
    CV = np.zeros((NX + 1, NY + 1, NZ + 1), dtype=bool)
    CV[1:NX, 1:NY, 1:NZ] = cv
    shp = (NX, NY, NZ)
    flags = np.zeros(shp + (3,), dtype=bool)
    # cells sharing the +axis edge at (i, j, k): lower corner (i, j-1|j, k-1|k) for x, etc.  CV is offset by 1.
    adj = [np.zeros(shp, dtype=bool) for _ in range(3)]
    for p in (0, 1):
        for q in (0, 1):
            adj[0] |= CV[1:, p:p + NY, q:q + NZ]
            adj[1] |= CV[p:p + NX, 1:, q:q + NZ]
            adj[2] |= CV[p:p + NX, q:q + NY, 1:]
    flags[:-1, :, :, 0] = adj[0][:-1] & (inside[:-1] != inside[1:])
    flags[:, :-1, :, 1] = adj[1][:, :-1] & (inside[:, :-1] != inside[:, 1:])
    flags[:, :, :-1, 2] = adj[2][:, :, :-1] & (inside[:, :, :-1] != inside[:, :, 1:])
    vid = np.cumsum(flags.reshape(-1)).reshape(flags.shape) - 1
    g, axis = np.nonzero(flags.reshape(-1, 3))
    ijk = np.stack(np.unravel_index(g, shp), axis=-1)
    ijk1 = ijk + np.eye(3, dtype=np.int64)[axis]
    v0 = t[tuple(ijk.T)]
    v1 = t[tuple(ijk1.T)]
    tt = v0 / (v0 - v1)
    verts = np.asarray(origin, dtype=np.float64) + voxel_size * ijk.astype(np.float64)
    verts[np.arange(len(g)), axis] += tt * voxel_size
    colors = None
    if color is not None:
        c0 = color[tuple(ijk.T)].astype(np.float64)
        c1 = color[tuple(ijk1.T)].astype(np.float64)
        colors = c0 + tt[:, None] * (c1 - c0)
    cube = np.zeros(cv.shape, dtype=np.int64)
    for c in range(8):
        a, b, d = c & 1, (c >> 1) & 1, (c >> 2) & 1
        cube |= inside[a:NX - 1 + a, b:NY - 1 + b, d:NZ - 1 + d].astype(np.int64) << c
    cells = np.stack(np.nonzero(cv), axis=-1)                   # cell order (C order of the lower corners)
    cc = cube[tuple(cells.T)]
    tri = tris[cc]                                              # [ncell, max, 3] edges
    e = np.where(tri < 0, 0, tri)
    corner = edges[e, 0]
    owner = cells[:, None, None, :] + np.stack([corner & 1, (corner >> 1) & 1, (corner >> 2) & 1], axis=-1)
    f = vid[owner[..., 0], owner[..., 1], owner[..., 2], e // 4]
    keep = (tri >= 0).all(axis=-1)
    faces = f[keep].reshape(-1, 3)
    return verts, faces, colors


# ---- mesh topology -------------------------------------------------------------------------------------------------

def directed_edges(faces):
    f = np.asarray(faces, dtype=np.int64)
    return np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])


def is_closed_oriented_manifold(faces):
    """Every directed edge appears exactly once and its reverse exists: a closed, consistently oriented 2-manifold
    (as far as edges tell; vertex links are checked by the Euler characteristic per component)."""
    de = directed_edges(faces)
    if len(de) == 0:
        return True
    key = de[:, 0] * (de.max() + 1) + de[:, 1]
    rev = de[:, 1] * (de.max() + 1) + de[:, 0]
    uniq = np.unique(key)
    return len(uniq) == len(key) and np.isin(rev, uniq).all()


def directed_edges_unique(faces):
    de = directed_edges(faces)
    if len(de) == 0:
        return True
    key = de[:, 0] * (de.max() + 1) + de[:, 1]
    return len(np.unique(key)) == len(key)


def component_labels(nv, faces):
    """Component label per vertex (union-find over the face edges); unused vertices are their own component."""
    parent = np.arange(nv)

    def find(x):
        while parent[x] != x:
            parent[x] = parent[parent[x]]
            x = parent[x]
        return x
    for a, b in directed_edges(faces):
        ra, rb = find(a), find(b)
        if ra != rb:
            parent[ra] = rb
    return np.array([find(v) for v in range(nv)])


def components(nv, faces):
    """Number of connected components of the vertices used by `faces`."""
    used = np.unique(np.asarray(faces).reshape(-1))
    return len(np.unique(component_labels(nv, faces)[used]))


def euler_per_component(nv, faces):
    """{component label: V - E + F} of each component."""
    f = np.asarray(faces, dtype=np.int64)
    lab = component_labels(nv, f)
    und = np.unique(np.sort(directed_edges(f), axis=1), axis=0)
    out = {}
    for l in np.unique(lab[np.unique(f.reshape(-1))]):
        out[int(l)] = int(np.unique(f[lab[f[:, 0]] == l]).size - (lab[und[:, 0]] == l).sum() + (lab[f[:, 0]] == l).sum())
    return out


def vertex_links_are_cycles(faces):
    """Every vertex's link (the edges opposite it in its faces) is one directed cycle: no pinched vertices."""
    f = np.asarray(faces, dtype=np.int64)
    link = {}
    for a, b, c in f:
        for v, p, q in ((a, b, c), (b, c, a), (c, a, b)):
            nxt = link.setdefault(int(v), {})
            if int(p) in nxt:
                return False
            nxt[int(p)] = int(q)
    for nxt in link.values():
        start = next(iter(nxt))
        x, n = nxt[start], 1
        while x != start:
            if x not in nxt:
                return False
            x, n = nxt[x], n + 1
        if n != len(nxt):
            return False
    return True


def euler(nv, faces):
    de = directed_edges(faces)
    und = np.unique(np.sort(de, axis=1), axis=0)
    return nv - len(und) + len(faces)


def signed_volume(verts, faces):
    v = np.asarray(verts, dtype=np.float64)[np.asarray(faces)]
    return float(np.einsum("fi,fi->f", v[:, 0], np.cross(v[:, 1], v[:, 2])).sum() / 6.0)


# ---- analytic sphere views -----------------------------------------------------------------------------------------

def sphere_depth(cam, spheres):
    """Camera-z depth [H,W] of the nearest hit of the rays of `cam` (synth.Camera) with spheres [(centre, r)]; 0 where
    no sphere is hit.  Pixel (x, y) has the camera ray ((x - cx)/fx, (y - cy)/fy, 1)."""
    vm = cam.viewmatrix.double().numpy()
    R, t = vm[:3, :3], vm[3, :3]                                # cam = x R + t
    W, H = cam.image_width, cam.image_height
    fx, fy = W / (2.0 * cam.tanfovx), H / (2.0 * cam.tanfovy)
    ys, xs = np.meshgrid(np.arange(H, dtype=np.float64), np.arange(W, dtype=np.float64), indexing="ij")
    d_cam = np.stack([(xs - cam.cx) / fx, (ys - cam.cy) / fy, np.ones_like(xs)], axis=-1)   # z = 1 in camera
    origin = -t @ R.T                                           # camera centre in world
    d_w = d_cam @ R.T
    best = np.full(xs.shape, np.inf)
    for cen, r in spheres:
        oc = origin - np.asarray(cen, dtype=np.float64)
        a = np.einsum("hwi,hwi->hw", d_w, d_w)
        b = 2.0 * np.einsum("hwi,i->hw", d_w, oc)
        c = oc @ oc - r * r
        disc = b * b - 4 * a * c
        s = (-b - np.sqrt(np.maximum(disc, 0.0))) / (2 * a)     # parameter along d_w = camera z
        best = np.where((disc >= 0) & (s > 0) & (s < best), s, best)
    return np.where(np.isfinite(best), best, 0.0)


def ring_cameras(W=256, H=256):
    """The 16 views of the tests: synth.make_camera k = 0..7 at elevations +30 and -30 degrees."""
    from relightable3dgaussian_b200 import synth
    return [synth.make_camera(k, W, H, elevation_deg=e) for e in (30.0, -30.0) for k in range(8)]
