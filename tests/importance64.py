"""fp64 restatement of the importance sampler (include/r3dg_b200.h, IMPORTANCE SAMPLING), written from the header
text: the env table on the env-filter stencil's cells, the lattice numbers, the env / GGX / cosine strategies, their
pdfs and the balance-heuristic area.  The table's CDFs are rounded to fp32 as the build does; everything else is fp64.
Also the quadrature truth and the estimates of the plane-under-a-source scene the quality tests use."""
import math

import numpy as np

MASK = 0xFFFFFFFF


def lowbias32(x):
    x = np.asarray(x, dtype=np.uint64) & MASK
    x ^= x >> 16
    x = (x * 0x7FEB352D) & MASK
    x ^= x >> 15
    x = (x * 0x846CA68B) & MASK
    x ^= x >> 16
    return x


def lattice(seed, q, s, n):
    """(u1, u2) [len(q), n] of the n samples of strategy s at points q (the header's integer formulas)."""
    q = np.asarray(q, dtype=np.uint64).reshape(-1, 1)
    h = lowbias32(lowbias32(lowbias32(seed) ^ q) ^ np.uint64(s))
    h1, h2 = lowbias32(h ^ np.uint64(0)), lowbias32(h ^ np.uint64(1))
    k = np.arange(n, dtype=np.uint64)[None]
    a = (((k << np.uint64(32)) // np.uint64(n)) + h1) & MASK
    b = (k * np.uint64(0x9E3779B9) + h2) & MASK
    return (a >> np.uint64(8)).astype(np.float64) * 2.0 ** -24, (b >> np.uint64(8)).astype(np.float64) * 2.0 ** -24


def counts(N, mix=(0.5, 0.25, 0.25)):
    n_env = int(N * mix[0] + 0.5)
    n_eg = int(N * (mix[0] + mix[1]) + 0.5)
    return n_env, n_eg - n_env, N - n_eg


# ---- env table --------------------------------------------------------------------------------------------------------
def bands(He):
    dt = math.pi / (He - 1)
    j = np.arange(He)
    return np.maximum((j - 0.5) * dt, 0.0), np.minimum((j + 0.5) * dt, math.pi)


def cell_solid_angle(He, We):
    lo, hi = bands(He)
    return (np.cos(lo) - np.cos(hi)) * (2 * math.pi / (We - 1))                # [He], constant along a row


def build_table(env):
    """env [He,We,3] -> dict(row_cdf [He+1], vers / covers [He+1] (1 -+ cos of the band edges), col_cdf [He,We] (all
    rounded to fp32), pdf [He,We-1] (fp64 from the rounded CDFs), weight [He,We-1])."""
    env = np.asarray(env, dtype=np.float64)
    He, We = env.shape[:2]
    C = We - 1
    lum = 0.2126 * env[..., 0] + 0.7152 * env[..., 1] + 0.0722 * env[..., 2]
    lum = np.where(np.isfinite(lum), np.maximum(lum, 0.0), 0.0)
    az = lum[:, :C].copy()
    az[:, 0] = np.maximum(az[:, 0], lum[:, C])                                 # texel column We-1 is azimuth 0
    rows = np.maximum(np.maximum(az[np.clip(np.arange(He) - 1, 0, He - 1)], az), az[np.clip(np.arange(He) + 1, 0, He - 1)])
    m = np.maximum(np.maximum(np.roll(rows, 1, axis=1), rows), np.roll(rows, -1, axis=1))
    omega = cell_solid_angle(He, We)
    w = m * omega[:, None]
    rw = w.sum(1)
    if not rw.sum() > 0:
        w = np.broadcast_to(omega[:, None], (He, C)).copy()
        rw = w.sum(1)
    cc = np.zeros((He, We))
    cc[:, 1:] = np.cumsum(w, 1) / np.where(rw > 0, rw, 1.0)[:, None]
    cc[rw <= 0, 1:] = np.arange(1, We) / C
    cc = cc.astype(np.float32).astype(np.float64)
    cc[:, 0], cc[:, C] = 0.0, 1.0
    rc = np.zeros(He + 1)
    rc[1:] = np.cumsum(rw) / rw.sum()
    rc = rc.astype(np.float32).astype(np.float64)
    rc[0], rc[He] = 0.0, 1.0
    lo, _ = bands(He)
    vs, cv = np.empty(He + 1), np.empty(He + 1)
    vs[0], vs[He], cv[0], cv[He] = 0.0, 2.0, 2.0, 0.0
    vs[1:He], cv[1:He] = 2 * np.sin(lo[1:] / 2) ** 2, 2 * np.cos(lo[1:] / 2) ** 2
    f32 = lambda x: x.astype(np.float32).astype(np.float64)
    pdf = np.diff(rc)[:, None] * np.diff(cc, axis=1) / omega[:, None]
    return dict(He=He, We=We, row_cdf=rc, vers=f32(vs), covers=f32(cv), col_cdf=cc, pdf=pdf, weight=w)


def from_gpu_table(t, He, We):
    """The same dict from a GPU table (r3dg_env_sampler_build's floats)."""
    t = np.asarray(t, dtype=np.float32)
    o = 4 + 2 * He
    rc, vs, cv = (t[o + k * (He + 1):o + (k + 1) * (He + 1)].astype(np.float64) for k in range(3))
    o += 3 * (He + 1)
    cc = t[o:o + He * We].reshape(He, We)
    pdf = t[o + He * We:].reshape(He, We - 1)
    return dict(He=He, We=We, row_cdf=rc, vers=vs, covers=cv, col_cdf=cc.astype(np.float64), pdf=pdf.astype(np.float64))


def _find(cdf, u):
    """the largest k in [0, len(cdf) - 2] with cdf[k] <= u"""
    return np.clip(np.searchsorted(cdf, u, side="right") - 1, 0, len(cdf) - 2)


def env_cell(tab, e):
    """(row, column) of the cells of env-space directions e [...,3], and the distance (radians) to the nearest edge."""
    He, We = tab["He"], tab["We"]
    dt, dp = math.pi / (He - 1), 2 * math.pi / (We - 1)
    th = np.arccos(np.clip(e[..., 2] / np.linalg.norm(e, axis=-1), -1, 1))
    c = (math.pi - np.arctan2(e[..., 1], e[..., 0])) / dp
    j = np.clip(np.floor(th / dt + 0.5), 0, He - 1).astype(int)
    i = np.floor(c + 0.5).astype(int) % (We - 1)
    fr = th / dt + 0.5
    dth = np.abs(fr - np.round(fr)) * dt
    fc = c + 0.5
    dph = np.abs(fc - np.round(fc)) * dp * np.sin(th)
    return j, i, np.minimum(dth, dph)


def env_sample(tab, T, u1, u2):
    He, We = tab["He"], tab["We"]
    j = _find(tab["row_cdf"], u1)
    rc = tab["row_cdf"]
    t1 = (u1 - rc[j]) / (rc[j + 1] - rc[j])
    cc = tab["col_cdf"][j]
    i = np.array([_find(c, u) for c, u in zip(cc.reshape(-1, We), u2.reshape(-1))]).reshape(u2.shape)
    c0, c1 = np.take_along_axis(cc, i[..., None], -1)[..., 0], np.take_along_axis(cc, i[..., None] + 1, -1)[..., 0]
    t2 = (u2 - c0) / (c1 - c0)
    vs, cv = tab["vers"], tab["covers"]
    v = vs[j] + t1 * (vs[j + 1] - vs[j])                   # northern rows: 1 - cos theta; southern: 1 + cos theta
    w = cv[j] + t1 * (cv[j + 1] - cv[j])
    north = 2 * j <= He - 1
    cz = np.where(north, 1 - v, w - 1)
    sz = np.sqrt(np.maximum(np.where(north, v * (2 - v), w * (2 - w)), 0))
    az = math.pi - (i - 0.5 + t2) * (2 * math.pi / (We - 1))
    e = np.stack([sz * np.cos(az), sz * np.sin(az), cz], -1)
    return e if T is None else e @ np.asarray(T, dtype=np.float64)          # T^T e as rows


def env_pdf(tab, T, d):
    e = d if T is None else d @ np.asarray(T, dtype=np.float64).T
    j, i, _ = env_cell(tab, e)
    return tab["pdf"][j, i]


# ---- GGX and cosine ---------------------------------------------------------------------------------------------------
def normalize(x):
    return x / np.maximum(np.linalg.norm(x, axis=-1, keepdims=True), 1e-12)


def rotate_from_z(n, s):
    """rotate_from_z: n [...,3] unit, s [...,3] -> the rotation taking +z to n applied to s (normalised)."""
    ax, ay, nz = -n[..., 1], n[..., 0], n[..., 2]
    c = np.maximum(nz + 1, 1e-7)
    x = (1 - ay * ay / c) * s[..., 0] + (ax * ay / c) * s[..., 1] + ay * s[..., 2]
    y = (ax * ay / c) * s[..., 0] + (1 - ax * ax / c) * s[..., 1] - ax * s[..., 2]
    z = -ay * s[..., 0] + ax * s[..., 1] + (1 - (ay * ay + ax * ax) / c) * s[..., 2]
    out = np.stack([x, y, z], -1)
    out = np.where((nz + 1 > 0)[..., None], out, -s)
    return normalize(out)


def ggx_frame(n, v, r):
    V = normalize(v)
    Ns = n * np.sign((n * V).sum(-1, keepdims=True))
    return V, Ns, np.maximum(np.asarray(r, dtype=np.float64) ** 4, 1e-7)   # Ns = 0 when n.V = 0: no lobe


def ggx_sample(V, Ns, a2, u1, u2):
    """V, Ns [M,1,3], a2 [M,1]; u [M,n] -> (l [M,n,3], ok [M,n])."""
    den = 1 + (a2 - 1) * u1
    sh, ch = np.sqrt(a2 * u1 / den), np.sqrt((1 - u1) / den)
    ph = 2 * math.pi * u2
    h = rotate_from_z(np.broadcast_to(Ns, u1.shape + (3,)), np.stack([sh * np.cos(ph), sh * np.sin(ph), ch], -1))
    vh = (V * h).sum(-1)
    lobe = np.abs(np.broadcast_to(Ns, h.shape)).sum(-1) > 0
    return normalize(2 * vh[..., None] * h - V), (vh > 0) & lobe


def ggx_pdf(V, Ns, a2, l):
    h = normalize(V + l)
    nh, vh = (Ns * h).sum(-1), (V * h).sum(-1)
    D = a2 / (math.pi * ((np.cross(np.broadcast_to(Ns, h.shape), h) ** 2).sum(-1) + a2 * nh * nh) ** 2)
    return np.where((nh > 0) & (vh > 0), D * nh / (4 * np.where(vh > 0, vh, 1.0)), 0.0)


def cos_sample(n, u1, u2):
    r, ph = np.sqrt(u1), 2 * math.pi * u2
    return rotate_from_z(np.broadcast_to(n, u1.shape + (3,)), np.stack([r * np.cos(ph), r * np.sin(ph), np.sqrt(1 - u1)], -1))


def cos_pdf(n, d):
    return np.maximum((n * d).sum(-1), 0) / math.pi


def sample(tab, T, normals, N, n_env, n_ggx, seed, q=None, viewdirs=None, roughness=None):
    """The sampler at M points: normals [M,3] (normalised here), viewdirs [M,3] and roughness [M] for GGX, q [M]
    (default 0..M-1).  Returns (dirs [M,N,3], areas [M,N], edge distance of the env cell [M,N] in radians)."""
    n = normalize(np.asarray(normals, dtype=np.float64))
    M = n.shape[0]
    q = np.arange(M) if q is None else np.asarray(q)
    n_cos = N - n_env - n_ggx
    parts, oks = [], []
    V = Ns = a2 = None
    if n_ggx > 0:
        V, Ns, a2 = ggx_frame(n, np.asarray(viewdirs, dtype=np.float64), roughness)
        V, Ns, a2 = V[:, None], Ns[:, None], np.asarray(a2).reshape(M, 1)
    for s, ns in enumerate((n_env, n_ggx, n_cos)):
        if ns == 0:
            continue
        u1, u2 = lattice(seed, q, s, ns)
        if s == 0:
            parts.append(env_sample(tab, T, u1, u2)); oks.append(np.ones_like(u1, dtype=bool))
        elif s == 1:
            l, ok = ggx_sample(V, Ns, a2, u1, u2)
            parts.append(l); oks.append(ok)
        else:
            parts.append(cos_sample(n[:, None], u1, u2)); oks.append(np.ones_like(u1, dtype=bool))
    d, ok = np.concatenate(parts, 1), np.concatenate(oks, 1)
    den = np.zeros(d.shape[:2])
    if n_env > 0:
        den = den + n_env * env_pdf(tab, T, d)
    if n_ggx > 0:
        den = den + n_ggx * ggx_pdf(V, Ns, a2, d)
    den = den + n_cos * cos_pdf(n[:, None], d)
    good = ok & (den > 0) & np.isfinite(den)
    area = np.where(good, N / np.where(good, den, 1.0), 0.0)
    e = d if T is None else d @ np.asarray(T, dtype=np.float64).T
    return d, area, env_cell(tab, e)[2]


# ---- the quality scene: a plane under a small bright source (test_pixel_shading_gpu's) --------------------------------
def plane_env():
    env = np.full((64, 128, 3), 0.05)
    env[14:17, 40:44] = 60.0
    return env


def plane_pixel(H=48, W=64, y=None, x=None):
    """(point, normal, campos) of pixel (y, x) of the 48 x 64 plane (default: the centre)."""
    y = H // 2 if y is None else y
    x = W // 2 if x is None else x
    ys, xs = np.linspace(-1, 1, H), np.linspace(-1.4, 1.4, W)
    return np.array([xs[x], ys[y], 0.0]), np.array([0.0, 0.0, 1.0]), np.array([0.0, -0.6, 1.2])


def env_lookup(env, d):
    """grid_sample(align_corners=True, zeros) of env at directions d [...,3] (the shading step's point lookup)."""
    He, We = env.shape[:2]
    ix = (1 - np.arctan2(d[..., 1], d[..., 0]) / math.pi) / 2 * (We - 1)
    iy = (np.arccos(np.clip(d[..., 2], -1, 1)) - 1e-6) / math.pi * (He - 1)
    x0, y0 = np.floor(ix), np.floor(iy)
    out = np.zeros(d.shape[:-1] + (3,))
    for dx in (0, 1):
        for dy in (0, 1):
            xs, ys = x0 + dx, y0 + dy
            w = (1 - np.abs(ix - xs)) * (1 - np.abs(iy - ys))
            ok = (xs >= 0) & (xs < We) & (ys >= 0) & (ys < He)
            tex = env[np.clip(ys, 0, He - 1).astype(int), np.clip(xs, 0, We - 1).astype(int)]
            out += np.where(ok[..., None], tex * w[..., None], 0.0)
    return out


def ggx_brdf(n, v, l, rough):
    """GGX_specular of neilf.py: n, v [3], l [...,3], rough scalar -> [...,1]."""
    L, V = normalize(l), normalize(v)
    H = normalize((L + V) / 2)
    Nn = n / np.linalg.norm(n) * np.sign(np.dot(V, n / np.linalg.norm(n)))
    NoL = np.clip((Nn * L).sum(-1, keepdims=True), 1e-6, 1)
    NoV = np.clip(np.dot(Nn, V), 1e-6, 1)
    NoH = np.clip((Nn * H).sum(-1, keepdims=True), 1e-6, 1)
    VoH = np.clip((V * H).sum(-1, keepdims=True), 1e-6, 1)
    a2 = (rough * rough) ** 2
    k = (rough * rough + 2 * rough + 1) / 8
    frac = (0.04 + 0.96 * np.power(2.0, (-5.55473 * VoH - 6.98316) * VoH)) * a2
    nom = np.clip(4 * math.pi * (NoH * NoH * (a2 - 1) + 1) ** 2 * (NoV * (1 - k) + k) * (NoL * (1 - k) + k), 1e-6, 4 * math.pi)
    return frac / nom


def integrand(env, p, n, campos, base, rough, d):
    """(f_d + f_s) L (n.d)+ [...,3] at directions d [...,3] (visibility 1)."""
    fs = ggx_brdf(n, campos - p, d, rough)
    ndl = np.maximum((d * n).sum(-1, keepdims=True), 0)
    return (base / math.pi + fs) * env_lookup(env, d) * ndl


def estimate(env, p, n, campos, base, rough, d, area):
    """the shading step's estimator mean_i (f_d + f_s) L_i area_i (n.d_i)+ at one point: d [N,3], area [N] -> [3]"""
    return (integrand(env, p, n, campos, base, rough, d) * area[:, None]).mean(0)


def truth(env, p, n, campos, base, rough, nt=1500, nphi=3000):
    """The hemisphere integral by midpoint quadrature in (theta, phi) around +z (n must be +z)."""
    th = (np.arange(nt) + 0.5) * (math.pi / 2 / nt)
    ph = (np.arange(nphi) + 0.5) * (2 * math.pi / nphi)
    acc = np.zeros(3)
    for k in range(0, nt, 100):                           # in slabs of theta, to bound the memory
        t = th[k:k + 100, None]
        d = np.stack([np.sin(t) * np.cos(ph), np.sin(t) * np.sin(ph), np.cos(t) * np.ones_like(ph)], -1)
        w = np.sin(t) * (math.pi / 2 / nt) * (2 * math.pi / nphi)
        acc += (integrand(env, p, n, campos, base, rough, d) * w[..., None]).sum((0, 1))
    return acc


def fibonacci_dirs(n, N):
    """the Fibonacci sampler's N directions around unit n [3] (area 2 pi each)"""
    i = np.arange(N)
    z = np.maximum(1 - 2 * i / (2 * N - 1), math.sin(math.radians(10)))
    r = np.sqrt(1 - z * z)
    th = i * math.pi * (3 - math.sqrt(5))
    s = np.stack([np.sin(th) * r, np.cos(th) * r, z], -1)
    return rotate_from_z(np.broadcast_to(n, s.shape), s)
