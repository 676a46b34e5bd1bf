"""TSDF fusion and marching cubes without a GPU: the table in csrc/mc_table.cuh (generated, crack-free, consistently
wound), the fp64 oracle on random fields and on fused analytic spheres, every host-side refusal of tsdf.py, and
formats.save_mesh_ply."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import tsdf_oracle as O
from helpers import ROOT
from relightable3dgaussian_b200 import formats, synth, tsdf

VS = 2.4 / 95                 # 96^3 points over [-1.2, 1.2]^3
ORIGIN = (-1.2, -1.2, -1.2)
DIMS = (96, 96, 96)


def test_header_is_generator_output():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "gen_mc_table.py"), "--check"])
    assert r.returncode == 0, "csrc/mc_table.cuh differs from tools/gen_mc_table.py's output"


def _face_segments(tris, cube):
    """Boundary segments of the cell's triangles (directed edges used once), grouped by the cube face they lie on."""
    edges, _, _ = O.parse_table()
    de = O.directed_edges(tris[cube][(tris[cube] >= 0).all(axis=1)]) if (tris[cube] >= 0).any() else np.zeros((0, 2), int)
    keys = {tuple(e) for e in de}
    bnd = [e for e in keys if (e[1], e[0]) not in keys]
    mid = lambda e: np.array([(edges[e][0] >> a & 1) + (edges[e][1] >> a & 1) for a in range(3)]) / 2.0
    out = {}
    for a, b in bnd:
        pa, pb = mid(a), mid(b)
        for d in range(3):
            for s in (0.0, 1.0):
                if pa[d] == s and pb[d] == s:
                    out.setdefault((d, int(s)), set()).add((a, b))
    return out


def test_table_faces_agree_between_neighbours():
    """Crack-freeness: for every pair of cells that share a face, the segments each draws on it coincide and run in
    opposite directions, for all 256 x 256 configurations whose shared corners agree."""
    edges, count, tris = O.parse_table()
    assert count.max() <= tris.shape[1] and all((tris[c] >= 0).all(axis=1).sum() == count[c] for c in range(256))
    segs = [_face_segments(tris, c) for c in range(256)]
    for d in range(3):
        bit = 1 << d
        lo = [c for c in range(8) if not c & bit]            # corners on the face d = 0
        # edge on the face d = 1 of the lower cell -> the same grid edge on the face d = 0 of the upper cell
        emap = {}
        for e, (a, b) in enumerate(edges):
            if a & bit and b & bit:
                emap[e] = int(np.nonzero([(x == a ^ bit and y == b ^ bit) for x, y in edges])[0][0])
        for c_lo in range(256):
            for c_up in range(256):
                if any(((c_lo >> (c | bit)) & 1) != ((c_up >> c) & 1) for c in lo):
                    continue
                s_lo = {(emap[a], emap[b]) for a, b in segs[c_lo].get((d, 1), set())}
                s_up = {(b, a) for a, b in segs[c_up].get((d, 0), set())}
                assert s_lo == s_up, (d, c_lo, c_up)


def _random_field(rng, n=12):
    f = rng.standard_normal((n, n, n)).astype(np.float32)
    f[rng.random(f.shape) < 0.15] = 0.0                      # exact zeros (outside: tsdf < 0 is inside)
    f[[0, -1], :, :] = np.abs(f[[0, -1], :, :]) + 0.1         # positive on the border: a closed surface
    f[:, [0, -1], :] = np.abs(f[:, [0, -1], :]) + 0.1
    f[:, :, [0, -1]] = np.abs(f[:, :, [0, -1]]) + 0.1
    return f


def test_random_fields_give_closed_oriented_manifolds():
    rng = np.random.default_rng(0)
    table = O.parse_table()
    seen = np.zeros(256, dtype=bool)
    genus0 = 0
    for trial in range(60):
        f = _random_field(rng)
        w = np.ones_like(f)
        v, fc, _ = O.marching_cubes(f, w, None, (0, 0, 0), 1.0, table)
        cube = np.zeros((11, 11, 11), dtype=np.int64)
        for c in range(8):
            a, b, d = c & 1, (c >> 1) & 1, (c >> 2) & 1
            cube |= (f[a:11 + a, b:11 + b, d:11 + d] < 0).astype(np.int64) << c
        seen[np.unique(cube)] = True
        assert O.is_closed_oriented_manifold(fc), trial
        assert O.vertex_links_are_cycles(fc), trial
        assert len(np.unique(fc)) == len(v), "unreferenced vertex"
        # a noise field's inside set has handles (a ring of inside points bounds a torus), so each component is a
        # closed orientable surface of some genus g: chi = 2 - 2g, even and at most 2.  The genus-0 meshes below
        # (fused spheres) pin chi = 2 per component.
        chis = O.euler_per_component(len(v), fc)
        assert all(c <= 2 and c % 2 == 0 for c in chis.values()), (trial, chis)
        assert sum(chis.values()) == O.euler(len(v), fc)
        genus0 += sum(c == 2 for c in chis.values())
    assert seen.all(), f"{(~seen).sum()} cube configurations never occurred"
    assert genus0 > 0


def _fuse(spheres, cams=None):
    cams = cams or O.ring_cameras()
    dep = np.stack([O.sphere_depth(c, spheres) for c in cams]).astype(np.float32)
    t, w, _, _ = O.integrate(np.ones(DIMS, np.float32), np.zeros(DIMS, np.float32), None, ORIGIN, VS, 4 * VS, dep,
                             None, O.cam_rows(cams))
    return O.marching_cubes(t.astype(np.float32), w.astype(np.float32), None, ORIGIN, VS)


def test_sphere_mesh():
    v, f, _ = _fuse([((0.0, 0.0, 0.0), 0.8)])
    assert len(v) == 19040
    assert O.is_closed_oriented_manifold(f) and O.vertex_links_are_cycles(f)
    assert O.euler(len(v), f) == 2 and O.components(len(v), f) == 1
    assert O.signed_volume(v, f) > 0                          # outward winding
    err = np.abs(np.linalg.norm(v, axis=1) - 0.8) / VS
    assert err.max() < 0.5, err.max()


def test_two_spheres_mesh():
    v, f, _ = _fuse([((-0.55, 0.0, 0.0), 0.4), ((0.55, 0.0, 0.0), 0.4)])
    assert O.is_closed_oriented_manifold(f) and O.vertex_links_are_cycles(f)
    assert O.components(len(v), f) == 2 and O.euler(len(v), f) == 4
    assert O.signed_volume(v, f) > 0


# ---- host-side refusals (no device is touched) ---------------------------------------------------------------------

def _settings(V=2, W=32, H=24):
    return [synth.make_camera(k, W, H) for k in range(V)]


def test_volume_refusals():
    with pytest.raises(ValueError, match="bbox_min"):
        tsdf.TSDFVolume((0, 0), (1, 1, 1), 0.1, 0.4, device="cpu")
    with pytest.raises(ValueError, match="bbox_max"):
        tsdf.TSDFVolume((0, 0, 0), (1, math.nan, 1), 0.1, 0.4, device="cpu")
    with pytest.raises(ValueError, match="must exceed"):
        tsdf.TSDFVolume((0, 0, 0), (1, 0, 1), 0.1, 0.4, device="cpu")
    for vs in (0.0, -1.0, math.inf, math.nan):
        with pytest.raises(ValueError, match="voxel_size"):
            tsdf.TSDFVolume((0, 0, 0), (1, 1, 1), vs, 0.4, device="cpu")
    for st in (0.0, -0.1, math.inf, math.nan):
        with pytest.raises(ValueError, match="sdf_trunc"):
            tsdf.TSDFVolume((0, 0, 0), (1, 1, 1), 0.1, st, device="cpu")
    with pytest.raises(ValueError, match="2\\^31"):
        tsdf.TSDFVolume((0, 0, 0), (1, 1, 1), 1 / 1400, 0.4, device="cpu")
    with pytest.raises(TypeError, match="color"):
        tsdf.TSDFVolume((0, 0, 0), (1, 1, 1), 0.1, 0.4, color="yes", device="cpu")
    vol = tsdf.TSDFVolume((-1.2,) * 3, (1.2,) * 3, VS, 4 * VS, device="cpu")
    assert vol.dims == DIMS and tuple(vol.tsdf.shape) == DIMS and tuple(vol.color.shape) == DIMS + (3,)
    assert (vol.tsdf == 1).all() and (vol.weight == 0).all() and (vol.color == 0).all()
    assert tsdf.TSDFVolume((0, 0, 0), (0.05, 0.05, 0.05), 0.1, 0.4, color=False, device="cpu").dims == (2, 2, 2)


def test_integrate_refusals():
    V, H, W = 2, 24, 32
    s = _settings(V, W, H)
    vol = tsdf.TSDFVolume((-1,) * 3, (1,) * 3, 0.25, 0.5, device="cpu")
    d, c = torch.ones(V, 1, H, W), torch.zeros(V, 3, H, W)
    with pytest.raises(TypeError, match="float32"):
        vol.integrate(d.double(), s, c)
    with pytest.raises(ValueError, match=r"\[V,1,H,W\]"):
        vol.integrate(d[:, 0], s, c)
    with pytest.raises(ValueError, match="views per call"):
        vol.integrate(torch.ones(65, 1, 2, 2), s * 33, torch.zeros(65, 3, 2, 2))
    with pytest.raises(ValueError, match="empty"):
        vol.integrate(torch.ones(V, 1, 0, W), s, torch.zeros(V, 3, 0, W))
    with pytest.raises(ValueError, match="required exactly"):
        vol.integrate(d, s)
    with pytest.raises(ValueError, match="required exactly"):
        tsdf.TSDFVolume((-1,) * 3, (1,) * 3, 0.25, 0.5, color=False, device="cpu").integrate(d, s, c)
    with pytest.raises(TypeError, match="float32"):
        vol.integrate(d, s, c.double())
    with pytest.raises(ValueError, match=r"\[V,3,H,W\]"):
        vol.integrate(d, s, c[:, :2])
    with pytest.raises(ValueError, match="settings for"):
        vol.integrate(d, s[:1], c)
    with pytest.raises(ValueError, match="the maps are"):
        vol.integrate(d, _settings(V, W + 1, H), c)
    with pytest.raises(ValueError, match="tanfovx / tanfovy"):
        vol.integrate(d, [s[0], s[1]._replace(tanfovx=0.0)], c)
    with pytest.raises(ValueError, match="non-finite"):
        vol.integrate(d, [s[0], s[1]._replace(cx=math.nan)], c)
    with pytest.raises(ValueError, match="non-finite"):
        vol.integrate(d, [s[0], s[1]._replace(tanfovy=math.inf)], c)
    for dt in (0.0, -1.0, math.nan):
        with pytest.raises(ValueError, match="depth_trunc"):
            vol.integrate(d, s, c, depth_trunc=dt)
    with pytest.raises(ValueError, match="contiguous float32"):
        bad = tsdf.TSDFVolume((-1,) * 3, (1,) * 3, 0.25, 0.5, device="cpu")
        bad.weight = bad.weight.double()
        bad.integrate(d, s, c)
    with pytest.raises(ValueError, match="CUDA"):             # every host check passed: only the device is missing
        vol.integrate(d, s, c, depth_trunc=3.0)
    with pytest.raises(ValueError, match="CUDA"):
        vol.integrate(d[:1], s[0], c[:1])                      # one settings object stands for V = 1
    with pytest.raises(ValueError, match="CUDA"):
        vol.extract()


# ---- PLY -----------------------------------------------------------------------------------------------------------

def _parse_mesh_ply(path):
    with open(path, "rb") as f:
        assert f.readline() == b"ply\n"
        assert f.readline() == b"format binary_little_endian 1.0\n"
        elems, cur = [], None
        while True:
            tok = f.readline().decode("ascii").split()
            if tok[0] == "end_header":
                break
            if tok[0] == "element":
                cur = (tok[1], int(tok[2]), [])
                elems.append(cur)
            elif tok[0] == "property":
                cur[2].append(tuple(tok[1:]))
        (vn, nv, vprops), (fn, nf, fprops) = elems
        assert vn == "vertex" and fn == "face" and fprops == [("list", "uchar", "int", "vertex_indices")]
        dt = [(p[1], {"float": "<f4", "uchar": "u1"}[p[0]]) for p in vprops]
        v = np.frombuffer(f.read(nv * np.dtype(dt).itemsize), dtype=dt)
        fr = np.frombuffer(f.read(nf * 13), dtype=[("n", "u1"), ("i", "<i4", (3,))])
        assert f.read() == b""
    assert (fr["n"] == 3).all()
    return v, fr["i"]


def test_save_mesh_ply_round_trip(tmp_path):
    rng = np.random.default_rng(1)
    verts = torch.from_numpy(rng.standard_normal((7, 3)).astype(np.float32))
    faces = torch.tensor([[0, 1, 2], [2, 3, 4], [4, 5, 6], [6, 0, 3]], dtype=torch.int32)
    colors = torch.tensor(rng.random((7, 3)), dtype=torch.float32)
    colors[0] = torch.tensor([-0.5, 1.5, 0.5])
    p = os.path.join(tmp_path, "sub", "mesh.ply")
    formats.save_mesh_ply(p, verts, faces, colors)
    v, f = _parse_mesh_ply(p)
    assert v.dtype.names == ("x", "y", "z", "red", "green", "blue")
    assert np.array_equal(np.stack([v["x"], v["y"], v["z"]], 1), verts.numpy())
    assert np.array_equal(f, faces.numpy())
    rgb = np.stack([v["red"], v["green"], v["blue"]], 1)
    assert np.array_equal(rgb, np.clip(np.rint(colors.double().numpy() * 255), 0, 255).astype(np.uint8))
    assert tuple(rgb[0]) == (0, 255, 128)
    formats.save_mesh_ply(p, verts.numpy(), faces.numpy())
    v, f = _parse_mesh_ply(p)
    assert v.dtype.names == ("x", "y", "z") and np.array_equal(f, faces.numpy())
    formats.save_mesh_ply(p, torch.zeros(0, 3), torch.zeros(0, 3, dtype=torch.int32))
    v, f = _parse_mesh_ply(p)
    assert len(v) == 0 and len(f) == 0
    with pytest.raises(ValueError, match="outside"):
        formats.save_mesh_ply(p, verts, faces + 5)
    with pytest.raises(ValueError, match="integer"):
        formats.save_mesh_ply(p, verts, faces.float())
    with pytest.raises(ValueError, match="colors"):
        formats.save_mesh_ply(p, verts, faces, colors[:3])
