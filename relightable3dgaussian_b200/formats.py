"""SURVEY.md §8(f)4 — the reference's two on-disk formats, as far as the hot path needs them: to stream a model
between ranks / runs and to persist the baked visibility instead of re-tracing it on every start
(scene/gaussian_model.py:312-342 re-bakes in `train.py` / `eval_*.py`).

  * checkpoint  `chkpnt<iter>.pth` = `torch.save((model.capture(), iteration), path)` (train.py:192-193) with the list
    layout of `GaussianModel.capture` (scene/gaussian_model.py:114-142): 15 fixed entries + 6 PBR entries;
  * point cloud `point_cloud.ply` written by `GaussianModel.save_ply` (:507-561): one binary little-endian `vertex`
    element, float32 properties named by `construct_list_of_attributes` (:507-533), SH-like tensors flattened
    channel-major (`transpose(1, 2).flatten(1)`).

Host-side Python like the reference's own (numpy + torch; the reference uses `plyfile`, which only wraps this header +
record layout).  Models are plain dicts of tensors keyed like the reference's optimizer groups: xyz, normal, f_dc,
f_rest, opacity, scaling, rotation [, base_color, roughness, incidents_dc, incidents_rest, visibility_dc,
visibility_rest].  `save_bake` / `load_bake` add what the reference never persists: the baked `[P,N,*]` tensors."""
import os

import numpy as np
import torch

GEOMETRY = ("xyz", "normal", "f_dc", "f_rest", "opacity", "scaling", "rotation")
PBR = ("base_color", "roughness", "incidents_dc", "incidents_rest", "visibility_dc", "visibility_rest")
_CHANNEL_MAJOR = ("f_dc", "f_rest", "incidents_dc", "incidents_rest", "visibility_dc", "visibility_rest")   # stored [P,K,C]
_PLY_PREFIX = dict(xyz=("x", "y", "z"), normal=("nx", "ny", "nz"), f_dc="f_dc_", f_rest="f_rest_", opacity=("opacity",),
                   scaling="scale_", rotation="rot_", base_color="base_color_", roughness=("roughness",),
                   incidents_dc="incidents_dc_", incidents_rest="incidents_rest_", visibility_dc="visibility_dc_",
                   visibility_rest="visibility_rest_")


def _keys(model):
    return GEOMETRY + (PBR if all(k in model for k in PBR) else ())


def attribute_names(model):
    """== GaussianModel.construct_list_of_attributes (scene/gaussian_model.py:507-533)."""
    names = []
    for k in _keys(model):
        t = model[k]
        width = int(np.prod(t.shape[1:]))
        pre = _PLY_PREFIX[k]
        names += list(pre) if isinstance(pre, tuple) else [f"{pre}{i}" for i in range(width)]
    return names


def save_ply(path, model):
    """== GaussianModel.save_ply (:535-561): binary little-endian PLY, one float32 property per attribute."""
    d = os.path.dirname(path)
    if d:
        os.makedirs(d, exist_ok=True)
    cols = []
    for k in _keys(model):
        t = model[k].detach().float().cpu()
        if k in _CHANNEL_MAJOR:
            t = t.transpose(1, 2)                                  # [P,K,C] -> [P,C,K]: channel-major flattening
        cols.append(t.reshape(t.shape[0], -1).contiguous().numpy())
    attrs = np.ascontiguousarray(np.concatenate(cols, axis=1).astype("<f4"))
    names = attribute_names(model)
    assert attrs.shape[1] == len(names)
    header = "ply\nformat binary_little_endian 1.0\nelement vertex %d\n" % attrs.shape[0]
    header += "".join(f"property float {n}\n" for n in names) + "end_header\n"
    with open(path, "wb") as f:
        f.write(header.encode("ascii"))
        f.write(attrs.tobytes())


def _read_ply(path):
    with open(path, "rb") as f:
        if f.readline().strip() != b"ply":
            raise ValueError("not a PLY file")
        fmt, n, names, in_vertex = None, 0, [], False
        while True:
            line = f.readline()
            if not line:
                raise ValueError("truncated PLY header")
            tok = line.decode("ascii").split()
            if not tok or tok[0] == "comment":
                continue
            if tok[0] == "format":
                fmt = tok[1]
            elif tok[0] == "element":
                in_vertex = tok[1] == "vertex"
                if in_vertex:
                    n = int(tok[2])
            elif tok[0] == "property" and in_vertex:
                if tok[1] not in ("float", "float32"):
                    raise ValueError(f"unsupported property type {tok[1]} (the reference writes float32 only)")
                names.append(tok[2])
            elif tok[0] == "end_header":
                break
        if fmt == "binary_little_endian":
            data = np.frombuffer(f.read(n * len(names) * 4), dtype="<f4").reshape(n, len(names))
        elif fmt == "ascii":
            data = np.loadtxt(f, dtype=np.float32, max_rows=n).reshape(n, len(names))
        else:
            raise ValueError(f"unsupported PLY format {fmt}")
    return names, data


def load_ply(path, max_sh_degree=3, use_pbr=None, device="cpu"):
    """== GaussianModel.load_ply (:568-666): dict of float32 tensors in the model's layouts
    (f_dc [P,1,3], f_rest [P,(D+1)^2-1,3], incidents like the SHs, visibility_dc [P,1,1], visibility_rest [P,15,1])."""
    names, data = _read_ply(path)
    col = {n: i for i, n in enumerate(names)}

    def numbered(prefix):
        ks = sorted((n for n in names if n.startswith(prefix)), key=lambda x: int(x.split("_")[-1]))
        return data[:, [col[k] for k in ks]]

    def sh_like(prefix, channels, coeffs):
        flat = numbered(prefix)
        assert flat.shape[1] == channels * coeffs, (prefix, flat.shape, channels, coeffs)
        return torch.from_numpy(flat.reshape(-1, channels, coeffs).copy()).transpose(1, 2).contiguous()

    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32))
    K = (max_sh_degree + 1) ** 2
    m = dict(xyz=t(data[:, [col["x"], col["y"], col["z"]]]), normal=t(data[:, [col["nx"], col["ny"], col["nz"]]]),
             f_dc=sh_like("f_dc_", 3, 1), f_rest=sh_like("f_rest_", 3, K - 1), opacity=t(data[:, [col["opacity"]]]),
             scaling=t(numbered("scale_")), rotation=t(numbered("rot")))
    has_pbr = "roughness" in col
    if use_pbr is None:
        use_pbr = has_pbr
    if use_pbr:
        if not has_pbr:
            raise ValueError("PLY has no PBR attributes")
        m.update(base_color=t(numbered("base_color")), roughness=t(data[:, [col["roughness"]]]),
                 incidents_dc=sh_like("incidents_dc_", 3, 1), incidents_rest=sh_like("incidents_rest_", 3, K - 1),
                 visibility_dc=sh_like("visibility_dc_", 1, 1), visibility_rest=sh_like("visibility_rest_", 1, 4 ** 2 - 1))
    return {k: v.to(device) for k, v in m.items()}


# ---- checkpoint tuple (scene/gaussian_model.py:114-142 capture, :144-183 restore; train.py:192-193) -------------------
_STATS = ("max_radii2D", "weights_accum", "xyz_gradient_accum", "normal_gradient_accum", "denom")


def capture(model, stats, optimizer_state, active_sh_degree=3, spatial_lr_scale=1.0):
    """The list `GaussianModel.capture()` returns: [active_sh_degree, xyz, normal, f_dc, f_rest, scaling, rotation,
    opacity, max_radii2D, weights_accum, xyz_gradient_accum, normal_gradient_accum, denom, optimizer.state_dict(),
    spatial_lr_scale (+ base_color, roughness, incidents_dc, incidents_rest, visibility_dc, visibility_rest)]."""
    out = [active_sh_degree, model["xyz"], model["normal"], model["f_dc"], model["f_rest"], model["scaling"], model["rotation"],
           model["opacity"]] + [stats[k] for k in _STATS] + [optimizer_state, spatial_lr_scale]
    if all(k in model for k in PBR):
        out += [model[k] for k in PBR]
    return out


def restore(captured):
    """Inverse of `capture`: (model dict, stats dict, optimizer state dict, active_sh_degree, spatial_lr_scale)."""
    if len(captured) < 15:
        raise ValueError("not a Relightable3DGaussian checkpoint list")
    deg, xyz, normal, f_dc, f_rest, scaling, rotation, opacity = captured[:8]
    model = dict(xyz=xyz, normal=normal, f_dc=f_dc, f_rest=f_rest, opacity=opacity, scaling=scaling, rotation=rotation)
    stats = dict(zip(_STATS, captured[8:13]))
    if len(captured) > 15:
        model.update(zip(PBR, captured[15:21]))
    return model, stats, captured[13], deg, captured[14]


def save_checkpoint(path, captured, iteration):
    torch.save((captured, iteration), path)                       # train.py:192-193


def load_checkpoint(path, map_location="cpu"):
    captured, iteration = torch.load(path, map_location=map_location, weights_only=False)
    return captured, iteration


# ---- the baked visibility (never persisted by the reference: 11.5 GB and a BVH bake per start at config #4) ------------
def save_bake(path, visibility, incident_dirs, incident_areas=None):
    """visibility [P,N,1] is in {0} U [0.9, 1]; incident_dirs are a pure function of the normals (r3dg_sample_incident_dirs)
    and areas are the constant 2*pi, so only the visibility (fp16 is exact enough? no — kept fp32) and N are essential;
    directions are stored on request for callers that do not want to regenerate them."""
    payload = {"format": "r3dg_b200.bake.v1", "sample_num": int(visibility.shape[1]), "visibility": visibility.detach().cpu()}
    if incident_dirs is not None:
        payload["incident_dirs"] = incident_dirs.detach().cpu()
    if incident_areas is not None:
        payload["incident_areas"] = incident_areas.detach().cpu()
    torch.save(payload, path)


def load_bake(path, normals=None, device="cpu"):
    """-> (visibility, incident_dirs, incident_areas); missing directions are regenerated from `normals` with the
    sampling kernel (GPU only)."""
    p = torch.load(path, map_location="cpu", weights_only=False)
    if p.get("format") != "r3dg_b200.bake.v1":
        raise ValueError("not a baked-visibility file")
    vis = p["visibility"].to(device)
    dirs, areas = p.get("incident_dirs"), p.get("incident_areas")
    if dirs is None:
        if normals is None:
            raise ValueError("the file holds no directions: pass the model's normals to regenerate them")
        from .raytracer import sample_incident_rays
        dirs, areas = sample_incident_rays(normals, False, p["sample_num"])
    else:
        dirs = dirs.to(device)
        areas = areas.to(device) if areas is not None else torch.full_like(vis, 2 * np.pi)
    return vis, dirs, areas


def save_mesh_ply(path, verts, faces, colors=None):
    """A triangle mesh (e.g. tsdf.TSDFVolume.extract) as a binary little-endian PLY that mesh tools read: a `vertex`
    element of float x, y, z (and uchar red, green, blue when `colors` [N,3] in [0, 1] is given, rounded and clamped)
    and a `face` element of `list uchar int vertex_indices`.  verts [N,3], faces [F,3] with indices in [0, N)."""
    v = verts.detach().cpu().numpy() if isinstance(verts, torch.Tensor) else np.asarray(verts)
    fc = faces.detach().cpu().numpy() if isinstance(faces, torch.Tensor) else np.asarray(faces)
    if v.ndim != 2 or v.shape[1] != 3:
        raise ValueError(f"save_mesh_ply: verts must be [N,3] (got {v.shape})")
    if fc.ndim != 2 or fc.shape[1] != 3 or not (fc.size == 0 or np.issubdtype(fc.dtype, np.integer)):
        raise ValueError(f"save_mesh_ply: faces must be integer [F,3] (got {fc.shape}, {fc.dtype})")
    if fc.size and (fc.min() < 0 or fc.max() >= v.shape[0]):
        raise ValueError(f"save_mesh_ply: face indices outside [0, {v.shape[0]})")
    fields = [("x", "<f4"), ("y", "<f4"), ("z", "<f4")]
    if colors is not None:
        c = colors.detach().cpu().numpy() if isinstance(colors, torch.Tensor) else np.asarray(colors)
        if c.shape != v.shape:
            raise ValueError(f"save_mesh_ply: colors must be [N,3] like verts (got {c.shape})")
        fields += [("red", "u1"), ("green", "u1"), ("blue", "u1")]
    vrec = np.empty(v.shape[0], dtype=fields)
    for i, n in enumerate("xyz"):
        vrec[n] = v[:, i]
    if colors is not None:
        c8 = np.clip(np.rint(np.nan_to_num(c.astype(np.float64)) * 255.0), 0, 255).astype(np.uint8)
        for i, n in enumerate(("red", "green", "blue")):
            vrec[n] = c8[:, i]
    frec = np.empty(fc.shape[0], dtype=[("n", "u1"), ("i", "<i4", (3,))])
    frec["n"] = 3
    frec["i"] = fc
    header = "ply\nformat binary_little_endian 1.0\nelement vertex %d\n" % v.shape[0]
    header += "".join(f"property {'float' if t == '<f4' else 'uchar'} {n}\n" for n, t in fields)
    header += "element face %d\nproperty list uchar int vertex_indices\nend_header\n" % fc.shape[0]
    d = os.path.dirname(path)
    if d:
        os.makedirs(d, exist_ok=True)
    with open(path, "wb") as f:
        f.write(header.encode("ascii"))
        f.write(vrec.tobytes())
        f.write(frec.tobytes())
